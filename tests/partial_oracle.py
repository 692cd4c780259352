"""use_partial_classes on the CPU oracle (models.py:807-828 single image, :2267-2289 batch graph).

The full 81-class box head runs; then its label logits are gathered at [0] + ids and its box logits at ids - 1 of the
[K, 80, 4] layout (after the class-agnostic tile, models.py:798-802), and the post-processing runs over len(ids) + 1
classes, so final labels are 1..len(ids) in the order of ids.  The mask head keeps its 80 channels and final_masks picks
channel (partial label - 1) of them, as the reference's gather_nd on the full mask logits does (models.py:954-958).

oracle.frcnn.forward and forward_multi (and the mask path inside forward) call frcnn.fastrcnn_head; inside
`partial_classes(ids)` that name is a head that applies the gather to the full head's outputs.  The gather works on the
logits, after the head, as the reference's graph does -- independent of the engine, which packs the selected weight
columns at load time instead."""
import contextlib

import numpy as np

from oracle import frcnn


def gather(cls_logits, box_logits, ids):
    """cls_logits [K, 81], box_logits [K, 80, 4] -> [K, len(ids) + 1], [K, len(ids), 4]."""
    ids = np.asarray(ids, np.int64)
    return (np.ascontiguousarray(cls_logits[:, np.concatenate([[0], ids])]),
            np.ascontiguousarray(box_logits[:, ids - 1]))


@contextlib.contextmanager
def partial_classes(ids):
    full = frcnn.fastrcnn_head

    def head(feat, W, cfg):
        cls, box, hidden = full(feat, W, cfg)
        return gather(cls, box, ids) + (hidden,)

    frcnn.fastrcnn_head = head
    try:
        yield
    finally:
        frcnn.fastrcnn_head = full
