"""use_bg_score on the CPU oracle (models.py:1263-1270, single-image graph only).

fastrcnn_predictions first drops every row whose argmax over `probs` [K, C] is column 0 and runs the per-class NMS and
the top-k over the K' kept rows, in their original order.  pred_indices[:, 0] is then a row's rank j among the kept rows,
and the caller gathers the UNFILTERED decoded boxes with it (models.py:925-930, and :888-889 in the small-object branch):
a detection's box is its class's box of ROI j, while its label and probability are the selected ROI i's.  The oracle keeps
that quirk; fpn_box_feat and final_masks follow the boxes.

tf.argmax leaves ties and NaN unspecified; the oracle assumes (as SURVEY.md Appendix B does for other TF ops) a scan that
moves only to a strictly greater value: ties go to the lowest column, so a row whose background equals its best class is
dropped, and a NaN never wins, so an all-NaN row has argmax 0.

`use_bg_score()` swaps oracle.frcnn.fastrcnn_predictions for the filtered one, so oracle.frcnn.forward, head_postprocess and
so_oracle.branch compose with it (as partial_oracle.partial_classes does for the head).  The batch graph's
fastrcnn_predictions_multi is not touched: it has no filter (models.py:2924-2976).  `literal()` transcribes the reference op
by op; the CPU tests check the efficient path against it."""
import contextlib

import numpy as np

from oracle import frcnn, tf_ops

F32 = np.float32
_UNFILTERED = frcnn.fastrcnn_predictions


def argmax(x):
    """tf.argmax(x, axis=1) of [K, C] under the oracle's assumption: first column of the maximum, NaN never greater."""
    x = np.asarray(x, F32)
    best = x[:, 0].copy()
    arg = np.zeros(x.shape[0], np.int64)
    for c in range(1, x.shape[1]):
        up = x[:, c] > best
        best = np.where(up, x[:, c], best)
        arg[up] = c
    return arg


def bg_rank(probs, count=None):
    """[K] int32: row i's rank among the rows below `count` (default all) whose argmax is not column 0, else -1."""
    probs = np.asarray(probs, F32)
    K = probs.shape[0]
    n = K if count is None else int(count)
    keep = np.zeros(K, bool)
    keep[:n] = argmax(probs[:n]) > 0
    rank = np.full(K, -1, np.int32)
    rank[keep] = np.arange(int(keep.sum()), dtype=np.int32)
    return rank


def fastrcnn_predictions(boxes, probs, cfg):
    """frcnn.fastrcnn_predictions over the non-background rows: (pred_indices [R, 2] = (rank j, class), probs [R])."""
    keep = np.nonzero(argmax(probs) > 0)[0]
    return _UNFILTERED(np.asarray(boxes)[keep], np.asarray(probs)[keep], cfg)


@contextlib.contextmanager
def use_bg_score():
    frcnn.fastrcnn_predictions = fastrcnn_predictions
    try:
        yield
    finally:
        frcnn.fastrcnn_predictions = _UNFILTERED


def final_outputs(boxes, probs, cfg):
    """(final_boxes [R, 4], final_labels [R] int64, final_probs [R]) of the filtered selection, boxes gathered from the
    unfiltered [K, C-1, 4] at the filtered index."""
    pred, fp = fastrcnn_predictions(boxes, probs, cfg)
    fb = np.asarray(boxes)[pred[:, 0], pred[:, 1]] if len(pred) else np.zeros((0, 4), F32)
    return fb.astype(F32), (pred[:, 1] + 1).astype(np.int64), np.asarray(fp, F32)


def literal(boxes, probs, cfg, no_score_filter=False):
    """models.py:1263-1304 then :925-932, one reference op at a time.  boxes [K, C-1, 4] (the caller's decoded_boxes),
    probs [K, C].  Returns (final_boxes, final_labels, final_probs)."""
    decoded_boxes = np.asarray(boxes, F32)
    probs = np.asarray(probs, F32)
    boxes = decoded_boxes
    # box_classes = tf.argmax(probs, axis=1)
    box_classes = argmax(probs)
    # nonBG_box_indices = tf.reshape(tf.where(tf.greater(box_classes, 0)), [-1])
    nonBG_box_indices = np.argwhere(box_classes > 0).reshape(-1)
    # probs = tf.gather(probs, nonBG_box_indices); boxes = tf.gather(boxes, nonBG_box_indices)
    probs = np.take(probs, nonBG_box_indices, axis=0)
    boxes = np.take(boxes, nonBG_box_indices, axis=0)
    # boxes = tf.transpose(boxes, [1, 0, 2]); probs = tf.transpose(probs[:, 1:], [1, 0])
    boxes = np.transpose(boxes, (1, 0, 2))
    probs = np.transpose(probs[:, 1:], (1, 0))
    # masks = tf.map_fn(nms_return_masks[_no_score_filter], (probs, boxes))   (models.py:1202-1238)
    masks = np.zeros(probs.shape, bool)
    for c in range(probs.shape[0]):
        prob, box = probs[c], boxes[c]
        if no_score_filter:
            selection = tf_ops.non_max_suppression(box, prob, cfg.result_per_im, cfg.fastrcnn_nms_iou_thres)
        else:
            ids = np.argwhere(prob > F32(cfg.result_score_thres)).reshape(-1)
            selection = tf_ops.non_max_suppression(np.take(box, ids, axis=0), np.take(prob, ids),
                                                   cfg.result_per_im, cfg.fastrcnn_nms_iou_thres)
            selection = np.take(ids, selection).astype(np.int32)
        sorted_selection = np.sort(np.asarray(selection, np.int64))          # -top_k(-selection)
        masks[c, sorted_selection] = True                                    # sparse_to_dense
    # selected_indices = tf.where(masks)   [N, 2] = (class, row), row-major
    selected_indices = np.argwhere(masks)
    # probs = tf.boolean_mask(probs, masks)
    probs = probs[masks]
    # topk_probs, topk_indices = tf.nn.top_k(probs, tf.minimum(result_per_im, tf.size(probs)))
    topk_probs, topk_indices = tf_ops.top_k(probs, min(cfg.result_per_im, probs.size))
    # filtered_selection = tf.reverse(tf.gather(selected_indices, topk_indices), axis=[1])
    filtered_selection = np.take(selected_indices, topk_indices, axis=0).reshape(-1, 2)[:, ::-1]
    pred_indices = filtered_selection
    # final_boxes = tf.gather_nd(decoded_boxes, pred_indices): the UNFILTERED boxes
    final_boxes = decoded_boxes[pred_indices[:, 0], pred_indices[:, 1]].reshape(-1, 4)
    # final_labels = tf.add(pred_indices[:, 1], 1)
    final_labels = (pred_indices[:, 1] + 1).astype(np.int64)
    return final_boxes.astype(F32), final_labels, np.asarray(topk_probs, F32)


def background_shift(cls_logits):
    """A shift of the background logit (column 0 of `cls_logits` [K, C]) that drops about half of the rows: the middle of
    the widest gap between the middle third's background-minus-best margins, so that no row sits near the tie."""
    lg = np.asarray(cls_logits, np.float64)
    m = np.sort(lg[:, 0] - lg[:, 1:].max(1))
    n = len(m)
    mid = m[n // 3:max(n - n // 3, n // 3 + 2)]
    g = int(np.argmax(np.diff(mid)))
    return F32(-(mid[g] + mid[g + 1]) / 2)


def with_background_shift(W, shift, name="fastrcnn/outputs/class/b"):
    """A copy of the weights with `shift` added to the background entry of the bias `name`."""
    W = dict(W)
    b = np.array(W[name], F32)
    b[0] += F32(shift)
    W[name] = b
    return W


def min_background_margin(probs):
    """The smallest |background - best class| of the rows' probabilities [K, C]."""
    p = np.asarray(probs, np.float64)
    return float(np.abs(p[:, 0] - p[:, 1:].max(1)).min()) if len(p) else np.inf
