"""Batched EfficientDet, the parts that need no GPU: the C ABI, the config struct and the batch-mode model object."""
import ctypes
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest

from object_detection_tracking_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _config(**over):
    c = dict(is_efficientdet=True, efficientdet_modelname="efficientdet-d0", short_edge_size=128, max_size=256,
             result_score_thres=1e-4, result_per_im=100, is_load_from_pb=False)
    c.update(over)
    return SimpleNamespace(**c)


def test_batch_entry_points_are_declared_and_exported():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b200det.h")).read(), flags=re.S)
    lib = _lib.load()
    for name in ("b2_effdet_detect_batch", "b2_effdet_replay"):
        assert re.search(r"\b%s\s*\(" % name, src), name
        assert hasattr(lib, name) and name in [s[0] for s in _lib.SYMBOLS]


def test_batch_is_the_last_config_field():
    src = open(os.path.join(ROOT, "include", "b200det.h")).read()
    body = src[src.index("typedef struct b2_effdet_config {"):src.index("} b2_effdet_config;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert [d.strip() for d in body.split(";") if d.strip()][-1] == "int batch"
    assert _lib.B2EffdetConfig._fields_[-1] == ("batch", ctypes.c_int32)
    assert _lib.B2EffdetConfig.batch.offset == ctypes.sizeof(_lib.B2EffdetConfig) - 4
    assert _lib.B2EffdetConfig().batch == 0                       # zero-initialised callers get a batch-1 context


def test_python_config_carries_the_batch():
    from object_detection_tracking_b200.effdet import _c_config
    from object_detection_tracking_b200.effdet_config import make_effdet_config
    cfg = make_effdet_config("efficientdet-d0", 128, 256)
    assert _c_config(cfg, "split", "efficientnet-b0").batch == 1
    assert _c_config(cfg, "fp16", "efficientnet-b0", 4).batch == 4


def test_get_model_returns_the_batch_surface():
    from object_detection_tracking_b200.backend import EfficientDet, EfficientDet_multi, get_model
    multi = get_model(_config(), is_multi=True)
    assert isinstance(multi, EfficientDet_multi) and multi.is_multi
    assert multi.final_valid_indices.name == "final_valid_indices:0"
    fd = multi.get_feed_dict_forward_multi([np.zeros((4, 6, 3), np.uint8), np.zeros((8, 5, 3), np.uint8)])
    assert [f.shape for f in fd[multi.image]] == [(4, 6, 3), (8, 5, 3)]     # frames of a batch may differ in size
    single = get_model(_config(), is_multi=False)
    assert type(single) is EfficientDet and not single.is_multi
    assert not hasattr(single, "final_valid_indices") and not hasattr(single, "get_feed_dict_forward_multi")


def test_batched_entry_point_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from object_detection_tracking_b200.effdet import EffdetEngine
    from object_detection_tracking_b200.effdet_config import make_effdet_config
    lib = _lib.load()
    frames = (ctypes.c_void_p * 1)()
    assert lib.b2_effdet_detect_batch(None, frames, None, None, 1, *([None] * 7)) == -1
    assert b"null argument" in lib.b2_last_error()
    cfg = make_effdet_config("efficientdet-d0", 128, 256, fpn_cell_repeats=1, box_class_repeats=1)
    with pytest.raises(RuntimeError, match="b2_effdet_create"):
        EffdetEngine(cfg, {}, backbone="efficientnet-b0", batch=2)
    from object_detection_tracking_b200.backend import Session, get_model
    model = get_model(_config(), is_multi=True)
    model.set_weights({})
    with pytest.raises(RuntimeError, match="b2_effdet_create"):
        Session().run([model.final_boxes], feed_dict=model.get_feed_dict_forward_multi([np.zeros((4, 4, 3), np.uint8)]))
    with pytest.raises(ValueError):
        EffdetEngine(cfg, {}, batch=0)
