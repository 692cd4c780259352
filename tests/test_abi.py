"""The C-ABI library loads without a GPU and exports exactly what include/b200det.h declares."""
import os
import re

import pytest

from object_detection_tracking_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "b200det.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b2_[a-z0-9_]+)\s*\(", src)))


def test_library_loads_and_exports_every_declared_symbol():
    lib = _lib.load()
    names = header_functions()
    assert "b2_detect_host" in names and "b2_cosine_cost" in names
    for n in names:
        assert hasattr(lib, n), "missing export %s" % n
    assert sorted(s[0] for s in _lib.SYMBOLS) == names
    assert lib.b2_version() == 1


def _header_struct_words(name):
    src = open(os.path.join(ROOT, "include", "b200det.h")).read()
    head = "typedef struct %s {" % name
    body = src[src.index(head) + len(head):src.index("} %s;" % name)]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    n = 0
    for decl in body.split(";"):
        decl = decl.strip()
        m = re.match(r"(int32_t|int|float)\s+(.*)", decl)
        if not m:
            continue
        for var in m.group(2).split(","):
            dims = [int(k) for k in re.findall(r"\[(\d+)\]", var)]
            n += int(__import__("numpy").prod(dims)) if dims else 1
    return n


def test_config_structs_match_header_size():
    import ctypes
    assert ctypes.sizeof(_lib.B2Config) == 4 * _header_struct_words("b2_config")
    assert ctypes.sizeof(_lib.B2EffdetConfig) == 4 * _header_struct_words("b2_effdet_config")
    assert ctypes.sizeof(_lib.B2ConvView) == 4 * _header_struct_words("b2_conv_view")


def test_compute_entry_points_fail_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from object_detection_tracking_b200.config import make_config
    from object_detection_tracking_b200.engine import Detector
    with pytest.raises(RuntimeError):
        Detector(make_config(), 1, 64, 64)
