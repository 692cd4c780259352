"""CPU-side checks of the ReID layer: synthetic state_dict layout, all-gather exchange (gloo, world 2)."""
import json
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from object_detection_tracking_b200.synth import osnet_param_shapes, synth_osnet_state


def test_osnet_state_layout_and_param_count():
    shapes = osnet_param_shapes()
    n_params = sum(int(np.prod(s)) for k, s in shapes.items() if "running_" not in k)
    # torchreid osnet_x1_0 with a 1-class classifier has 2 170 021 params (SURVEY 8c); classifier = 512 + 1
    assert n_params == 2170021 - 513
    st = synth_osnet_state(1)
    assert set(st) == set(shapes) and st["conv3.0.conv1.conv.weight"].shape == (96, 256, 1, 1)
    assert all(v.dtype == np.float32 for v in st.values())
    np.testing.assert_array_equal(st["fc.0.weight"], synth_osnet_state(1)["fc.0.weight"])


def _reference_shapes(golden_dir, model):
    """State-dict shapes of the reference's torchreid model (tests/golden/make_golden.py: torchreid_state_shapes)."""
    with open(os.path.join(golden_dir, "torchreid_state_shapes.json")) as f:
        return {k: tuple(v) for k, v in json.load(f)[model].items()}


def test_state_layout_matches_reference_model(golden_dir):
    assert _reference_shapes(golden_dir, "osnet_x1_0") == {k: tuple(v) for k, v in osnet_param_shapes().items()}


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    from object_detection_tracking_b200.reid import allgather_gallery
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    local = torch.full((3 + 2 * rank, 8), float(rank + 1))
    allf, counts = allgather_gallery(local)
    q.put((rank, counts, allf.shape[0], float(allf[:3].mean()), float(allf[3:].mean())))
    dist.barrier()
    dist.destroy_process_group()


def test_gallery_allgather_world2_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for r in res:
        assert r[1] == [3, 5] and r[2] == 8 and r[3] == 1.0 and r[4] == 2.0    # ragged galleries, rank order


def test_resnet101_reid_state_layout_and_param_count():
    from object_detection_tracking_b200.synth import resnet101_reid_param_shapes, synth_resnet101_reid_state
    shapes = resnet101_reid_param_shapes()
    n_params = sum(int(np.prod(s)) for k, s in shapes.items() if "running_" not in k)
    assert n_params == 44549160 - 2048 * 1000 - 1000          # torchvision resnet101 minus its 1000-way fc
    assert shapes["layer3.22.conv2.weight"] == (256, 256, 3, 3) and shapes["layer2.0.downsample.0.weight"] == (512, 256, 1, 1)
    assert "layer1.1.downsample.0.weight" not in shapes
    a = synth_resnet101_reid_state(7)["layer4.2.conv3.weight"]
    assert a.dtype == np.float32 and a.shape == (2048, 512, 1, 1)


def test_resnet101_state_layout_matches_reference_model(golden_dir):
    from object_detection_tracking_b200.synth import resnet101_reid_param_shapes
    assert _reference_shapes(golden_dir, "resnet101") == {k: tuple(v) for k, v in resnet101_reid_param_shapes().items()}
