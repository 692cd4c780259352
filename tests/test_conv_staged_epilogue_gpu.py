"""The staged conv epilogue (results through shared-memory slots and TMA stores, the residual prefetched by TMA) against
a plain PyTorch fp32 conv.  b2_op_conv2d writes dense fp16 planes with an unshifted residual, so every case here takes
the staged path; the cases cover the tile edges the slot ring has to get right."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# name: (B, H, W, Cin, Cout, R, relu, residual)
CASES = {
    "res_ragged_m_dead_half": (1, 13, 23, 256, 256, 1, 1, True),    # M=299: last tile has 43 rows (one warpgroup idle)
    "res_ragged_m":           (2, 10, 10, 64, 128, 1, 1, True),     # M=200: last tile has 72 rows, K = 1 K-block
    "res_cout80":             (1, 12, 20, 256, 80, 1, 1, True),     # block_n 128, second chunk clipped at column 80
    "res_cout15":             (1, 12, 20, 64, 15, 1, 0, True),      # block_n 64, Cout_pad 16
    "res_bn64":               (1, 16, 24, 256, 64, 1, 1, True),     # block_n 64, 4 K-blocks
    "res_many_tiles":         (1, 92, 160, 128, 512, 1, 1, True),   # 460 tiles on 132 SMs: the residual ring wraps
    "res_many_tiles_bn64":    (2, 50, 60, 64, 64, 1, 1, True),      # 47 tiles of one chunk each
    "res_3x3":                (1, 23, 40, 64, 128, 3, 1, True),
    "no_res_many_tiles":      (1, 92, 160, 256, 256, 1, 1, False),  # single-slot ring, two chunks per tile
    "no_res_3x3":             (2, 20, 28, 64, 80, 3, 1, False),
    "swish_res":              (1, 16, 24, 256, 128, 1, 2, True),    # relu == 2: the EfficientDet instantiations
    "swish_no_res":           (1, 20, 30, 64, 64, 1, 2, False),
}


def reference(spec, seed):
    B, H, W, Cin, Cout, R, relu, use_res = spec
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, H, W, Cin)).astype(np.float32)
    w = (rng.standard_normal((R, R, Cin, Cout)) / np.sqrt(R * R * Cin)).astype(np.float32)
    bias = rng.standard_normal(Cout).astype(np.float32)
    p = R // 2
    ref = F.conv2d(torch.from_numpy(x).permute(0, 3, 1, 2), torch.from_numpy(w).permute(3, 2, 0, 1).contiguous(),
                   torch.from_numpy(bias), padding=p)
    res = None
    if use_res:
        res = rng.standard_normal((B, H, W, Cout)).astype(np.float32)
        ref = ref + torch.from_numpy(res).permute(0, 3, 1, 2)
    if relu == 1:
        ref = torch.relu(ref)
    elif relu == 2:
        ref = ref * torch.sigmoid(ref)
    return x, w, bias, res, ref.permute(0, 2, 3, 1).contiguous().numpy()


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("split,tol", [(True, 2e-5), (False, 3e-3)])
def test_staged_epilogue_matches_torch_fp32(name, split, tol):
    from object_detection_tracking_b200 import engine
    spec = CASES[name]
    x, w, bias, res, ref = reference(spec, seed=len(name))
    R = spec[5]
    out = engine.op_conv2d(x, w, bias, res, pad=(R // 2,) * 4, relu=spec[6], impl="tcgen05", split=split)
    assert out.shape == ref.shape
    assert np.isfinite(out).all()
    assert np.abs(out - ref).max() <= tol * np.abs(ref).max()
