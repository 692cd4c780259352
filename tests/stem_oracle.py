"""numpy references of the ResNet stems' ingest (csrc/stem.cu): the frame normalisations, the detector's compact 16-lane
operand and the ReID engines' 64-lane operand, and the 7x7 stride-2 conv + BatchNorm + ReLU they feed, in float64 with an
element-wise error bound.

The packs are written from the index formulas of stem.cu, not from its kernels:
  V[b][y][x][ry*6 + sx*3 + c]          = P[b][2y + ry - 3][2x + sx - 3][c]          (detector, lanes 12..15 zero)
  U[b][y][q][s*12 + ry*6 + sx*3 + c]   = P[b][2y + ry - 3][2(q + s) + sx - 3][c]    (ReID, lanes 48..63 zero)
with P the normalised frame and zero outside it.  tests/test_stem_oracle_cpu.py pins this module against oracle/frcnn.py
and torch; tests/test_stem_kernels_gpu.py checks the kernels and the engines' stems against it."""
import numpy as np
import torch
import torch.nn.functional as F

import conv_oracle as co
import elementwise_oracle as eo

# models.py:345-355: the detector's frames are BGR, so its constants are the ImageNet ones reversed
DET_MEAN = np.array([0.485, 0.456, 0.406][::-1], np.float32)
DET_STD = np.array([0.229, 0.224, 0.225][::-1], np.float32)
# torchvision Normalize of the ReID extractor (feature_extractor.py:190-196), RGB crops
REID_MEAN = np.array([0.485, 0.456, 0.406], np.float32)
REID_STD = np.array([0.229, 0.224, 0.225], np.float32)

TF_BN_EPS = 1e-5      # nn.py:1723 (oracle.frcnn.BN_EPS)
TORCH_BN_EPS = 1e-5   # nn.BatchNorm2d default
K_GEMM = 256          # the stem conv as the engines run it: a 4x1 conv over 64-lane pixels


def normalize(frame, mode):
    """The frame normalised in float32, one rounding per op as the kernels do it.  mode "detector": x * float32(1/255),
    - mean, / std with BGR constants; mode "reid": x / 255, - mean, / std with RGB constants (ToTensor + Normalize)."""
    x = np.asarray(frame).astype(np.float32)
    if mode == "detector":
        x = x * np.float32(1.0 / 255)
        return (x - DET_MEAN) / DET_STD
    assert mode == "reid", mode
    x = x / np.float32(255)
    return (x - REID_MEAN) / REID_STD


def _taps(P, Hu, Wx):
    """tap[ry][sx] [B][Hu][Wx][3] = P[b][2y + ry - 3][2x + sx - 3][c], zero outside P."""
    P = np.asarray(P)
    B, H, W, _ = P.shape
    Pp = np.zeros((B, 3 + max(H, 2 * Hu), 3 + max(W, 2 * Wx), 3), P.dtype)
    Pp[:, 3:3 + H, 3:3 + W] = P
    return [[Pp[:, ry:ry + 2 * Hu:2, sx:sx + 2 * Wx:2][:, :Hu, :Wx] for sx in range(2)] for ry in range(2)]


def pack16(P, Hu, Wv):
    """The detector's operand [B][Hu][Wv][16] of the normalised frame P [B][H][W][3]."""
    t = _taps(P, Hu, Wv)
    V = np.zeros(P.shape[:1] + (Hu, Wv, 16), np.asarray(P).dtype)
    for ry in range(2):
        for sx in range(2):
            V[..., ry * 6 + sx * 3:ry * 6 + sx * 3 + 3] = t[ry][sx]
    return V


def pack64(P, Hu, Wu):
    """The ReID engines' operand [B][Hu][Wu][64] of the normalised frame P [B][H][W][3]."""
    t = _taps(P, Hu, Wu + 3)
    U = np.zeros(P.shape[:1] + (Hu, Wu, 64), np.asarray(P).dtype)
    for s in range(4):
        for ry in range(2):
            for sx in range(2):
                k = s * 12 + ry * 6 + sx * 3
                U[..., k:k + 3] = t[ry][sx][:, :, s:s + Wu]
    return U


def detector_pads(H, W, mult=32):
    """nn.py:871-877 with tf_pad_reverse: [3, 2 + pad-to-mult] on each axis -> (top, bottom, left, right)."""
    return 3, 2 + (-H) % mult, 3, 2 + (-W) % mult


REID_PADS = (3, 3, 3, 3)   # torchvision's conv1: 7x7 stride 2, padding 3


def out_hw(H, W, pads):
    return (H + pads[0] + pads[1] - 7) // 2 + 1, (W + pads[2] + pads[3] - 7) // 2 + 1


def held(frame, mode, split=True):
    """The normalised frame as the operand planes hold it, float64: hi + lo/2048 exactly (split), hi (fp16)."""
    return co.represent(normalize(frame, mode), split)


def bn_fold(bn):
    """bn = (gamma, beta, mean, var, eps) -> (scale, shift) in float64, the engines' fold_bn: gamma / sqrt(var + eps),
    beta - mean * scale.  None -> no norm (scale 1, shift 0)."""
    if bn is None:
        return None, None
    g, b, m, v, eps = bn
    scale = np.asarray(g, np.float64) / np.sqrt(np.asarray(v, np.float64) + eps)
    return scale, np.asarray(b, np.float64) - np.asarray(m, np.float64) * scale


def _conv(x, w, pads):
    """float64 7x7 stride-2 VALID conv of NHWC x after zero padding pads = (t, b, l, r), HWIO w."""
    xt = torch.from_numpy(np.ascontiguousarray(x, np.float64)).permute(0, 3, 1, 2)
    xt = F.pad(xt, (pads[2], pads[3], pads[0], pads[1]))
    wt = torch.from_numpy(np.ascontiguousarray(w, np.float64)).permute(3, 2, 0, 1).contiguous()
    return F.conv2d(xt, wt, stride=2).permute(0, 2, 3, 1).numpy()


def stem_conv64(frame, W, bn, pads, mode, split=True, relu=True):
    """The stem of frame [B][H][W][3] in float64: the frame normalised in fp32 by `mode` as the planes hold it (mode None:
    `frame` is already the normalised input, taken as is), zero padded by pads = (t, b, l, r), 7x7 stride-2 VALID conv
    with HWIO W [7][7][3][Cout], BatchNorm bn = (gamma, beta, mean, var, eps) (None: none), ReLU when relu.

    Returns dict(ref, pre, bound, shift32): pre is the output before the ReLU, shift32 the fp32 bias an all-padding window
    gives, and bound bounds |engine output - ref| element-wise for the engines' conv (conv_tc, split or fp16 precision).
    The engines fold the BatchNorm into the weights (W * scale rounded to fp32, then their planes) and the bias
    (shift rounded to fp32); the error of those roundings is taken exactly, conv(|x~|, |W~ - W scale|) + |shift32 -
    shift|, and the conv kernel's own arithmetic is conv_oracle.bound's at K = 256."""
    if mode is None:
        x32 = None
        xr = np.asarray(frame, np.float64)
    else:
        x32 = normalize(frame, mode)
        xr = co.represent(x32, split)
    W64 = np.asarray(W, np.float32).astype(np.float64)
    Cout = W64.shape[3]
    scale, shift = bn_fold(bn)
    if scale is None:
        scale, shift = np.ones(Cout), np.zeros(Cout)
    Wf = (W64 * scale).astype(np.float32)             # the engines' folded weights, as uploaded
    Wr = co.represent(Wf, split)
    conv = _conv(xr, W64, pads)
    pre = conv * scale + shift
    ref = np.maximum(pre, 0.0) if relu else pre
    shift32 = shift.astype(np.float32)
    S = _conv(np.abs(xr), np.abs(Wr), pads)
    L = _conv(co.lo_part(x32), co.lo_part(Wf), pads) if (split and x32 is not None) else None
    Ew = _conv(np.abs(xr), np.abs(Wr - W64 * scale), pads) + np.abs(shift32.astype(np.float64) - shift)
    b = np.broadcast_to(np.abs(shift32.astype(np.float64)), S.shape)
    bound = co.bound(K_GEMM, S, b, 0.0, ref, "split" if split else "fp16", L=L, relu=int(relu))
    bound = bound + Ew * (1 + 2.0 ** -10)
    return dict(ref=ref, pre=pre, bound=bound, shift32=shift32, S=S)


def padding_only(H, W, pads, hw):
    """Masks (rows, cols) of the stem outputs whose 7x7 window reads no pixel of the frame."""
    Ho, Wo = hw
    rows = np.array([not (2 * p + 6 >= pads[0] and 2 * p <= pads[0] + H - 1) for p in range(Ho)])
    cols = np.array([not (2 * q + 6 >= pads[2] and 2 * q <= pads[2] + W - 1) for q in range(Wo)])
    return rows, cols


def det_bn(Wt, name="conv0"):
    """The detector's BatchNorm arrays of `name` (Tensorpack names) as stem_conv64's bn."""
    return (Wt[name + "/bn/gamma"], Wt[name + "/bn/beta"], Wt[name + "/bn/mean/EMA"], Wt[name + "/bn/variance/EMA"],
            TF_BN_EPS)


def torch_bn(state, prefix):
    """A torch BatchNorm2d's arrays of a state dict as stem_conv64's bn."""
    return tuple(np.asarray(state[prefix + k]) for k in (".weight", ".bias", ".running_mean", ".running_var")) + \
        (TORCH_BN_EPS,)


def oihw_to_hwio(w):
    return np.ascontiguousarray(np.asarray(w, np.float32).transpose(2, 3, 1, 0))


def raw_planes(v, split):
    """uint16 planes of fp32 v (lo None in fp16 precision)."""
    return eo.raw(np.asarray(v, np.float32), split)
