"""Float64 references of the element-wise and reduction kernels around the GEMMs -- the depthwise convs, the pools, the
BiFPN node combine, MBConv's squeeze-excite, OSNet's channel gate and 4-stream sum, EfficientNet's stem im2col -- written
plainly from each op's semantics, and the fp16 plane format the kernels hold activations in.

tests/test_elementwise_oracle_cpu.py pins every function here against an independent implementation (torch ops and the
project's CPU oracles); tests/test_elementwise_kernels_gpu.py checks the kernels against them.  The *_f32 functions
restate a kernel's float32 arithmetic in its own operation order, for the outputs that must match bit for bit."""
import numpy as np
from scipy.special import expit

LO_SCALE = 2048.0
U = 2.0 ** -24              # fp32 unit roundoff (round to nearest)
PLANE_REL = 2.0 ** -22      # relative error of storing a value as split planes (hi + lo/2048)
PLANE_ABS = 2.0 ** -36      # ... plus this absolute error where lo is an fp16 subnormal
FP16_REL = 2.0 ** -11       # relative error of storing a value as the hi plane alone (fp16 precision)
FP16_ABS = 2.0 ** -25       # ... plus this absolute error where hi is an fp16 subnormal


# ---- the plane format --------------------------------------------------------------------------------------------
def planes(x, split=True):
    """fp32 x -> its (hi, lo) fp16 planes exactly as planes.cuh splits: hi = fp16(x), lo = fp16((x - hi) * 2048) with the
    difference and the product in fp32.  lo is None in fp16 precision (split false)."""
    x = np.asarray(x, np.float32)
    hi = x.astype(np.float16)
    if not split:
        return hi, None
    lo = ((x - hi.astype(np.float32)) * np.float32(LO_SCALE)).astype(np.float16)
    return hi, lo


def value(hi, lo=None):
    """The fp32 value the kernels read from planes: hi + lo/2048 rounded once (their fmaf).  The float64 sum is exact
    (hi and lo/2048 span fewer than 53 bits), so rounding it to fp32 is that one rounding."""
    v = hi.astype(np.float64)
    if lo is not None:
        v = v + lo.astype(np.float64) / LO_SCALE
    return v.astype(np.float32)


def representable(x, split=True):
    """x moved to a value the planes hold exactly (the value of x's planes): v = representable(x) satisfies
    value(*planes(v)) == v bit for bit, so a test input built with it is exactly what the kernel reads, and a kernel that
    copies or re-splits such a value stores planes(v).  One round trip is not always enough: a value halfway between two
    fp16 numbers, or -0 (whose lo is +0, so that it reads back as +0), moves once more and then stays."""
    return value(*planes(value(*planes(x, split)), split))


def raw(x, split=True):
    """The planes of fp32 x as uint16 bit patterns (lo None in fp16 precision): what a bit-exact kernel output holds."""
    hi, lo = planes(x, split)
    return hi.view(np.uint16), None if lo is None else lo.view(np.uint16)


def joined(hi, lo=None):
    """The value of raw uint16 planes in float64 (exact)."""
    v = hi.view(np.float16).astype(np.float64)
    return v if lo is None else v + lo.view(np.float16).astype(np.float64) / LO_SCALE


def store_bound(v, split=True):
    """Bound on |planes value - v| when the kernel stores v: 2^-22 |v| (+ 2^-36) split, 2^-11 |v| (+ 2^-25) in fp16."""
    v = np.abs(np.asarray(v, np.float64))
    return PLANE_REL * v + PLANE_ABS if split else FP16_REL * v + FP16_ABS


# ---- activations ---------------------------------------------------------------------------------------------------
def sigmoid(x):
    return expit(np.asarray(x, np.float64))


def swish(x):
    x = np.asarray(x, np.float64)
    return x * expit(x)


def relu(x):
    return np.maximum(np.asarray(x, np.float64), 0.0)


# ---- depthwise convs -----------------------------------------------------------------------------------------------
def same_pad(n, k, s):
    """TF 'SAME' along one axis: (output size ceil(n / s), pad before = max((out - 1) s + k - n, 0) // 2)."""
    out = -(-n // s)
    return out, max((out - 1) * s + k - n, 0) // 2


def _window_taps(x, K, stride, pad_t, pad_l, Ho, Wo, fill):
    """For x [B][H][W][C]: an iterator of (r, s, tap) with tap [B][Ho][Wo][C] = x[b][y*stride - pad_t + r]
    [x*stride - pad_l + s][c], `fill` outside the map."""
    B, H, W, C = x.shape
    pb = max(0, (Ho - 1) * stride + K - pad_t - H)
    pr = max(0, (Wo - 1) * stride + K - pad_l - W)
    xp = np.full((B, pad_t + H + pb, pad_l + W + pr, C), fill, np.float64)
    xp[:, pad_t:pad_t + H, pad_l:pad_l + W] = x
    for r in range(K):
        for s in range(K):
            yield r, s, xp[:, r:r + (Ho - 1) * stride + 1:stride, s:s + (Wo - 1) * stride + 1:stride]


def depthwise(x, w, bias=None, stride=1, pad=(0, 0), out_hw=None):
    """Depthwise conv of x [B][H][W][C] with w [K][K][C]: out[b][y][x][c] = bias[c] + sum_{r,s} x[b][y*stride - pad_t + r]
    [x*stride - pad_l + s][c] w[r][s][c], zero outside the map.  Returns (out, S) in float64 with S = |bias| + sum |x w|
    the magnitude the rounding error scales with."""
    x = np.asarray(x, np.float64)
    w = np.asarray(w, np.float64)
    K = w.shape[0]
    Ho, Wo = out_hw if out_hw is not None else x.shape[1:3]
    b = np.zeros(x.shape[3]) if bias is None else np.asarray(bias, np.float64)
    out = np.broadcast_to(b, (x.shape[0], Ho, Wo, x.shape[3])).copy()
    S = np.abs(out)
    for r, s, tap in _window_taps(x, K, stride, pad[0], pad[1], Ho, Wo, 0.0):
        out += tap * w[r, s]
        S += np.abs(tap * w[r, s])
    return out, S


# ---- pools ---------------------------------------------------------------------------------------------------------
def maxpool_stem(x, out_hw):
    """The stems' 3x3 stride-2 max-pool: window rows 2y - 1 .. 2y + 1 (columns alike) clipped to the map, output out_hw.
    nn.MaxPool2d(3, 2, 1) when out_hw = ceil(H/2) x ceil(W/2); TF's pad [1, 0] + VALID 3x3/2 when out_hw = floor(H/2) x
    floor(W/2)."""
    x = np.asarray(x, np.float64)
    Ho, Wo = out_hw
    out = np.full((x.shape[0], Ho, Wo, x.shape[3]), -np.inf)
    for _, _, tap in _window_taps(x, 3, 2, 1, 1, Ho, Wo, -np.inf):
        out = np.maximum(out, tap)
    return out


def maxpool_same(x, out_hw, pads):
    """BiFPN's 3x3 stride-2 max-pool with TF SAME padding (resample_feature_map): window rows 2y - pad_t + r."""
    x = np.asarray(x, np.float64)
    Ho, Wo = out_hw
    out = np.full((x.shape[0], Ho, Wo, x.shape[3]), -np.inf)
    for _, _, tap in _window_taps(x, 3, 2, pads[0], pads[1], Ho, Wo, -np.inf):
        out = np.maximum(out, tap)
    return out


def upsample2(x):
    """Nearest-neighbour 2x upsampling."""
    return np.repeat(np.repeat(np.asarray(x, np.float64), 2, axis=1), 2, axis=2)


def avgpool2(x):
    """nn.AvgPool2d(2): floor(H/2) x floor(W/2) means of 2x2 blocks."""
    x = np.asarray(x, np.float64)
    Ho, Wo = x.shape[1] // 2, x.shape[2] // 2
    t = x[:, :2 * Ho, :2 * Wo]
    return (t[:, 0::2, 0::2] + t[:, 0::2, 1::2] + t[:, 1::2, 0::2] + t[:, 1::2, 1::2]) / 4.0


def avgpool2_f32(x):
    """avgpool2_kernel's arithmetic: ((x00 + x01) + x10) + x11 in fp32, then * 0.25."""
    x = np.asarray(x, np.float32)
    Ho, Wo = x.shape[1] // 2, x.shape[2] // 2
    t = x[:, :2 * Ho, :2 * Wo]
    return ((t[:, 0::2, 0::2] + t[:, 0::2, 1::2]) + t[:, 1::2, 0::2] + t[:, 1::2, 1::2]) * np.float32(0.25)


def gap(x):
    """nn.AdaptiveAvgPool2d(1) of x [B][H][W][C] (or [B][HW][C]): [B][C]."""
    x = np.asarray(x, np.float64)
    return x.reshape(x.shape[0], -1, x.shape[-1]).mean(axis=1)


# ---- BiFPN ---------------------------------------------------------------------------------------------------------
def resample(x, th, tw):
    """resample_feature_map without its 1x1 conv: (mode, (pad_t, pad_l), x at th x tw).  Same size: as is (mode 0);
    twice as large: 3x3/2 max-pool with TF SAME padding (mode 1); half the size: nearest 2x upsampling (mode 2)."""
    H, W = x.shape[1:3]
    if (H, W) == (th, tw):
        return 0, (0, 0), np.asarray(x, np.float64)
    if H > th and W > tw:
        assert (H - 1) // th + 1 == 2 and (W - 1) // tw + 1 == 2
        (oh, pt), (ow, pl) = same_pad(H, 3, 2), same_pad(W, 3, 2)
        assert (oh, ow) == (th, tw)
        return 1, (pt, pl), maxpool_same(x, (th, tw), (pt, pl))
    assert (2 * H, 2 * W) == (th, tw)
    return 2, (0, 0), upsample2(x)


def fastattn(weights):
    """The fastattn edge weights relu(w_i) / (sum_i relu(w_i) + 1e-4), float64."""
    r = np.maximum(np.asarray(weights, np.float64), 0.0)
    return r / (r.sum() + 1e-4)


def bifpn_combine(inputs, th, tw, weights=None, act=False):
    """A BiFPN node: its inputs resampled to th x tw, combined by the plain sum (weights None) or fastattn, then swish
    when act.  Returns (out, S, pre): S = sum_i |term_i| of the combine, pre the combine before the activation."""
    xs = [resample(x, th, tw)[2] for x in inputs]
    f = np.ones(len(xs)) if weights is None else fastattn(weights)
    terms = [x * fi for x, fi in zip(xs, f)]
    pre = sum(terms)
    S = sum(np.abs(t) for t in terms)
    return (swish(pre) if act else pre), S, pre


def bifpn_combine_f32(inputs, th, tw, weights=None):
    """bifpn_combine_kernel's arithmetic without the swish: term_i = (x_i * w_i) / denom (or x_i) in fp32, summed in input
    order; relu(w_i) and denom = add_n(relu(w)) + 1e-4 in fp32 as bifpn_set_weights makes them."""
    xs = [resample(x, th, tw)[2].astype(np.float32) for x in inputs]
    if weights is None:
        terms = xs
    else:
        r = [np.float32(max(np.float32(w), np.float32(0))) for w in weights]
        tot = r[0]
        for t in r[1:]:
            tot = np.float32(tot + t)
        denom = np.float32(tot + np.float32(1e-4))
        terms = [(x * ri) / denom for x, ri in zip(xs, r)]
    acc = terms[0]
    for t in terms[1:]:
        acc = acc + t
    return acc


# ---- squeeze-excite ------------------------------------------------------------------------------------------------
def mbconv_se(x, creal, w1, b1, w2, b2):
    """MBConv's squeeze-excite of x [B][HW][Cpad] (channels [0, creal) live): gate [B][Cpad] = sigmoid(swish(mean(x) @ w1
    + b1) @ w2 + b2) in the live columns, 0 in the padded ones.  Returns (gate, parts) with the intermediate values and
    magnitudes the error bound needs: mean, h (= mean @ w1 + b1), S1 (= |b1| + |mean| @ |w1|), r (= swish(h)), a (the
    gate's logit), S2 (= |b2| + |r| @ |w2|)."""
    x = np.asarray(x, np.float64)
    w1, b1, w2, b2 = (np.asarray(t, np.float64) for t in (w1, b1, w2, b2))
    m = x[..., :creal].mean(axis=1)
    h = m @ w1 + b1
    r = swish(h)
    a = r @ w2 + b2
    gate = np.zeros((x.shape[0], x.shape[2]))
    gate[:, :creal] = sigmoid(a)
    parts = dict(mean=m, h=h, S1=np.abs(b1) + np.abs(m) @ np.abs(w1), r=r, a=a, S2=np.abs(b2) + np.abs(r) @ np.abs(w2))
    return gate, parts


def channel_gate(pooled, w1, b1, w2, b2):
    """OSNet's ChannelGate MLP on pooled rows [N][Creal]: sigmoid(relu(p @ w1^T + b1) @ w2^T + b2), w1 [Cr][Creal] and
    w2 [Creal][Cr] the 1x1 convs' [out][in] weights.  Returns (gates, h, S1, S2) as mbconv_se's parts."""
    p = np.asarray(pooled, np.float64)
    w1, b1, w2, b2 = (np.asarray(t, np.float64) for t in (w1, b1, w2, b2))
    h = p @ w1.T + b1
    r = relu(h)
    a = r @ w2.T + b2
    return sigmoid(a), h, np.abs(b1) + np.abs(p) @ np.abs(w1.T), np.abs(b2) + np.abs(r) @ np.abs(w2.T)


def gated_sum4(streams, gates):
    """OSBlock's x2 = sum_k gate_k * x_k: streams [4][B][HW][C], gates [B][4][C] -> ([B][HW][C], sum_k |gate_k x_k|)."""
    s = np.asarray(streams, np.float64)
    g = np.asarray(gates, np.float64)
    terms = s * g.transpose(1, 0, 2)[:, :, None, :]
    return terms.sum(axis=0), np.abs(terms).sum(axis=0)


def gated_sum4_f32(streams, gates):
    """gated_sum4_kernel's arithmetic: acc = 0, then acc + x_k * gate_k in fp32 for k = 0..3."""
    s = np.asarray(streams, np.float32)
    g = np.asarray(gates, np.float32)
    acc = np.zeros(s.shape[1:], np.float32)
    for k in range(4):
        acc = acc + s[k] * g[:, k][:, None, :]
    return acc


# ---- EfficientNet's stem operand -----------------------------------------------------------------------------------
def stem_im2col(img, out_hw, pad):
    """The 3x3/2 patches of img [H][W][3] as 64-column pixels [Ho][Wo][64]: column (r*3 + s)*3 + c = img[2y - pad_t + r]
    [2x - pad_l + s][c] (0 outside the image), columns 27..63 zero."""
    img = np.asarray(img, np.float64)
    Ho, Wo = out_hw
    out = np.zeros((Ho, Wo, 64))
    for r, s, tap in _window_taps(img[None], 3, 2, pad[0], pad[1], Ho, Wo, 0.0):
        out[:, :, (r * 3 + s) * 3:(r * 3 + s) * 3 + 3] = tap[0]
    return out
