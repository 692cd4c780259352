"""The element-wise and reduction kernels around the GEMMs, one at a time through their single-op entries, against the
float64 reference of tests/elementwise_oracle.py: EfficientNet's depthwise strip kernel and MBConv squeeze-excite, the
BiFPN node combine, the stems' max-pool, OSNet's depthwise conv, pools, channel gate and gated sum, EfficientNet's stem
im2col.  The geometries are the ones where such kernels break: SAME pads of 0, 1 and 2, ragged last strips, maps of one
row or column, odd maps, padded channels, grid-stride loops past the launch's block cap, chunk boundaries.

Every input is built with eo.representable, so it is exactly what the kernel reads.  Two kinds of check:
  * bit-exact: outputs that involve no rounding, or only IEEE-rounded fp32 operations in a known order, must hold the
    raw planes of the float32 restatement (eo.raw of eo.*_f32);
  * error-bounded: each element's |kernel - float64 reference| within a bound derived next to the test from the
    kernel's operation order.  Throughout, U = 2^-24 is the fp32 unit roundoff; a sum of n terms accumulated in fp32 is
    off by at most (n - 1) U sum|terms| to first order, and every bound rounds n up by one to cover the second-order
    terms (below n^2 U^2 sum|terms|); storing a value v as split planes adds 2^-22 |v| + 2^-36 (eo.store_bound; 2^-11 |v|
    + 2^-25 as the hi plane alone in fp16 precision).
Elements are compared one by one, so an error in a small element is not hidden by a large one elsewhere."""
import numpy as np
import pytest

import elementwise_oracle as eo

pytestmark = pytest.mark.gpu

U = eo.U
SIGMOID_REL = 6 * U   # expf (2 ulp = 4 U), 1 + e and the reciprocal (U each): relative error of the kernels' sigmoid
SWISH_D = 1.1         # max |d swish / dx| = 1.0998


def _engine():
    from object_detection_tracking_b200 import engine
    return engine


def rep(x, split=True):
    return eo.representable(np.asarray(x, np.float32), split)


def assert_bits(hi, lo, expect, split, what=""):
    """The raw planes equal eo.raw(expect) bit for bit."""
    eh, el = eo.raw(np.asarray(expect, np.float32), split)
    bad = hi != eh
    if split:
        bad |= lo != el
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError("%s: %d elements differ, first %s: got (%04x, %04x) expected (%04x, %04x) = %r" % (
            what, bad.sum(), i, hi[i], lo[i] if split else 0, eh[i], el[i] if split else 0, np.float32(expect[i])))


def assert_within(got, ref, bnd, what=""):
    got = np.asarray(got, np.float64)
    assert np.isfinite(got).all(), "%s: non-finite output" % what
    err = np.abs(got - ref)
    if not (err <= bnd).all():
        i = np.unravel_index(np.argmax(err - bnd), err.shape)
        raise AssertionError("%s: element %s |err| %.3g > bound %.3g (ref %.6g, got %.6g)" % (
            what, i, err[i], bnd[i], ref[i], got[i]))


def got_planes(hi, lo, split):
    return eo.joined(hi, lo if split else None)


def act_bound(pre_err, pre, act):
    """Error after the activation of a value off by pre_err: swish is 1.1-Lipschitz and the kernels evaluate it as
    x * (1 / (1 + expf(-x))), relative error SIGMOID_REL + U of |swish(x)| <= |x| (+1 U for second order; where expf
    overflows, the kernel's 0 is within 2^-126 |x| of the true value, inside the store bound's absolute term); ReLU is
    1-Lipschitz and exact."""
    if act == "swish":
        return SWISH_D * pre_err + (SIGMOID_REL + 2 * U) * (np.abs(pre) + pre_err)
    return pre_err


# ==== EfficientNet's depthwise strip kernel ==========================================================================
# (H, W, C): with SAME padding at every (K, S) these give Wo % TX (TX = 4 at stride 1, 2 at stride 2) every residue and
# Wo < TX, H = 1 and W = 1, odd and even maps (pad_before 0, 1 and 2), C = 8 (one vector) and multiples of 8 that are not
# multiples of 64.
STRIP_MAPS = [(1, 1, 8), (1, 13, 24), (9, 1, 8), (6, 6, 72), (7, 9, 16), (10, 14, 40), (5, 11, 8), (12, 7, 136),
              (8, 8, 8), (3, 12, 24), (4, 2, 8), (13, 5, 16)]
KS = [(3, 1), (3, 2), (5, 1), (5, 2)]


def run_strip(rng, H, W, C, K, S, act, with_bias, split, scale=1.0, bias=None):
    (Ho, pt), (Wo, pl) = eo.same_pad(H, K, S), eo.same_pad(W, K, S)
    x = rep(rng.standard_normal((1, H, W, C)), split)
    w = (rng.standard_normal((K, K, C)) * scale / K).astype(np.float32)
    if bias is None and with_bias:
        bias = rng.standard_normal(C).astype(np.float32)
    out, hi, lo = _engine().op_depthwise(x, w, bias, stride=S, pad=(pt, pl), out_hw=(Ho, Wo), act=act, split=split)
    pre, Sabs = eo.depthwise(x, w, bias, S, (pt, pl), (Ho, Wo))
    ref = eo.swish(pre) if act == "swish" else pre
    # bias, then K*K fmaf in (r, s) order: K*K roundings, each at most U of a partial sum <= Sabs; +1 (second order)
    b = act_bound((K * K + 1) * U * Sabs, pre, act)
    b = b + eo.store_bound(np.abs(ref) + b, split)
    got = got_planes(hi, lo, split)
    assert_within(got, ref, b, "depthwise K%d/S%d %dx%dx%d %s" % (K, S, H, W, C, act))
    return (pt, pl), (Ho, Wo)


@pytest.mark.parametrize("K,S", KS, ids=["k3s1", "k3s2", "k5s1", "k5s2"])
@pytest.mark.parametrize("geo", range(len(STRIP_MAPS)))
def test_strip_depthwise_same_geometries(K, S, geo):
    H, W, C = STRIP_MAPS[geo]
    rng = np.random.default_rng(1000 * K + 100 * S + geo)
    act = "swish" if geo % 2 == 0 else "none"
    pads, _ = run_strip(rng, H, W, C, K, S, act, with_bias=geo % 3 != 0, split=True)
    assert pads == (eo.same_pad(H, K, S)[1], eo.same_pad(W, K, S)[1])


def test_strip_maps_cover_every_pad_before_and_tail():
    """Over STRIP_MAPS, pad_before takes 0, 1 and 2 (stride 2: odd and even maps), and Wo takes every residue mod TX
    and values below TX."""
    pads = {(K, S): {eo.same_pad(n, K, S)[1] for H, W, _ in STRIP_MAPS for n in (H, W)} for K, S in KS}
    assert pads == {(3, 1): {1}, (3, 2): {0, 1}, (5, 1): {2}, (5, 2): {1, 2}}
    for S, TX in ((1, 4), (2, 2)):
        wos = {eo.same_pad(W, 3, S)[0] for _, W, _ in STRIP_MAPS}
        assert {wo % TX for wo in wos} == set(range(TX)) and min(wos) < TX


@pytest.mark.parametrize("K,S", KS, ids=["k3s1", "k3s2", "k5s1", "k5s2"])
def test_strip_depthwise_fp16(K, S):
    rng = np.random.default_rng(77 + K + S)
    for H, W, C in [(7, 9, 16), (1, 13, 24), (12, 7, 136)]:
        run_strip(rng, H, W, C, K, S, "swish", True, split=False)


@pytest.mark.parametrize("K,S", KS, ids=["k3s1", "k3s2", "k5s1", "k5s2"])
def test_strip_depthwise_swish_at_large_magnitude(K, S):
    """Biases from -100 to 100 put the swish inputs where expf(-x) overflows (x < -88.7) or vanishes: every output is
    finite and within the bound."""
    rng = np.random.default_rng(5 + K * S)
    C = 64
    bias = np.linspace(-100, 100, C).astype(np.float32)
    run_strip(rng, 9, 10, C, K, S, "swish", True, split=True, scale=0.5, bias=bias)


def test_strip_depthwise_grid_stride_loop():
    """K3/S1 at 384x384x256: 384 rows x 96 strips x 32 channel vectors = 1,179,648 items, more than the launch's
    132 * 64 blocks x 128 threads = 1,081,344, so some threads take a second item."""
    rng = np.random.default_rng(384)
    H, W, C = 384, 384, 256
    assert H * (W // 4) * (C // 8) > 132 * 64 * 128
    run_strip(rng, H, W, C, 3, 1, "swish", True, split=True)


# ==== OSNet's depthwise 3x3 ==========================================================================================
# B >= 3 with a different offset per image, H*W not a multiple of 32; the last map is above the launch's grid cap
# (3 x 97 x 93 pixels x 48 vectors = 1,298,916 items > 132 * 32 blocks x 256 threads = 1,081,344).
OSNET_DW = [(3, 5, 7, 8, True), (4, 13, 11, 72, True), (3, 1, 9, 16, False), (3, 97, 93, 384, True)]


@pytest.mark.parametrize("case", range(len(OSNET_DW)))
def test_osnet_depthwise(case):
    B, H, W, C, split = OSNET_DW[case]
    rng = np.random.default_rng(50 + case)
    x = rep(rng.standard_normal((B, H, W, C)) + np.arange(B)[:, None, None, None] * 3.0, split)
    w = (rng.standard_normal((3, 3, C)) / 3).astype(np.float32)
    b = rng.standard_normal(C).astype(np.float32)
    out, hi, lo = _engine().op_depthwise(x, w, b, stride=1, pad=(1, 1), act="relu", impl="osnet", split=split)
    pre, Sabs = eo.depthwise(x, w, b, 1, (1, 1))
    ref = eo.relu(pre)
    # up to 9 fmaf from 0, then + bias: 10 roundings (+1); ReLU is 1-Lipschitz
    bnd = 11 * U * Sabs
    assert_within(got_planes(hi, lo, split), ref, bnd + eo.store_bound(ref + bnd, split), "osnet dw %s" % (OSNET_DW[case],))


# ==== the stems' max-pool ============================================================================================
def tied_nonneg(rng, shape, split=True):
    """Values >= 0 on a few hi levels with many different lo: windows hold equal hi planes whose lo differ, in every
    order; some zeros."""
    base = rng.choice(np.float32([0.5, 1.0, 1.5, 3.0]), shape)
    ulp = np.spacing(base.astype(np.float16)).astype(np.float32)
    x = base + rng.uniform(-0.45, 0.45, shape).astype(np.float32) * ulp
    x[rng.random(shape) < 0.05] = 0
    x = rep(x, split)
    assert (x >= 0).all()
    return x


def maxpool_out(caller, H, W):
    # the detector's plan (engine.cu): pad [1, 0] then 3x3/2 VALID, (H + 1 - 3) / 2 + 1 = floor(H / 2);
    # the ReID engines (reid_engine.cu): nn.MaxPool2d(3, 2, 1), (H - 1) / 2 + 1 = ceil(H / 2)
    return ((H - 2) // 2 + 1, (W - 2) // 2 + 1) if caller == "detector" else ((H - 1) // 2 + 1, (W - 1) // 2 + 1)


@pytest.mark.parametrize("caller", ["detector", "reid"])
@pytest.mark.parametrize("H,W", [(8, 12), (9, 7), (6, 11), (13, 13), (2, 3)])
@pytest.mark.parametrize("split", [True, False], ids=["split", "fp16"])
def test_maxpool_bit_exact(caller, H, W, split):
    """The (hi, lo) pair of the largest joined value, ties of hi broken by lo; windows cut by the border."""
    rng = np.random.default_rng(H * 100 + W + (caller == "reid"))
    x = tied_nonneg(rng, (2, H, W, 64), split)
    Ho, Wo = maxpool_out(caller, H, W)
    out, hi, lo = _engine().op_pool(x, "max", out_hw=(Ho, Wo), split=split)
    assert_bits(hi, lo, eo.maxpool_stem(x, (Ho, Wo)).astype(np.float32), split, "maxpool %s %dx%d" % (caller, H, W))


def test_maxpool_ties_are_exercised():
    """The tie inputs above hold many windows whose largest hi occurs more than once."""
    rng = np.random.default_rng(9 * 100 + 7)
    x = tied_nonneg(rng, (2, 9, 7, 64))
    hi = eo.planes(x)[0].astype(np.float64)
    m = eo.maxpool_stem(hi, (4, 3))
    n_tied = sum((t == m) for _, _, t in eo._window_taps(hi, 3, 2, 1, 1, 4, 3, -np.inf))
    assert (n_tied >= 2).mean() > 0.3


# ==== OSNet's pools ==================================================================================================
@pytest.mark.parametrize("B,H,W,C", [(3, 5, 7, 8), (3, 8, 6, 24), (4, 9, 9, 64), (3, 2, 2, 8)])
@pytest.mark.parametrize("split", [True, False], ids=["split", "fp16"])
def test_avgpool2_bit_exact(B, H, W, C, split):
    """AvgPool2d(2) of odd maps drops the last row / column; the kernel's ((x00 + x01) + x10) + x11, * 0.25 in fp32."""
    rng = np.random.default_rng(B * H * W + C)
    x = rep(rng.standard_normal((B, H, W, C)) + np.arange(B)[:, None, None, None], split)
    out, hi, lo = _engine().op_pool(x, "avg2", split=split)
    assert out.shape == (B, H // 2, W // 2, C)
    assert_bits(hi, lo, eo.avgpool2_f32(x), split, "avgpool2 %dx%d" % (H, W))


@pytest.mark.parametrize("B,H,W,C,ld", [(3, 5, 7, 64, 64), (3, 9, 13, 192, 256), (2, 16, 8, 128, 192), (1, 1, 1, 64, 64)])
@pytest.mark.parametrize("split", [True, False], ids=["split", "fp16"])
def test_gap(B, H, W, C, ld, split):
    rng = np.random.default_rng(H * W + C + ld)
    x = rep(rng.standard_normal((B, H, W, C)) + np.arange(B)[:, None, None, None] * 2, split)
    init = np.full((B, ld), -7.25, np.float32)
    out, _, _ = _engine().op_pool(x, "gap", out_ld=ld, out_init=init, split=split)
    ref = eo.gap(x)
    # each of 32 lanes sums ceil(HW / 32) pixels, then 32 lane sums in sequence, then / HW: ceil(HW/32) + 32 + 1
    # roundings of at most U sum|x| / HW each (+1)
    n = -(-H * W // 32) + 34
    assert_within(out[:, :C], ref, n * U * eo.gap(np.abs(x)), "gap")
    assert (out[:, C:] == np.float32(-7.25)).all(), "gap wrote past C"


# ==== OSNet's channel gate and gated sum =============================================================================
def gate_bounds(pooled_abs, HW, creal, w1, w2, gates, S1, S2):
    """Bound on the gates (from the kernels' gap and gate_mlp):
      pooled  (ceil(HW/32) + 34) U mean|x|                                    (as test_gap)
      fc1     b1 + Creal fmaf in order: (Creal + 1) U S1, plus |w1| . err(pooled); ReLU is 1-Lipschitz
      fc2     b2 + Cr fmaf: (Cr + 1) U S2, plus |w2| . err(hidden)
      sigmoid derivative <= 1/4, evaluated with relative error SIGMOID_REL (+U)."""
    cr = w1.shape[0]
    e_p = (-(-HW // 32) + 34) * U * pooled_abs[:, :creal]
    e_h = (creal + 1) * U * S1 + e_p @ np.abs(w1.T)
    e_a = (cr + 1) * U * S2 + e_h @ np.abs(w2.T)
    return 0.25 * e_a + (SIGMOID_REL + U) * gates


# (B, HW, C, Creal, Cr, split): OSNet's widths (mid = 64, 96, 128 live of 64, 128, 128), H*W not a multiple of 32, and
# the largest gate_mlp takes (Creal 512, Cr 64)
GATE_CASES = [(3, 35, 64, 64, 4, True), (3, 117, 128, 96, 6, True), (4, 33, 512, 512, 64, True),
              (3, 35, 128, 128, 8, False)]


@pytest.mark.parametrize("case", range(len(GATE_CASES)))
def test_channel_gate(case):
    B, HW, C, creal, cr, split = GATE_CASES[case]
    rng = np.random.default_rng(300 + case)
    s = rng.standard_normal((4, B, HW, C)) + np.arange(4)[:, None, None, None] * 0.5 + \
        np.arange(B)[None, :, None, None] * 0.25
    s[..., creal:] = 0   # padded channels hold zeros, as the engine's conv outputs do
    s = rep(s, split)
    w1 = (rng.standard_normal((cr, creal)) / np.sqrt(creal)).astype(np.float32)
    b1 = rng.standard_normal(cr).astype(np.float32)
    w2 = (rng.standard_normal((creal, cr)) / np.sqrt(cr)).astype(np.float32)
    b2 = rng.standard_normal(creal).astype(np.float32)
    gates, out, hi, lo = _engine().op_channel_gate(s, creal, w1, b1, w2, b2, split=split)
    pooled = np.stack([eo.gap(s[k]) for k in range(4)], axis=1).reshape(B * 4, C)
    pooled_abs = np.stack([eo.gap(np.abs(s[k])) for k in range(4)], axis=1).reshape(B * 4, C)
    g, _, S1, S2 = eo.channel_gate(pooled[:, :creal], w1, b1, w2, b2)
    eg = gate_bounds(pooled_abs, HW, creal, w1, w2, g, S1, S2)
    assert_within(gates.reshape(B * 4, C)[:, :creal], g, eg, "gates")
    assert (gates.reshape(B * 4, C)[:, creal:] == 0).all(), "padded gate columns must be exactly 0"
    g_full = np.zeros((B, 4, C))
    g_full[..., :creal] = g.reshape(B, 4, creal)
    e_full = np.zeros((B, 4, C))
    e_full[..., :creal] = eg.reshape(B, 4, creal)
    ref, Sabs = eo.gated_sum4(s, g_full)
    # the sum: |s_k| err(gate_k) per term, and 4 products + 3 additions in fp32: 4 roundings of a term's path (+1)
    b = np.abs(s).transpose(1, 2, 0, 3).reshape(B, HW, 4, C)
    b = (b * e_full[:, None]).sum(axis=2) + 5 * U * (Sabs + (b * e_full[:, None]).sum(axis=2))
    assert_within(got_planes(hi, lo, split), ref, b + eo.store_bound(np.abs(ref) + b, split), "gated sum")


# (B, HW, C, split); the last is above the launch's grid cap: 3 x 23707 pixels x 16 vectors = 1,137,936 items
GSUM_CASES = [(3, 35, 64, True), (4, 117, 128, False), (3, 23707, 128, True)]


@pytest.mark.parametrize("case", range(len(GSUM_CASES)))
def test_gated_sum4_bit_exact(case):
    """With the gates given: acc = 0, then acc + x_k * gate_k in fp32, k = 0..3."""
    B, HW, C, split = GSUM_CASES[case]
    rng = np.random.default_rng(400 + case)
    s = rep(rng.standard_normal((4, B, HW, C)) + np.arange(B)[None, :, None, None], split)
    gates = rng.uniform(0, 1, (B, 4, C)).astype(np.float32)
    gates[:, :, -8:] = 0
    g_out, out, hi, lo = _engine().op_channel_gate(s, C, gates=gates, split=split)
    assert np.array_equal(g_out, gates)
    assert_bits(hi, lo, eo.gated_sum4_f32(s, gates), split, "gated_sum4 %s" % (GSUM_CASES[case],))


# ==== MBConv's squeeze-excite ========================================================================================
def cdiv(a, b):
    return -(-a // b)


def se_chunks(HW):
    return min(max(cdiv(HW, 512), 1), 1024)   # effnet.cu se_chunks


def se_gate_bound(x, creal, w1, w2, parts, gate, Cpad):
    """Bound on the gate from se_partial / se_fc1 / se_fc2 (effnet.cu):
      mean   a pixel's value passes the pairwise add of 4 loads (2 roundings), the thread's running sum (ceil(chunk / 128)),
             the 32 thread sums (32), the lanes' sums over chunk partials (ceil(nchunks / 32)), the 5-step butterfly (5),
             then * inv_hw with inv_hw itself rounded (2): n U mean|x| (+1)
      hidden warps' fmaf over their channels (ceil(ceil(C / 32) / 8)), the 8 warp sums (8), b1 + the 32 block sums (32):
             n1 U S1, plus |w1| . err(mean); swish 1.1-Lipschitz, evaluated to (SIGMOID_REL + 2U) |h|
      logit  4 groups of ceil(nr / 4) fmaf, ((p0 + p1) + (p2 + p3)) and + b2 (3): n2 U S2, plus |w2| . err(hidden)
      gate   sigmoid derivative <= 1/4, evaluated with relative error SIGMOID_REL (+U)."""
    B, HW, _ = x.shape
    nr = w1.shape[1]
    nch = se_chunks(HW)
    n_m = 2 + cdiv(cdiv(HW, nch), 128) + 32 + cdiv(nch, 32) + 5 + 2 + 1
    e_m = n_m * U * np.abs(x[..., :creal]).mean(axis=1)
    n1 = cdiv(cdiv(creal, 32), 8) + 8 + 32 + 1
    e_h = n1 * U * parts["S1"] + e_m @ np.abs(w1)
    e_r = SWISH_D * e_h + (SIGMOID_REL + 2 * U) * (np.abs(parts["h"]) + e_h)
    n2 = cdiv(nr, 4) + 3 + 1
    e_a = n2 * U * parts["S2"] + e_r @ np.abs(w2)
    e = np.zeros((B, Cpad))
    e[:, :creal] = 0.25 * e_a + (SIGMOID_REL + U) * gate[:, :creal]
    return e


def se_case(rng, B, HW, creal, nr, cout, split=True, fold=True):
    Cp = -(-creal // 64) * 64
    x = rng.standard_normal((B, HW, Cp)).astype(np.float32) * 0.5 + 0.25
    x[..., creal:] = 5.0   # padded channels take no part in the mean
    x = rep(x, split)
    w1 = (rng.standard_normal((creal, nr)) * 4 / np.sqrt(creal)).astype(np.float32)
    b1 = rng.standard_normal(nr).astype(np.float32)
    w2 = (rng.standard_normal((nr, creal)) * 2 / np.sqrt(nr)).astype(np.float32)
    b2 = rng.standard_normal(creal).astype(np.float32)
    rows = -(-cout // 16) * 16   # the projection's Cout_pad rows
    w = None
    if fold:
        w = np.zeros((rows, Cp), np.float32)
        w[:cout, :creal] = rng.standard_normal((cout, creal)) * 10.0 ** rng.uniform(-2, 1, (cout, creal))
    gate, folded, hi, lo = _engine().op_mbconv_se(x, creal, w1, b1, w2, b2, w=w, split=split)
    ref, parts = eo.mbconv_se(x, creal, w1, b1, w2, b2)
    eg = se_gate_bound(x, creal, w1, w2, parts, ref, Cp)
    assert_within(gate, ref, eg, "se gate HW %d Creal %d nr %d" % (HW, creal, nr))
    assert (gate[:, creal:] == 0).all(), "padded gate columns must be exactly 0"
    if fold:
        fr = w.astype(np.float64) * ref[0]
        # w[o][c] * gate[c] in fp32: |w| err(gate) + U |w gate| (+1), then stored as planes
        fb = np.abs(w) * eg[0] + 2 * U * np.abs(fr)
        assert_within(got_planes(hi, lo, split), fr, fb + eo.store_bound(np.abs(fr) + fb, split), "se fold")
        zero = np.ones(w.shape, bool)
        zero[:cout, :creal] = False
        assert (hi[zero] == 0).all() and (not split or (lo[zero] == 0).all()), \
            "padded rows and columns of the folded weight must be exactly +0"


# (HW, Creal, nr, Cout): HW around a chunk (511, 512, 513) and at the b7 stem level (768 x 768 = 589,824 pixels, where
# se_chunks saturates at 1024 and a chunk holds 576 pixels); Creal 32, 96, 240, 1152 (pad64: 64, 128, 256, 1152);
# nr 1 to se_max_nr() = 192; the projection's rows padded to 16
SE_CASES = [(1, 32, 1, 16), (511, 96, 4, 24), (512, 240, 48, 40), (513, 1152, 192, 200), (589824, 32, 160, 16),
            (513, 240, 192, 80), (1, 1152, 48, 320), (512, 96, 160, 24)]


@pytest.mark.parametrize("case", range(len(SE_CASES)))
def test_mbconv_se_gate_and_fold(case):
    HW, creal, nr, cout = SE_CASES[case]
    se_case(np.random.default_rng(500 + case), 1, HW, creal, nr, cout)


def test_mbconv_se_chunking_reaches_saturation():
    assert se_chunks(589824) == 1024 and -(-589824 // 1024) > 512


def test_mbconv_se_gate_only_batched():
    """Three images through se_squeeze / se_excite (swish, no fold): each image's gate from its own pixels."""
    se_case(np.random.default_rng(600), 3, 513, 240, 48, 40, fold=False)


@pytest.mark.parametrize("case", [1, 3])
def test_mbconv_se_fp16(case):
    HW, creal, nr, cout = SE_CASES[case]
    se_case(np.random.default_rng(700 + case), 1, HW, creal, nr, cout, split=False)


# ==== the BiFPN node combine =========================================================================================
TH, TW = 6, 8


def bifpn_source(mode, idx):
    """A source map for a node of TH x TW: same size (mode 0); 2x finer (mode 1), odd in H, W or both by input index so
    that the SAME pads (pad_t, pad_l) are (1, 0), (0, 1) and (1, 1); 2x coarser (mode 2)."""
    if mode == 0:
        return TH, TW
    if mode == 2:
        return TH // 2, TW // 2
    return [(2 * TH - 1, 2 * TW), (2 * TH, 2 * TW - 1), (2 * TH - 1, 2 * TW - 1)][idx]


BIFPN_MIXES = [(m,) for m in range(3)] + [(a, b) for a in range(3) for b in range(3)] + \
              [(a, b, c) for a in range(3) for b in range(3) for c in range(3)]


@pytest.mark.parametrize("mix", BIFPN_MIXES, ids=lambda m: "".join(map(str, m)))
def test_bifpn_combine(mix):
    """Plain sum and fastattn combine without swish bit-exact; with swish (the node's op_after_combine input)
    error-bounded.  B = 2, every mode mix of 1, 2 and 3 inputs."""
    rng = np.random.default_rng(int("".join(map(str, mix)), 3) + 10 * len(mix))
    B, C = 2, 24
    xs = [rep(rng.standard_normal((B,) + bifpn_source(m, i) + (C,)) + np.arange(B)[:, None, None, None])
          for i, m in enumerate(mix)]
    eng = _engine()
    weights = [0.8, -0.2, 1.7][:len(mix)]
    for wts in (None, weights):
        out, hi, lo, res = eng.op_bifpn_combine(xs, (TH, TW), weights=wts)
        for i, m in enumerate(mix):
            mode, pads, _ = eo.resample(xs[i], TH, TW)
            assert mode == m and tuple(res[i]) == (mode,) + pads, (i, tuple(res[i]), mode, pads)
        assert_bits(hi, lo, eo.bifpn_combine_f32(xs, TH, TW, wts), True, "combine %s weights %s" % (mix, wts))
    # with swish: the combine's n products, n quotients and n - 1 additions (fp32, IEEE), and denom's rounding
    # (n - 1 additions and + 1e-4f, whose own error is 1e-4 U): at most 2n + 1 roundings of a term's path (+1)
    out, hi, lo, _ = eng.op_bifpn_combine(xs, (TH, TW), weights=weights, swish=True)
    ref, Sabs, pre = eo.bifpn_combine(xs, TH, TW, weights, act=True)
    b = act_bound((2 * len(mix) + 2) * U * Sabs, pre, "swish")
    assert_within(got_planes(hi, lo, True), ref, b + eo.store_bound(np.abs(ref) + b), "combine swish %s" % (mix,))


def test_bifpn_combine_fp16_swish():
    rng = np.random.default_rng(8)
    xs = [rep(rng.standard_normal((2,) + bifpn_source(m, i) + (16,)), False) for i, m in enumerate((1, 0, 2))]
    out, hi, lo, _ = _engine().op_bifpn_combine(xs, (TH, TW), weights=[0.5, 1.5, 0.1], swish=True, split=False)
    ref, Sabs, pre = eo.bifpn_combine(xs, TH, TW, [0.5, 1.5, 0.1], act=True)
    b = act_bound(8 * U * Sabs, pre, "swish")
    assert_within(got_planes(hi, None, False), ref, b + eo.store_bound(np.abs(ref) + b, False), "combine fp16")


# ==== EfficientNet's stem im2col =====================================================================================
@pytest.mark.parametrize("H,W", [(1, 1), (7, 10), (12, 9), (33, 64)])
@pytest.mark.parametrize("split", [True, False], ids=["split", "fp16"])
def test_stem_im2col_bit_exact(H, W, split):
    """Each live column the image value's planes; the 37 dead columns of every pixel +0 in both planes."""
    rng = np.random.default_rng(H * 1000 + W)
    img = (rng.standard_normal((H, W, 3)) * 10.0 ** rng.uniform(-3, 2, (H, W, 3))).astype(np.float32)
    (Ho, pt), (Wo, pl) = eo.same_pad(H, 3, 2), eo.same_pad(W, 3, 2)
    out, hi, lo = _engine().op_stem_im2col(img, (Ho, Wo), (pt, pl), split=split)
    assert_bits(hi, lo, eo.stem_im2col(img, (Ho, Wo), (pt, pl)).astype(np.float32), split, "stem im2col")
    assert (hi[..., 27:] == 0).all() and (not split or (lo[..., 27:] == 0).all())


# ==== argument checks ================================================================================================
def test_bad_arguments_return_errors():
    eng = _engine()
    x = np.zeros((1, 4, 4, 12), np.float32)
    with pytest.raises(RuntimeError, match="multiple of 8"):
        eng.op_depthwise(x, np.zeros((3, 3, 12), np.float32))
    with pytest.raises(RuntimeError, match="one image"):
        eng.op_depthwise(np.zeros((2, 4, 4, 8), np.float32), np.zeros((3, 3, 8), np.float32))
    with pytest.raises(RuntimeError, match="ceil"):
        eng.op_pool(np.zeros((1, 4, 4, 8), np.float32), "max", out_hw=(3, 2))
    with pytest.raises(RuntimeError, match="se_max_nr"):
        eng.op_mbconv_se(np.zeros((1, 4, 64), np.float32), 64, np.zeros((64, 193)), np.zeros(193),
                         np.zeros((193, 64)), np.zeros(64))
    with pytest.raises(RuntimeError, match="downsampling|upsampling"):
        eng.op_bifpn_combine([np.zeros((1, 5, 5, 8), np.float32)], (2, 2))
