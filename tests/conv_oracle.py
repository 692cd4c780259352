"""Float64 reference of the conv kernels' contract (ConvDesc, csrc/common.h), with an element-wise error bound.

The reference convolves the operands as the kernels hold them -- the (hi, lo') planes x~ = hi + lo'/2048 in split
precision, the fp16 hi plane in fp16 precision -- with every term in float64, so what is left between a kernel's output
and the reference is the kernel's own arithmetic.  `bound` bounds that arithmetic per output element.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

LO_SCALE = 2048.0
U = 2.0 ** -24            # fp32 unit roundoff (round to nearest)
ULP = 2.0 ** -23          # fp32 ulp relative to the value, at most
ACC_DELTA = {1: 6.8e-8, 2: 1.7e-7}   # conv_tc.cu kAccDelta (chunks of one K-block), kAccDelta2 (two or more)


def split_planes(x):
    """fp32 -> (hi, lo') fp16 planes as planes.cuh splits them: hi = rn(x), lo' = rn((x - hi) * 2048), in fp32."""
    x = np.asarray(x, dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        hi = x.astype(np.float16)
        lo = ((x - hi.astype(np.float32)) * np.float32(LO_SCALE)).astype(np.float16)
    return hi, lo


def join(hi, lo=None):
    """The value planes represent, in float64."""
    v = hi.astype(np.float64)
    return v if lo is None else v + lo.astype(np.float64) / LO_SCALE


def represent(x, split=True):
    """x as the kernels hold it: hi + lo'/2048 (split) or hi (fp16), float64."""
    hi, lo = split_planes(x)
    return join(hi, lo if split else None)


def lo_part(x):
    """|lo'| / 2048 of x's planes: the part of x~ the split MMA multiplies by the other operand's hi plane only."""
    return np.abs(split_planes(x)[1].astype(np.float64)) / LO_SCALE


def view_of(buf, in_H, in_W, Cin):
    """The view [B][in_H][in_W][Cin] of buffer buf [B][pitch_H][pitch_W][in_ld] at its origin.  Pixel (b, h, w) starts at
    element ((b * pitch_H + h) * pitch_W + w) * in_ld of the buffer, so in_ld < Cin reads overlapping windows."""
    B, PH, PW, ld = buf.shape
    flat = np.ascontiguousarray(buf).reshape(-1)
    last = ((B - 1) * PH + in_H - 1) * PW * ld + (in_W - 1) * ld + Cin
    assert in_H <= PH and in_W <= PW and last <= flat.size, "view outside the buffer"
    es = flat.itemsize
    v = np.lib.stride_tricks.as_strided(flat, (B, in_H, in_W, Cin), (PH * PW * ld * es, PW * ld * es, ld * es, es),
                                        writeable=False)
    return np.array(v)


def out_size(n, pad0, pad1, k, stride, dil):
    return (n + pad0 + pad1 - ((k - 1) * dil + 1)) // stride + 1


def _conv64(x, w, stride, dil, pad):
    """Plain float64 conv of NHWC x with HWIO w; pad (t, b, l, r), negative b / r crop."""
    pt, pb, pl, pr = pad
    H, W = x.shape[1:3]
    xt = torch.from_numpy(np.ascontiguousarray(x)).permute(0, 3, 1, 2)
    xt = xt[:, :, :H + min(pb, 0), :W + min(pr, 0)]
    xt = F.pad(xt, (pl, max(pr, 0), pt, max(pb, 0)))
    wt = torch.from_numpy(np.ascontiguousarray(w)).permute(3, 2, 0, 1).contiguous()
    return F.conv2d(xt, wt, stride=stride, dilation=dil).permute(0, 2, 3, 1).numpy()


def reference(x, w, bias=None, res=None, view=None, stride=1, dil=1, pad=(0, 0, 0, 0), res_shift=0, off=(0, 0),
              relu=0, split=True):
    """The conv of buffer x [B][pitch_H][pitch_W][in_ld] (view (in_H, in_W, Cin) at its origin) with HWIO w, all Cout_pad
    columns (zero weights and bias past Cout), as float64 arrays [B][Ho][Wo][Cout_pad]:
      ref  the output: conv + bias + residual (read at the placed coordinates >> res_shift), then the activation
      pre  the same before the activation
      S    sum_k |x~_k w~_k|, the scale every accumulation error is relative to
      L    sum_k |lo_x,k lo_w,k| / 2048^2, the product the split MMA drops (0 in fp16 precision)
      b, r |bias| and |residual~| at each element."""
    B = x.shape[0]
    in_H, in_W, Cin = view if view is not None else x.shape[1:]
    R, S_, _, Cout = w.shape
    Cp = (Cout + 15) // 16 * 16
    xv = view_of(np.asarray(x, np.float32), in_H, in_W, Cin)
    wp = np.zeros((R, S_, Cin, Cp), np.float32)
    wp[..., :Cout] = w
    xr, wr = represent(xv, split), represent(wp, split)
    conv = _conv64(xr, wr, stride, dil, pad)
    Ssum = _conv64(np.abs(xr), np.abs(wr), stride, dil, pad)
    L = _conv64(lo_part(xv), lo_part(wp), stride, dil, pad) if split else np.zeros_like(conv)
    Ho, Wo = conv.shape[1:3]
    bb = np.zeros(Cp)
    if bias is not None:
        bb[:Cout] = np.asarray(bias, np.float32)
    pre = conv + bb
    r = np.zeros_like(conv)
    if res is not None:
        rr = represent(res, split)
        rows = (np.arange(Ho) + off[0]) >> res_shift
        cols = (np.arange(Wo) + off[1]) >> res_shift
        r = rr[:, rows][:, :, cols][..., :Cp]
        pre = pre + r
    if relu == 1:
        ref = np.maximum(pre, 0.0)
    elif relu == 2:
        ref = pre / (1.0 + np.exp(-pre))
    else:
        ref = pre
    return dict(ref=ref, pre=pre, S=Ssum, L=L, b=np.broadcast_to(np.abs(bb), conv.shape), r=np.abs(r),
                K=R * S_ * Cin, Ho=Ho, Wo=Wo, Cp=Cp)


def place(window, out_init, off):
    """out_init with the [B][Ho][Wo][Cp] window written at (off_h, off_w), columns [0, Cp)."""
    out = np.array(out_init, dtype=np.float64)
    Ho, Wo, Cp = window.shape[1:]
    out[:, off[0]:off[0] + Ho, off[1]:off[1] + Wo, :Cp] = window
    return out


def bound(K, S, b, r, ref, precision="split", L=None, chunk_kb=None, impl="tc", out="planes", relu=0):
    """Bound on |kernel output - reference| at each element.

    K        the reduction length R*S*Cin (K-blocks of 64 for the tensor-core kernel)
    S, b, r  sum_k |x~ w~|, |bias|, |residual~| at the element; ref the reference output
    L        sum_k |lo_x lo_w| / 2048^2 (split precision; default: its bound 2^-22 (1 + 2^-8) S for normal-range operands)
    chunk_kb the tensor-core accumulation chunk in K-blocks (ACC's acc_kb; None = the whole K in one accumulator)
    impl     "tc" (wgmma) or "simt" (fmaf chains); out "planes" (fp16 planes of the precision) or "f32"

    Terms, all relative to S unless said otherwise:
    * Dropped lo.lo (split): acc1 takes hi_x lo_w' + lo_x' hi_w and no lo_x' lo_w' -- exactly L, which is at most
      2^-11 (1 + 2^-9) |x~| * 2^-11 (1 + 2^-9) |w~| per product, i.e. 2^-22 (1 + 2^-8) S, while both operands are normal fp16.
    * Truncating accumulation inside a chunk (tc): a wgmma.k16 adds its 16 exact fp16 products into the fp32 accumulator
      and truncates; aligning the terms and truncating the sum each lose less than one ulp of the sum of magnitudes, so a
      step loses at most 2 ULP = 2^-22 of the magnitudes it has summed so far, which is at most the chunk's share S_c of S.
      A chunk of n = 4 * chunk_kb steps loses at most n 2^-22 S_c; summed over the chunks, n 2^-22 S.
      The cross-term accumulator acc1 is never restarted: 4 K/64 steps over magnitudes of at most 2^-10 (1 + 2^-9) S
      after the 1/2048 scale.  fp16 precision has acc0 alone, in one chunk.
    * Round-to-nearest folds of chunk sums (ACC): one fp32 add per chunk after the first, each within U of a running
      sum of at most S.
    * The combine fmaf(acc1, 1/2048, sum) and the acc_delta nudge fmaf(v, delta, v): U + delta + U of |v| <= S (the
      nudge moves v by delta |v| rounded, at most delta + U; delta 1.7e-7 for chunks of two or more K-blocks).
    * CUDA cores (simt): K fmaf per accumulator, each within U of a partial of at most S (acc0) or 2^-10 (1 + 2^-9) S
      (acc1, twice as many), plus the combine.
    * Epilogue: + bias, + residual hi, fmaf with the residual lo': three fp32 roundings, each within U of at most
      S + |b| + |r~|.
    * Activation: ReLU is 1-Lipschitz and exact; swish x * sigmoid(x) has |d/dx| <= 1.1, and expf, the add, the
      division and __fmul_rn add at most 8 U of |out|.
    * Output split: hi = rn(v) within 2^-11 |v| (fp16 precision: that is the output); in split precision lo' = rn((v - hi)
      * 2048) leaves at most half an ulp of lo', 2^-11 |lo'| / 2048 <= 2^-22 |v|, or 2^-25 / 2048 = 2^-36 absolute when lo'
      is an fp16 subnormal.  fp32 outputs are not rounded again.
    """
    S = np.asarray(S, np.float64)
    split = precision == "split"
    nkb = max(1, -(-K // 64))
    cross = 2.0 ** -10 * (1 + 2.0 ** -9) if split else 0.0
    if L is None:
        L = 2.0 ** -22 * (1 + 2.0 ** -8) * S if split else 0.0
    if impl == "tc":
        ckb = nkb if chunk_kb is None or chunk_kb <= 0 else min(chunk_kb, nkb)
        chunks = -(-nkb // ckb)
        acc = 4 * ckb * 2.0 ** -22 + 4 * nkb * 2.0 ** -22 * cross + (chunks - 1) * U
        if split:
            acc += 2 * U + ACC_DELTA[2]
    else:
        acc = K * U + 2 * K * U * cross + (U if split else 0.0)
    e = (acc * (1 + 1e-3)) * S + (L if split else 0.0)
    e = e + 3 * U * (S * (1 + 1e-3) + np.abs(b) + np.abs(r))
    ref = np.abs(np.asarray(ref, np.float64))
    if relu == 2:
        e = 1.1 * e + 8 * U * ref
    if out == "planes":
        e = e + (2.0 ** -22 * (ref + e) + 2.0 ** -36 if split else 2.0 ** -11 * (1 + 2.0 ** -10) * (ref + e) + 2.0 ** -25)
    return e


def acc_statistics(out, ref, S):
    """Normalised error e = (out - ref) / S over the elements with S > 0: (mean of sign(ref) e, RMS of e, standard error
    of that mean)."""
    m = S > 0
    e = (np.asarray(out, np.float64)[m] - ref[m]) / S[m]
    t = np.sign(ref[m]) * e
    return float(t.mean()), float(np.sqrt(np.mean(e * e))), float(t.std() / np.sqrt(t.size))


def acc_bias_bound(chunk_kb):
    """|mean sign(ref) e| with ACC on, for coherent sums (every product >= 0, so each chunk's partial sums grow to its
    total): a chunk of n = 4 chunk_kb wgmma steps truncates each partial toward zero by less than one ulp, at most
    ULP (1 + 2 + ... + n) / n = ULP (n + 1) / 2 of the chunk sum; the delta nudge adds back at most delta + U.  Without ACC
    the same truncation acts over all K / 16 steps, a bias that grows with K and leaves this bound at K >= 2048.  The
    nudge is taken as the larger delta: a single-chunk layer planned with acc_kb >= 2 uses it too."""
    n = 4 * chunk_kb
    return ULP * (n + 1) / 2 + ACC_DELTA[2] + U


def acc_rms_bound(K, chunk_kb, L_over_S):
    """RMS of e with ACC on: the bias bound, and the zero-mean parts as independent errors (a step's error lies in an
    interval of width 2 ULP of its partial: variance at most (2^-22)^2 / 3 of its chunk's share of S squared, whose sum
    over chunks is at most 1), the folds (U^2 / 3 each) and the dropped lo.lo product (at most L / S)."""
    nkb = max(1, K // 64)
    ckb = min(chunk_kb, nkb)
    var = (4 * ckb * 2.0 ** -44 + (-(-nkb // ckb)) * U * U) / 3
    return float(np.sqrt(acc_bias_bound(ckb) ** 2 + var + np.mean(np.square(L_over_S))))
