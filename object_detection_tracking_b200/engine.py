"""Python owner of a b2_ctx: the thin host layer above the C ABI (ctypes only; torch/numpy arrays are
just buffers).  One Detector = one device = one fixed (batch, H, W) launch plan."""
from __future__ import annotations

import ctypes
from ctypes import c_char_p, c_float, c_int32, c_int64, c_void_p

import numpy as np

from . import _lib
from .config import normalize_config
from .masks import MaskEncoder


class Detector:
    def __init__(self, cfg, batch: int, height: int, width: int, device: int = 0, input_dtype: str = "float32",
                 precision: str = "split", conv_impl: str = "tcgen05", use_cuda_graph: bool = True,
                 multi_semantics: bool = False, accum_chunk: int = 0):
        self.lib = _lib.load()
        self.cfg = normalize_config(cfg)
        self.batch, self.height, self.width = int(batch), int(height), int(width)
        self.device = int(device)
        self.input_dtype = input_dtype
        self.precision = precision
        self._c = _lib.make_config(self.cfg, batch, height, width, input_dtype, precision, conv_impl, use_cuda_graph,
                                   multi_semantics, accum_chunk)
        self._ext = _lib.make_config_ext(self.cfg)
        self._ext2 = _lib.make_config_ext2(self.cfg)
        self._ext3 = _lib.make_config_ext3(self.cfg)
        self._ext4 = _lib.make_config_ext4(self.cfg)
        self._ctx = c_void_p(0)
        _lib.check(self.lib.b2_create_ex4(ctypes.byref(self._ctx), self.device, ctypes.byref(self._c),
                                          ctypes.byref(self._ext), ctypes.byref(self._ext2), ctypes.byref(self._ext3),
                                          ctypes.byref(self._ext4)), "b2_create")
        self.R = int(self.cfg.result_per_im)
        self.C = int(self.cfg.fpn_num_channel)
        self._pinned = None

    # -- lifetime ---------------------------------------------------------------------------------
    def close(self):
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            self.lib.b2_destroy(self._ctx)
            self._ctx = c_void_p(0)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- weights ----------------------------------------------------------------------------------
    def load_weights(self, weights: dict):
        """`weights`: name -> float32 ndarray in the reference's Tensorpack-npz naming."""
        names = sorted(weights.keys())
        arrs = [np.ascontiguousarray(weights[k], dtype=np.float32) for k in names]
        n = len(names)
        c_names = (c_char_p * n)(*[k.encode() for k in names])
        c_data = (c_void_p * n)(*[a.ctypes.data for a in arrs])
        c_numel = (c_int64 * n)(*[a.size for a in arrs])
        _lib.check(self.lib.b2_load_weights(self._ctx, c_names, c_data, c_numel, n), "b2_load_weights")

    # -- the hot call -----------------------------------------------------------------------------
    def _np_dtype(self):
        return np.uint8 if self.input_dtype == "uint8" else np.float32

    def alloc_outputs(self, feat_mode: int = 0, pinned: bool = False):
        B, R, C = self.batch, self.R, self.C
        shapes = dict(boxes=((B, R, 4), np.float32), probs=((B, R), np.float32), labels=((B, R), np.int32),
                      valid=((B,), np.int32),
                      feat=({0: (B * R, C, 7, 7), 1: (B * R, C), 2: (B * R, C), 3: (B * R, 49)}[feat_mode], np.float32))
        if pinned:
            import torch
            tmap = {np.float32: torch.float32, np.int32: torch.int32}
            return {k: torch.empty(s, dtype=tmap[d]).pin_memory() for k, (s, d) in shapes.items()}
        return {k: np.empty(s, dtype=d) for k, (s, d) in shapes.items()}

    def detect_host(self, frames, out: dict | None = None, feat_mode: int = 0, want_feat: bool = True):
        """frames: [B,H,W,3] host array (numpy or pinned torch) of the configured dtype.  Returns dict of
        host arrays (boxes [B,100,4], probs, labels, valid, feat)."""
        if isinstance(frames, np.ndarray):
            frames = np.ascontiguousarray(frames, dtype=self._np_dtype())
            assert frames.shape == (self.batch, self.height, self.width, 3), frames.shape
        if out is None:
            out = self.alloc_outputs(feat_mode)
        _lib.check(self.lib.b2_detect_host(self._ctx, _lib.ptr(frames), _lib.ptr(out["boxes"]), _lib.ptr(out["probs"]),
                                           _lib.ptr(out["labels"]), _lib.ptr(out["valid"]),
                                           _lib.ptr(out["feat"]) if want_feat else c_void_p(0), feat_mode),
                   "b2_detect_host")
        return out

    def detect_host_resize(self, frames_u8, out: dict | None = None, feat_mode: int = 0, want_feat: bool = True):
        """Source-resolution uint8 frames [B,h,w,3] (BGR): upload, resize on the device to the configured height x width
        (cv2.resize INTER_LINEAR arithmetic, nn.py:1540-1545), then the pass.  Needs input_dtype="float32"."""
        frames_u8 = np.ascontiguousarray(frames_u8, dtype=np.uint8)
        assert frames_u8.ndim == 4 and frames_u8.shape[0] == self.batch and frames_u8.shape[3] == 3, frames_u8.shape
        if out is None:
            out = self.alloc_outputs(feat_mode)
        _lib.check(self.lib.b2_detect_host_resize(self._ctx, _lib.ptr(frames_u8), int(frames_u8.shape[1]),
                                                  int(frames_u8.shape[2]), _lib.ptr(out["boxes"]), _lib.ptr(out["probs"]),
                                                  _lib.ptr(out["labels"]), _lib.ptr(out["valid"]),
                                                  _lib.ptr(out["feat"]) if want_feat else c_void_p(0), feat_mode),
                   "b2_detect_host_resize")
        return out

    def box_features(self, frame, boxes) -> np.ndarray:
        """RCNN_FPN_givenbox (models.py:1816-1967): [n, 256] mean-pooled ROI features of the given boxes on one frame
        (batch-1 context)."""
        frame = np.ascontiguousarray(frame, dtype=self._np_dtype())
        assert frame.shape == (self.height, self.width, 3), frame.shape
        boxes = np.ascontiguousarray(boxes, dtype=np.float32).reshape(-1, 4)
        out = np.empty((len(boxes), self.C), dtype=np.float32)
        _lib.check(self.lib.b2_box_features(self._ctx, _lib.ptr(frame), _lib.ptr(boxes), len(boxes), _lib.ptr(out)),
                   "b2_box_features")
        return out

    def get_masks(self) -> np.ndarray:
        """final_masks of the last pass (config.add_mask): [B, result_per_im, 28, 28] float32 (models.py:958-961)."""
        out = np.empty((self.batch, int(self.cfg.result_per_im), 28, 28), dtype=np.float32)
        _lib.check(self.lib.b2_get_masks(self._ctx, _lib.ptr(out), out.nbytes), "b2_get_masks")
        return out

    def encode_masks(self, boxes_scaled, im_shape, image: int = 0) -> list:
        """COCO RLE of the final_masks of image `image` of the last pass (config.add_mask), pasted as fill_full_mask pastes
        them: boxes_scaled float32 [n, 4] are that image's first n final boxes divided by the resize scale, im_shape the
        source frame's (H, W).  The masks are read in place on the GPU (masks.py)."""
        if getattr(self, "_mask_encoder", None) is None:
            self._mask_encoder = MaskEncoder(self.device)
        return self._mask_encoder.encode_engine(self._ctx, image, boxes_scaled, im_shape)

    def get_small_objects(self) -> dict:
        """The small-object branch's outputs of the last pass (config.use_small_object_head, models.py:880-897): boxes
        [n, 4] float32, probs [n] float32 (logits, models.py:884), labels [n] int32 in 1..C, plus class_counts [C] (boxes
        each small class kept by its NMS) and status (0, or 1 when those counts differ: then n = 0)."""
        R, C = self.R, len(self.cfg.small_object_class_ids)
        boxes, probs = np.empty((R, 4), np.float32), np.empty((R,), np.float32)
        labels, count = np.empty((R,), np.int32), np.empty((1,), np.int32)
        counts, status = np.empty((C,), np.int32), np.empty((1,), np.int32)
        _lib.check(self.lib.b2_get_small_objects(self._ctx, *[_lib.ptr(a) for a in (boxes, probs, labels, count, counts,
                                                                                      status)]), "b2_get_small_objects")
        n = int(count[0])
        return dict(boxes=boxes[:n].copy(), probs=probs[:n].copy(), labels=labels[:n].copy(), class_counts=counts,
                    status=int(status[0]))

    def submit_host(self, frames, out: dict, slot: int, feat_mode: int = 0, want_feat: bool = True):
        """Asynchronous detect_host: enqueue upload + pass + download for `slot` (0/1) and return; `frames` and the
        arrays of `out` must stay alive (pinned for real overlap) until wait(slot).  Streaming drivers alternate slots
        so that the upload of the next batch overlaps the pass of the current one."""
        if isinstance(frames, np.ndarray):
            frames = np.ascontiguousarray(frames, dtype=self._np_dtype())     # a copy only when the caller's array needs one
            assert frames.shape == (self.batch, self.height, self.width, 3), frames.shape
        if not hasattr(self, "_inflight"):
            self._inflight = {}
        self._inflight[int(slot)] = (frames, out)                             # keep the buffers alive until wait()
        _lib.check(self.lib.b2_submit_host(self._ctx, _lib.ptr(frames), _lib.ptr(out["boxes"]), _lib.ptr(out["probs"]),
                                           _lib.ptr(out["labels"]), _lib.ptr(out["valid"]),
                                           _lib.ptr(out["feat"]) if want_feat else c_void_p(0), feat_mode, int(slot)),
                   "b2_submit_host")

    def submit_host_resize(self, frames_u8, out: dict, slot: int, feat_mode: int = 0, want_feat: bool = True):
        """submit_host for uint8 source frames [B,h,w,3] that are resized on the device (detect_host_resize, pipelined)."""
        if isinstance(frames_u8, np.ndarray):
            frames_u8 = np.ascontiguousarray(frames_u8, dtype=np.uint8)
        assert frames_u8.shape[0] == self.batch and frames_u8.shape[3] == 3, frames_u8.shape
        if not hasattr(self, "_inflight"):
            self._inflight = {}
        self._inflight[int(slot)] = (frames_u8, out)
        _lib.check(self.lib.b2_submit_host_resize(self._ctx, _lib.ptr(frames_u8), int(frames_u8.shape[1]),
                                                  int(frames_u8.shape[2]), _lib.ptr(out["boxes"]), _lib.ptr(out["probs"]),
                                                  _lib.ptr(out["labels"]), _lib.ptr(out["valid"]),
                                                  _lib.ptr(out["feat"]) if want_feat else c_void_p(0), feat_mode, int(slot)),
                   "b2_submit_host_resize")

    def wait(self, slot: int):
        _lib.check(self.lib.b2_wait(self._ctx, int(slot)), "b2_wait")
        getattr(self, "_inflight", {}).pop(int(slot), None)

    def detect_device(self, frames_dev, out_dev: dict | None = None, feat_mode: int = 0, sync: bool = True):
        """frames_dev / out_dev: torch CUDA tensors (or None to leave results in the context)."""
        o = out_dev or {}
        _lib.check(self.lib.b2_detect(self._ctx, _lib.ptr(frames_dev), _lib.ptr(o.get("boxes")),
                                      _lib.ptr(o.get("probs")), _lib.ptr(o.get("labels")), _lib.ptr(o.get("valid")),
                                      _lib.ptr(o.get("feat")), feat_mode, int(sync)), "b2_detect")
        return out_dev

    # -- stage access (parity tests) ----------------------------------------------------------------
    def stage_shape(self, name: str):
        shape = (c_int64 * 4)()
        dt = c_int32(0)
        _lib.check(self.lib.b2_stage_shape(self._ctx, name.encode(), shape, ctypes.byref(dt)), "b2_stage_shape")
        return tuple(int(v) for v in shape), (np.int32 if dt.value == 1 else np.float32)

    def get_stage(self, name: str) -> np.ndarray:
        shape, dt = self.stage_shape(name)
        a = np.empty(shape, dtype=dt)
        _lib.check(self.lib.b2_get_stage(self._ctx, name.encode(), _lib.ptr(a), a.nbytes), "b2_get_stage")
        return a

    def set_stage(self, name: str, value: np.ndarray):
        if name == "image":
            a = np.ascontiguousarray(value, dtype=self._np_dtype())
        else:
            _, dt = self.stage_shape(name)
            a = np.ascontiguousarray(value, dtype=dt)
        _lib.check(self.lib.b2_set_stage(self._ctx, name.encode(), _lib.ptr(a), a.nbytes), "b2_set_stage")

    def run_phases(self, mask: int = 255):
        _lib.check(self.lib.b2_run_phases(self._ctx, int(mask)), "b2_run_phases")

    def phase_times(self) -> dict:
        ms = (c_float * 8)()
        _lib.check(self.lib.b2_phase_times(self._ctx, ms), "b2_phase_times")
        return {n: float(ms[i]) for i, n in enumerate(_lib.PHASE_NAMES)}

    def kernel_launches(self) -> int:
        return int(self.lib.b2_kernel_launches(self._ctx))

    def profile_steps(self, reps: int = 3) -> list:
        """Per launch group: dict(name, kind, ms, flops, bytes) -- device time from CUDA events."""
        n = int(self.lib.b2_num_steps(self._ctx))
        ms = (c_float * n)()
        nout = ctypes.c_int(0)
        _lib.check(self.lib.b2_profile_steps(self._ctx, int(reps), ms, n, ctypes.byref(nout)), "b2_profile_steps")
        out = []
        buf = ctypes.create_string_buffer(256)
        for i in range(nout.value):
            fl, by, kind = ctypes.c_double(0), ctypes.c_double(0), ctypes.c_int(0)
            _lib.check(self.lib.b2_step_info(self._ctx, i, buf, 256, ctypes.byref(fl), ctypes.byref(by),
                                             ctypes.byref(kind)), "b2_step_info")
            out.append(dict(name=buf.value.decode(), kind=kind.value, ms=float(ms[i]), flops=fl.value, bytes=by.value))
        return out


def cosine_cost(gallery: np.ndarray, seg_offsets: np.ndarray, dets: np.ndarray, device: int = 0,
                precision: str = "split") -> np.ndarray:
    """[T, N] appearance cost = per-track min over gallery rows of (1 - cosine) on the GPU."""
    lib = _lib.load()
    gallery = np.ascontiguousarray(gallery, dtype=np.float32)
    dets = np.ascontiguousarray(dets, dtype=np.float32)
    seg = np.ascontiguousarray(seg_offsets, dtype=np.int32)
    T = seg.shape[0] - 1
    N, D = dets.shape
    cost = np.zeros((T, N), dtype=np.float32)
    if T == 0 or N == 0:
        return cost
    _lib.check(lib.b2_cosine_cost(device, _lib.ptr(gallery), _lib.ptr(seg), T, _lib.ptr(dets), N, D,
                                  {"fp16": 0, "split": 1}[precision], _lib.ptr(cost)), "b2_cosine_cost")
    return cost


def op_conv2d(x, w, bias=None, res=None, stride=1, dil=1, pad=(0, 0, 0, 0), relu=False, res_shift=0,
              impl="tcgen05", split=True, a_mode=-1, device=0) -> np.ndarray:
    """Single convolution through the C ABI (NHWC activations, HWIO kernel) -- used by the kernel tests."""
    lib = _lib.load()
    x = np.ascontiguousarray(x, dtype=np.float32)
    w = np.ascontiguousarray(w, dtype=np.float32)
    B, H, W, Cin = x.shape
    R, S, _, Cout = w.shape
    pt, pb, pl, pr = pad
    Ho = (H + pt + pb - ((R - 1) * dil + 1)) // stride + 1
    Wo = (W + pl + pr - ((S - 1) * dil + 1)) // stride + 1
    out = np.zeros((B, Ho, Wo, Cout), dtype=np.float32)
    b = None if bias is None else np.ascontiguousarray(bias, dtype=np.float32)
    r = None if res is None else np.ascontiguousarray(res, dtype=np.float32)
    _lib.check(lib.b2_op_conv2d(device, _lib.ptr(x), _lib.ptr(w), _lib.ptr(b), _lib.ptr(r), B, H, W, Cin, R, S, Cout,
                                stride, dil, pt, pb, pl, pr, int(relu), int(res_shift),
                                {"tcgen05": 0, "simt": 1}[impl], int(split), int(a_mode), _lib.ptr(out)),
               "b2_op_conv2d")
    return out


def op_conv2d_view(x, w, bias=None, res=None, view=None, stride=1, dil=1, pad=(0, 0, 0, 0), out_init=None, off=(0, 0),
                   out_f32=False, res_shift=0, relu=0, acc_kb=0, a_mode=-1, force_epi=-1, impl="tcgen05", split=True,
                   images=None, device=0):
    """Single convolution with the whole conv-kernel contract through the C ABI -- used by the kernel tests.

    x [B, pitch_H, pitch_W, in_ld] is the whole input buffer and view = (in_H, in_W, Cin) the view at its origin (default:
    all of it; in_ld < Cin reads overlapping windows).  w is HWIO [R, S, Cin, Cout]; res [B, res_H, res_W, ldr] is read at
    the placed output coordinates >> res_shift.  out_init [B, out_H, out_W, ldc] is the output buffer before the launch
    (default: zeros of [B, Ho, Wo, Cout_pad]); the Ho x Wo result lands at off = (off_h, off_w).  images = (b0, nb) launches
    over those images only.  Returns (out, hi, lo, flag): the whole buffer after the launch as fp32, the raw fp16 planes
    as uint16 (None for an fp32 output; lo None in fp16 precision) and the range-monitor word."""
    lib = _lib.load()
    x = np.ascontiguousarray(x, dtype=np.float32)
    w = np.ascontiguousarray(w, dtype=np.float32)
    B, PH, PW, ld = x.shape
    in_H, in_W, Cin = view if view is not None else (PH, PW, ld)
    R, S, _, Cout = w.shape
    pt, pb, pl, pr = pad
    if out_init is None:
        Ho = (in_H + pt + pb - ((R - 1) * dil + 1)) // stride + 1
        Wo = (in_W + pl + pr - ((S - 1) * dil + 1)) // stride + 1
        out_init = np.zeros((B, max(Ho, 1), max(Wo, 1), (Cout + 15) // 16 * 16), dtype=np.float32)
    out_init = np.ascontiguousarray(out_init, dtype=np.float32)
    a = _lib.B2ConvView()
    a.B, a.pitch_H, a.pitch_W, a.in_ld, a.in_H, a.in_W, a.Cin = B, PH, PW, ld, in_H, in_W, Cin
    a.R, a.S, a.stride, a.dil, a.pad_t, a.pad_b, a.pad_l, a.pad_r = R, S, stride, dil, pt, pb, pl, pr
    a.Cout = Cout
    _, a.out_H, a.out_W, a.ldc = out_init.shape
    a.off_h, a.off_w = off
    a.out_f32 = int(bool(out_f32))
    b = None if bias is None else np.ascontiguousarray(bias, dtype=np.float32)
    r = None if res is None else np.ascontiguousarray(res, dtype=np.float32)
    if r is not None:
        _, a.res_H, a.res_W, a.ldr = r.shape
        a.res_shift = res_shift
    a.relu, a.acc_kb, a.a_mode, a.force_epi = int(relu), acc_kb, a_mode, force_epi
    a.impl, a.split = {"tcgen05": 0, "simt": 1}[impl], int(bool(split))
    a.b0, a.nb = images if images is not None else (0, 0)
    out = np.empty_like(out_init)
    hi = lo = None
    if not out_f32:
        hi = np.empty(out_init.shape, dtype=np.uint16)
        lo = np.empty(out_init.shape, dtype=np.uint16) if split else None
    flag = np.zeros(1, dtype=np.uint32)
    _lib.check(lib.b2_op_conv2d_view(device, ctypes.byref(a), _lib.ptr(x), _lib.ptr(w), _lib.ptr(b), _lib.ptr(r),
                                     _lib.ptr(out_init), _lib.ptr(out), _lib.ptr(hi), _lib.ptr(lo), _lib.ptr(flag)),
               "b2_op_conv2d_view")
    return out, hi, lo, int(flag[0])


def op_group_conv2d(x, w, bias=None, res=None, stride=1, dil=1, pad=(0, 0, 0, 0), relu=False, impl="tcgen05",
                    split=True, device=0) -> np.ndarray:
    """Grouped convolution through the C ABI -- used by the kernel tests: x [B, H, W, C] NHWC, HWIO kernel
    w [R, S, C / groups, C] (TF's grouped conv2d, nn.py:352-355), res [B, Ho, Wo, C]."""
    lib = _lib.load()
    x = np.ascontiguousarray(x, dtype=np.float32)
    w = np.ascontiguousarray(w, dtype=np.float32)
    B, H, W, C = x.shape
    R, S, cg, Cout = w.shape
    assert Cout == C and C % cg == 0, (w.shape, C)
    pt, pb, pl, pr = pad
    Ho = (H + pt + pb - ((R - 1) * dil + 1)) // stride + 1
    Wo = (W + pl + pr - ((S - 1) * dil + 1)) // stride + 1
    out = np.zeros((B, Ho, Wo, C), dtype=np.float32)
    b = None if bias is None else np.ascontiguousarray(bias, dtype=np.float32)
    r = None if res is None else np.ascontiguousarray(res, dtype=np.float32)
    assert r is None or r.shape == out.shape, r.shape
    _lib.check(lib.b2_op_group_conv2d(device, _lib.ptr(x), _lib.ptr(w), _lib.ptr(b), _lib.ptr(r), B, H, W, C, R, S,
                                      C // cg, stride, dil, pt, pb, pl, pr, int(relu), {"tcgen05": 0, "simt": 1}[impl],
                                      int(split), _lib.ptr(out)),
               "b2_op_group_conv2d")
    return out


def op_group_norm(x, gamma, beta, view=None, res=None, res_shift=0, relu=False, per_roi=False, split=True,
                  in_place=True, device=0) -> np.ndarray:
    """GroupNorm (32 groups) of a NHWC buffer x [B, pitch_H, pitch_W, C] through the C ABI -- used by the kernel tests.
    view = (off_h, off_w, H, W) restricts it to a window (default: the whole buffer); res [B, rH, rW, C] is added after
    the normalisation at (y >> res_shift, x >> res_shift), then ReLU.  Returns the buffer after the op (in_place) or a
    zero-initialised output buffer of which only the view is written."""
    lib = _lib.load()
    x = np.ascontiguousarray(x, dtype=np.float32)
    B, PH, PW, C = x.shape
    oh, ow, H, W = view if view is not None else (0, 0, PH, PW)
    r = None if res is None else np.ascontiguousarray(res, dtype=np.float32)
    rH, rW = (0, 0) if r is None else r.shape[1:3]
    out = np.zeros_like(x)
    _lib.check(lib.b2_op_group_norm(device, _lib.ptr(x), _lib.ptr(r), _lib.ptr(np.ascontiguousarray(gamma, np.float32)),
                                    _lib.ptr(np.ascontiguousarray(beta, np.float32)), B, PH, PW, C, H, W, oh, ow, rH, rW,
                                    int(res_shift), int(relu), int(per_roi), int(split), int(in_place), _lib.ptr(out)),
               "b2_op_group_norm")
    return out


def op_squeeze_excite(x, w1, b1, w2, b2, res=None, split=True, device=0):
    """The SE-ResNet bottleneck's squeeze-excite through the C ABI -- used by the kernel tests: x [B, H, W, C] NHWC,
    dense w1 [C, nr], w2 [nr, C].  Returns (relu(x * gate[b] + res), gate [B, C])."""
    lib = _lib.load()
    x = np.ascontiguousarray(x, dtype=np.float32)
    B, H, W, C = x.shape
    w1 = np.ascontiguousarray(w1, dtype=np.float32)
    nr = w1.shape[1]
    assert w1.shape == (C, nr) and np.shape(w2) == (nr, C), (w1.shape, np.shape(w2))
    r = None if res is None else np.ascontiguousarray(res, dtype=np.float32)
    assert r is None or r.shape == x.shape, r.shape
    out = np.empty_like(x)
    gate = np.empty((B, C), dtype=np.float32)
    _lib.check(lib.b2_op_squeeze_excite(device, _lib.ptr(x), _lib.ptr(r), _lib.ptr(w1),
                                        _lib.ptr(np.ascontiguousarray(b1, np.float32)),
                                        _lib.ptr(np.ascontiguousarray(w2, np.float32)),
                                        _lib.ptr(np.ascontiguousarray(b2, np.float32)), B, H, W, C, nr, int(split),
                                        _lib.ptr(out), _lib.ptr(gate)),
               "b2_op_squeeze_excite")
    return out, gate


def op_relation(h, boxes, count, weights, split=True, device=0) -> np.ndarray:
    """One relation module of the box head (relation_network nn.py:115-190) through the C ABI -- used by the kernel tests:
    h [B, K, D] head rows, boxes [B, K, 4] proposals (x1, y1, x2, y2), count [B] valid rows per image, `weights` the
    module's arrays keyed by their names under the module scope (geo_emb/W, geo_emb/b, geo_conv/W, geo_conv/b,
    query_linear/W, key_linear/W, output_linear/W).  Returns h + RM(h, boxes) [B, K, D]; rows i >= count[b] are h."""
    lib = _lib.load()
    h = np.ascontiguousarray(h, dtype=np.float32)
    B, K, D = h.shape
    boxes = np.ascontiguousarray(boxes, dtype=np.float32)
    count = np.ascontiguousarray(count, dtype=np.int32)
    assert boxes.shape == (B, K, 4) and count.shape == (B,), (boxes.shape, count.shape)
    shapes = {"geo_emb/W": (4, 64), "geo_emb/b": (64,), "geo_conv/W": (1, 1, 64, 16), "geo_conv/b": (16,),
              "query_linear/W": (D, D), "key_linear/W": (D, D), "output_linear/W": (16 * D, D)}
    w = {k: np.ascontiguousarray(weights[k], dtype=np.float32) for k in shapes}
    for k, s in shapes.items():
        assert w[k].size == int(np.prod(s)), (k, w[k].shape, s)
    out = np.empty_like(h)
    _lib.check(lib.b2_op_relation(device, _lib.ptr(h), _lib.ptr(boxes), _lib.ptr(count),
                                  *[_lib.ptr(w[k]) for k in shapes], B, K, D, int(split), _lib.ptr(out)),
               "b2_op_relation")
    return out


def op_deform_sample(x, offsets, split=True, device=0) -> np.ndarray:
    """The deformable conv's bilinear sampler through the C ABI -- used by the kernel tests: x [B, H, W, C] NHWC,
    offsets [B, ceil(H/2), ceil(W/2), 18] (channel 2k the y, 2k + 1 the x offset of tap k).  Returns the sampled operand
    [B, ceil(H/2), ceil(W/2), 9, C] as its planes store it."""
    lib = _lib.load()
    x = np.ascontiguousarray(x, dtype=np.float32)
    B, H, W, C = x.shape
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    off = np.ascontiguousarray(offsets, dtype=np.float32)
    assert off.shape == (B, Ho, Wo, 18), off.shape
    out = np.empty((B, Ho, Wo, 9, C), dtype=np.float32)
    _lib.check(lib.b2_op_deform_sample(device, _lib.ptr(x), _lib.ptr(off), B, H, W, C, int(split), _lib.ptr(out)),
               "b2_op_deform_sample")
    return out


def op_deform_conv2d(x, offset_w, offset_b, w, impl="tcgen05", split=True, return_offsets=False, device=0):
    """A deformable conv2 (deformable_conv2d nn.py:1642-1712 with its conv2_offset, nn.py:470-486) through the C ABI --
    used by the kernel tests: x [B, H, W, C] NHWC, offset_w [3, 3, C, 18], offset_b [18], w [3, 3, C, Cout].  Returns
    out [B, ceil(H/2), ceil(W/2), Cout], and the offsets [B, ceil(H/2), ceil(W/2), 18] with return_offsets."""
    lib = _lib.load()
    x = np.ascontiguousarray(x, dtype=np.float32)
    B, H, W, C = x.shape
    ow = np.ascontiguousarray(offset_w, dtype=np.float32)
    ob = np.ascontiguousarray(offset_b, dtype=np.float32)
    w = np.ascontiguousarray(w, dtype=np.float32)
    Cout = w.shape[3]
    assert ow.shape == (3, 3, C, 18) and ob.shape == (18,) and w.shape == (3, 3, C, Cout), (ow.shape, ob.shape, w.shape)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    out = np.empty((B, Ho, Wo, Cout), dtype=np.float32)
    off = np.empty((B, Ho, Wo, 18), dtype=np.float32)
    _lib.check(lib.b2_op_deform_conv2d(device, _lib.ptr(x), _lib.ptr(ow), _lib.ptr(ob), _lib.ptr(w), B, H, W, C, Cout,
                                       {"tcgen05": 0, "simt": 1}[impl], int(split), _lib.ptr(out), _lib.ptr(off)),
               "b2_op_deform_conv2d")
    return (out, off) if return_offsets else out


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def op_mask_head(boxes, count, labels, num_class, feats=None, level_hw=None, strides=(4, 8, 16, 32), weights=None,
                 logits=None, split=True, outputs=("roi", "fcn", "up", "logits"), device=0) -> dict:
    """The mask head (models.py:934-961, 1173-1199) through the engine's builder -- used by the kernel tests: feats p2..p5
    [B, pitch_H, pitch_W, 256] each, level_hw their cropped (H, W), boxes [B, R, 4], count [B], labels [B, R] (1 ..
    num_class - 1 below the count), `weights` the maskrcnn/* arrays under their checkpoint names.  Returns a dict: roi
    [M, 14, 14, 256] (M = B R), fcn [4, M, 14, 14, 256], up [M, 14, 14, 1024] (the deconv's (tap, channel) outputs), each
    with its raw planes "<name>_hi" / "<name>_lo" (lo None in fp16 precision); logits [M * 784, ld]; masks [B, R, 28, 28].
    `outputs` names the ones fetched besides masks.  logits given ([M * 784, ld]) runs the own-class sigmoid alone on them:
    the dict then holds masks only."""
    lib = _lib.load()
    boxes = _f32(boxes)
    B, R = boxes.shape[:2]
    count = np.ascontiguousarray(count, dtype=np.int32)
    labels = np.ascontiguousarray(labels, dtype=np.int32)
    assert boxes.shape == (B, R, 4) and count.shape == (B,) and labels.shape == (B, R), (boxes.shape, count.shape,
                                                                                         labels.shape)
    M, C, ld = B * R, 256, (num_class - 1 + 15) // 16 * 16
    out = dict(masks=np.empty((B, R, 28, 28), np.float32))
    null = (c_void_p(0),) * 3
    if logits is not None:
        lg = _f32(logits)
        assert lg.shape == (M * 784, ld), (lg.shape, (M * 784, ld))
        _lib.check(lib.b2_op_mask_head(device, None, None, None, C, B, R, None, _lib.ptr(count), _lib.ptr(labels),
                                       int(num_class), None, None, None, 0, _lib.ptr(lg), int(split), *null, *null, *null,
                                       None, _lib.ptr(out["masks"])),
                   "b2_op_mask_head")
        return out
    fs = [_f32(f) for f in feats]
    assert len(fs) == 4 and all(f.shape[0] == B and f.shape[3] == C for f in fs), [f.shape for f in fs]
    flat = np.ascontiguousarray(np.concatenate([f.ravel() for f in fs]))
    hw = np.array([[f.shape[1], f.shape[2], h, w] for f, (h, w) in zip(fs, level_hw)], np.int32)
    st = np.asarray(strides, np.float32)
    names = sorted(weights)
    arrs = [_f32(weights[k]) for k in names]
    for k, shape in (("roi", (M, 14, 14, C)), ("fcn", (4, M, 14, 14, C)), ("up", (M, 14, 14, 4 * C))):
        if k in outputs:
            out[k], out[k + "_hi"], out[k + "_lo"] = _plane_outputs(shape, split)
    if "logits" in outputs:
        out["logits"] = np.empty((M * 784, ld), np.float32)
    planes = [_lib.ptr(out.get(k + s)) for k in ("roi", "fcn", "up") for s in ("", "_hi", "_lo")]
    _lib.check(lib.b2_op_mask_head(device, _lib.ptr(flat), _lib.ptr(hw), _lib.ptr(st), C, B, R, _lib.ptr(boxes),
                                   _lib.ptr(count), _lib.ptr(labels), int(num_class),
                                   (c_char_p * len(names))(*[k.encode() for k in names]),
                                   (c_void_p * len(names))(*[a.ctypes.data for a in arrs]),
                                   (c_int64 * len(names))(*[a.size for a in arrs]), len(names), None, int(split), *planes,
                                   _lib.ptr(out.get("logits")), _lib.ptr(out["masks"])),
               "b2_op_mask_head")
    return out


def _plane_outputs(shape, split):
    """fp32 output and its raw planes (uint16; lo None in fp16 precision) of a plane-output op."""
    return (np.empty(shape, np.float32), np.empty(shape, np.uint16),
            np.empty(shape, np.uint16) if split else None)


def op_depthwise(x, w, bias=None, stride=1, pad=(0, 0), out_hw=None, act="none", impl="effnet", split=True, device=0):
    """One depthwise conv through the C ABI -- used by the kernel tests: x [B, H, W, C] NHWC, w [K, K, C], bias [C].
    impl "effnet": EfficientNet's strip kernel (B = 1; pad = (pad_t, pad_l), output size out_hw; act "none" / "swish");
    impl "osnet": OSNet's 3x3 stride-1 pad-1 conv + bias + ReLU (act "relu").  Returns (out, hi, lo) as
    op_conv2d_view does."""
    lib = _lib.load()
    x = _f32(x)
    w = _f32(w)
    B, H, W, C = x.shape
    K = w.shape[0]
    assert w.shape == (K, K, C), w.shape
    Ho, Wo = out_hw if out_hw is not None else (H, W)
    out, hi, lo = _plane_outputs((B, Ho, Wo, C), split)
    _lib.check(lib.b2_op_depthwise(device, _lib.ptr(x), _lib.ptr(w), _lib.ptr(_f32(bias)), B, H, W, C, K, stride,
                                   pad[0], pad[1], Ho, Wo, {"none": 0, "relu": 1, "swish": 2}[act],
                                   {"effnet": 0, "osnet": 1}[impl], int(split), _lib.ptr(out), _lib.ptr(hi),
                                   _lib.ptr(lo)),
               "b2_op_depthwise")
    return out, hi, lo


def op_pool(x, kind, out_hw=None, out_ld=None, out_init=None, split=True, device=0):
    """One pool through the C ABI -- used by the kernel tests: x [B, H, W, C] NHWC.  kind "max": the stems' 3x3/2
    max-pool (inputs >= 0) with the caller's output size out_hw; "avg2": AvgPool2d(2); "gap": the global average pool
    into a [B, out_ld] fp32 buffer that starts as out_init (default zeros).  Returns (out, hi, lo); hi, lo are None for
    "gap"."""
    lib = _lib.load()
    x = _f32(x)
    B, H, W, C = x.shape
    k = {"max": 0, "avg2": 1, "gap": 2}[kind]
    hi = lo = None
    Ho = Wo = 0
    if k == 2:
        ld = out_ld or C
        out = np.zeros((B, ld), np.float32) if out_init is None else np.array(out_init, np.float32, copy=True)
        assert out.shape == (B, ld), out.shape
    else:
        ld = 0
        Ho, Wo = out_hw if k == 0 else (H // 2, W // 2)
        out, hi, lo = _plane_outputs((B, Ho, Wo, C), split)
    _lib.check(lib.b2_op_pool(device, _lib.ptr(x), k, B, H, W, C, Ho, Wo, ld, int(split), _lib.ptr(out), _lib.ptr(hi),
                              _lib.ptr(lo)),
               "b2_op_pool")
    return out, hi, lo


def op_bifpn_combine(inputs, out_hw, weights=None, swish=False, split=True, device=0):
    """One BiFPN node combine through the C ABI -- used by the kernel tests: inputs a list of 1 to 3 [B, H_i, W_i, C]
    maps, each resampled to out_hw as the EfficientDet engine does; weights the raw fastattn weights (None: plain sum).
    Returns (out, hi, lo, resample) with resample [n, 3] = (mode, pad_t, pad_l) per input."""
    lib = _lib.load()
    xs = [_f32(t) for t in inputs]
    B, C = xs[0].shape[0], xs[0].shape[3]
    assert all(t.shape[0] == B and t.shape[3] == C for t in xs), [t.shape for t in xs]
    flat = np.ascontiguousarray(np.concatenate([t.ravel() for t in xs]))
    hw = np.array([t.shape[1:3] for t in xs], np.int32)
    wts = None if weights is None else _f32(np.asarray(weights, np.float32).reshape(len(xs)))
    Ho, Wo = out_hw
    out, hi, lo = _plane_outputs((B, Ho, Wo, C), split)
    res = np.zeros((len(xs), 3), np.int32)
    _lib.check(lib.b2_op_bifpn_combine(device, _lib.ptr(flat), _lib.ptr(hw), _lib.ptr(wts), len(xs), B, Ho, Wo, C,
                                       int(bool(swish)), int(split), _lib.ptr(out), _lib.ptr(hi), _lib.ptr(lo),
                                       _lib.ptr(res)),
               "b2_op_bifpn_combine")
    return out, hi, lo, res


def op_mbconv_se(x, creal, w1, b1, w2, b2, w=None, split=True, device=0):
    """MBConv's squeeze-excite through the C ABI -- used by the kernel tests: x [B, HW, Cpad] with channels [0, creal)
    live, w1 [creal, nr], b1 [nr], w2 [nr, creal], b2 [creal]; w the projection's master weight [rows, Cpad] (B = 1) or
    None.  Returns (gate [B, Cpad], folded, hi, lo): the folded weight joined and as raw planes (None without w)."""
    lib = _lib.load()
    x = _f32(x)
    B, HW, Cp = x.shape
    w1 = _f32(w1)
    nr = w1.shape[1]
    assert w1.shape == (creal, nr) and np.shape(w2) == (nr, creal), (w1.shape, np.shape(w2))
    w = _f32(w)
    rows = 0 if w is None else w.shape[0]
    assert w is None or w.shape == (rows, Cp), w.shape
    gate = np.empty((B, Cp), np.float32)
    folded = hi = lo = None
    if w is not None:
        folded, hi, lo = _plane_outputs((rows, Cp), split)
    _lib.check(lib.b2_op_mbconv_se(device, _lib.ptr(x), _lib.ptr(w1), _lib.ptr(_f32(b1)), _lib.ptr(_f32(w2)),
                                   _lib.ptr(_f32(b2)), _lib.ptr(w), B, HW, Cp, creal, nr, rows, int(split),
                                   _lib.ptr(gate), _lib.ptr(folded), _lib.ptr(hi), _lib.ptr(lo)),
               "b2_op_mbconv_se")
    return gate, folded, hi, lo


def op_channel_gate(streams, creal, w1=None, b1=None, w2=None, b2=None, gates=None, split=True, device=0):
    """OSNet's ChannelGate and 4-stream gated sum through the C ABI -- used by the kernel tests: streams [4, B, HW, C]
    with channels [0, creal) live, w1 [Cr, creal], b1 [Cr], w2 [creal, Cr], b2 [creal]; gates [B, 4, C] given instead
    runs the gated sum alone.  Returns (gates [B, 4, C], out, hi, lo) with out [B, HW, C]."""
    lib = _lib.load()
    s = _f32(streams)
    _, B, HW, C = s.shape
    assert s.shape[0] == 4, s.shape
    cr = 1 if w1 is None else np.shape(w1)[0]
    g_in = _f32(gates)
    assert g_in is None or g_in.shape == (B, 4, C), g_in.shape
    g_out = np.empty((B, 4, C), np.float32)
    out, hi, lo = _plane_outputs((B, HW, C), split)
    _lib.check(lib.b2_op_channel_gate(device, _lib.ptr(s), _lib.ptr(_f32(w1)), _lib.ptr(_f32(b1)), _lib.ptr(_f32(w2)),
                                      _lib.ptr(_f32(b2)), _lib.ptr(g_in), B, HW, C, creal, cr, int(split),
                                      _lib.ptr(g_out), _lib.ptr(out), _lib.ptr(hi), _lib.ptr(lo)),
               "b2_op_channel_gate")
    return g_out, out, hi, lo


def op_stem_im2col(img, out_hw, pad, split=True, device=0):
    """EfficientNet's stem im2col through the C ABI -- used by the kernel tests: img [H, W, 3] fp32, out_hw = (Ho, Wo),
    pad = (pad_t, pad_l).  Returns (out, hi, lo) of the [Ho, Wo, 64] operand."""
    lib = _lib.load()
    img = _f32(img)
    H, W, _ = img.shape
    Ho, Wo = out_hw
    out, hi, lo = _plane_outputs((Ho, Wo, 64), split)
    _lib.check(lib.b2_op_stem_im2col(device, _lib.ptr(img), H, W, Ho, Wo, pad[0], pad[1], int(split), _lib.ptr(out),
                                     _lib.ptr(hi), _lib.ptr(lo)),
               "b2_op_stem_im2col")
    return out, hi, lo


def op_stem_pack(frames, layout, out_hw, split=True, device=0):
    """The ResNet stems' operand pack through the C ABI -- used by the kernel tests: frames [B, H, W, 3] uint8 or float32
    (float32 for the detector only).  layout "detector": the compact [B, Hu, Wv, 16] operand of conv0 (BGR frames, the
    detector's normalisation); "reid": the [B, Hu, Wu, 64] operand of the ReID engines' conv1 (RGB crops, torchvision
    ToTensor + Normalize).  out_hw = (Hu, Wv) or (Hu, Wu).  Returns (out, hi, lo) as op_conv2d_view does."""
    lib = _lib.load()
    frames = np.ascontiguousarray(frames)
    if frames.dtype != np.uint8:
        frames = _f32(frames)
    B, H, W, ch = frames.shape
    assert ch == 3, frames.shape
    k = {"detector": 0, "reid": 1}[layout]
    Hu, Wu = out_hw
    out, hi, lo = _plane_outputs((B, Hu, Wu, 16 if k == 0 else 64), split)
    _lib.check(lib.b2_op_stem_pack(device, _lib.ptr(frames), int(frames.dtype == np.uint8), B, H, W, k, Hu, Wu,
                                   int(split), _lib.ptr(out), _lib.ptr(hi), _lib.ptr(lo)),
               "b2_op_stem_pack")
    return out, hi, lo


def op_distance_operand(x, ld=None, normalize=False, eps=0.0, device=0):
    """The distance GEMMs' operand conversion through the C ABI -- used by the kernel tests: x [rows, D] fp32 to planes
    [rows, ld] (ld default D), normalised rows x / max(|x|, eps) or x itself.  Returns (hi, lo, sqnorm, range_flag) with
    raw uint16 planes; sqnorm and range_flag are None for normalised rows."""
    lib = _lib.load()
    x = _f32(x)
    rows, D = x.shape
    ld = D if ld is None else int(ld)
    hi, lo = np.empty((rows, ld), np.uint16), np.empty((rows, ld), np.uint16)
    sq = None if normalize else np.empty(rows, np.float32)
    flag = np.zeros(1, np.uint32)
    _lib.check(lib.b2_op_distance_operand(device, _lib.ptr(x), rows, D, ld, int(bool(normalize)), float(eps),
                                          _lib.ptr(hi), _lib.ptr(lo), _lib.ptr(sq), _lib.ptr(flag)),
               "b2_op_distance_operand")
    return hi, lo, sq, None if normalize else int(flag[0])


def op_distance_epilogue(kind, dots, cols=None, na2=None, nb2=None, seg_a=None, seg_b=None, gate=None, fill=0.0,
                         device=0):
    """One distance epilogue through the C ABI -- used by the kernel tests: dots [rows, ld] fp32 with the first `cols`
    columns live (default ld).  kind "cosine" / "euclidean": the [rows, cols] matrix; "cosine_segmin": the [T, cols]
    per-segment minimum over seg_a [T + 1]; "pair_segmin": the [N, M] block minimum over seg_a [N + 1] and seg_b [M + 1],
    gate [N, M] (uint8, None = all pairs), fill."""
    lib = _lib.load()
    k = {"cosine": 0, "euclidean": 1, "cosine_segmin": 2, "pair_segmin": 3}[kind]
    dots = _f32(dots)
    rows, ld = dots.shape
    cols = ld if cols is None else int(cols)
    sa = None if seg_a is None else np.ascontiguousarray(seg_a, np.int32)
    sb = None if seg_b is None else np.ascontiguousarray(seg_b, np.int32)
    na, nb = (0 if sa is None else len(sa) - 1), (0 if sb is None else len(sb) - 1)
    g = None if gate is None else np.ascontiguousarray(gate, np.uint8)
    na2, nb2 = _f32(na2), _f32(nb2)
    shape = (rows, cols) if k < 2 else (na, cols) if k == 2 else (na, nb)
    if g is not None:
        assert g.shape == shape, (g.shape, shape)
    out = np.empty(shape, np.float32)
    _lib.check(lib.b2_op_distance_epilogue(device, k, _lib.ptr(dots), rows, cols, ld, _lib.ptr(na2), _lib.ptr(nb2),
                                           _lib.ptr(sa), na, _lib.ptr(sb), nb, _lib.ptr(g),
                                           float(fill), _lib.ptr(out)),
               "b2_op_distance_epilogue")
    return out


def op_att_pool(x, split=True, device=0) -> np.ndarray:
    """The attention box head's pool (use_att_frcnn_head, models.py:1064-1089) through the C ABI -- used by the kernel
    tests: x [M, 49, C] ROIAlign rows (bin-major, as the engine stores them), converted to the engine's planes.  Returns
    [M, C] float32, the sum over the 49 bins read back from its planes; a row with a non-finite input is all NaN."""
    lib = _lib.load()
    x = np.ascontiguousarray(x, dtype=np.float32)
    M, nb, C = x.shape
    assert nb == 49, x.shape
    out = np.empty((M, C), dtype=np.float32)
    _lib.check(lib.b2_op_att_pool(device, _lib.ptr(x), M, C, int(split), _lib.ptr(out)), "b2_op_att_pool")
    return out


def op_so_attend(h, boxes, ref, ref_boxes, weights, split=True, device=0) -> np.ndarray:
    """person_object_relation (nn.py:194-270) through the C ABI as the engine runs it -- used by the kernel tests: query
    rows h [K, D] with boxes [K, 4], person rows ref [R, D] with boxes [R, 4]; `weights` maps geo_emb/W, geo_emb/b,
    geo_conv/W, geo_conv/b, query_linear/W, key_linear/W, output_linear/W (any prefix) to arrays.  Returns [K, D] float32
    = h + the module's output, read back from its planes."""
    lib = _lib.load()
    h, boxes, ref, ref_boxes = (np.ascontiguousarray(a, dtype=np.float32) for a in (h, boxes, ref, ref_boxes))
    K, D = h.shape
    R = ref.shape[0]
    names = ("geo_emb/W", "geo_emb/b", "geo_conv/W", "geo_conv/b", "query_linear/W", "key_linear/W", "output_linear/W")
    ws = [np.ascontiguousarray(next(v for k, v in weights.items() if k.endswith(n)), dtype=np.float32) for n in names]
    out = np.empty((K, D), dtype=np.float32)
    _lib.check(lib.b2_op_so_attend(device, _lib.ptr(h), _lib.ptr(boxes), K, _lib.ptr(ref), _lib.ptr(ref_boxes), R,
                                   *[_lib.ptr(w) for w in ws], D, int(split), _lib.ptr(out)), "b2_op_so_attend")
    return out


def get_new_hw(h, w, size, max_size):
    """nn.py:1548-1560: (neww, newh) of resizeImage for an h x w frame."""
    scale = size * 1.0 / min(h, w)
    if h < w:
        newh, neww = size, scale * w
    else:
        newh, neww = scale * h, size
    if max(newh, neww) > max_size:
        scale = max_size * 1.0 / max(newh, neww)
        newh = newh * scale
        neww = neww * scale
    return int(neww + 0.5), int(newh + 0.5)


def resize_frames(frames_u8, new_w, new_h, device=0):
    """The ingest resize alone: uint8 [n,h,w,3] -> float32 [n,new_h,new_w,3] on the GPU (b2_resize_frames)."""
    frames_u8 = np.ascontiguousarray(frames_u8, dtype=np.uint8)
    n, h, w, _ = frames_u8.shape
    out = np.empty((n, int(new_h), int(new_w), 3), dtype=np.float32)
    _lib.check(_lib.load().b2_resize_frames(int(device), _lib.ptr(frames_u8), n, h, w, int(new_h), int(new_w), _lib.ptr(out)),
               "b2_resize_frames")
    return out
