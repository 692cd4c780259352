"""Mask paste and COCO RLE on the GPU (csrc/mask_rle.cu): what the drivers do with final_masks (obj_detect_tracking.py:
716-739, obj_detect_imgs.py:501-527), bit-exact with nn.fill_full_mask (cv2.resize, OpenCV 4.13 default dispatch) and
pycocotools.mask.encode + counts.decode("ascii").

    fill_full_mask(box, mask, im_shape)       drop-in for nn.fill_full_mask: [H, W] uint8
    fill_full_masks(boxes, masks, im_shape)   [R, H, W] uint8
    encode_masks(boxes, masks, im_shape)      [{"size": [H, W], "counts": str}] per box, the drivers' `rle`

`boxes` are float32 [R, 4], already divided by the resize scale (float32 / a Python float stays float32 in NumPy, as in
the drivers); `masks` float32 [R, 28, 28], a NumPy array or a CUDA torch tensor.  A box whose patch NumPy could not paste
(a corner int(box[:2] + 0.5) below 0, or a patch the frame's edge cuts short, which fill_full_mask refuses too) raises
ValueError before any device work."""
from __future__ import annotations

import ctypes
from ctypes import c_void_p

import numpy as np

from . import _lib

MASK_REFUSED = -2   # kMaskRefused: an input refused on the host


def _check(rc: int, what: str):
    if rc == MASK_REFUSED:
        msg = _lib.load().b2_last_error()
        raise ValueError(msg.decode() if msg else what)
    _lib.check(rc, what)


def _boxes(boxes) -> np.ndarray:
    if hasattr(boxes, "detach"):                     # torch tensor
        boxes = boxes.detach().cpu().numpy()
    boxes = np.asarray(boxes)
    if boxes.dtype != np.float32:
        # int() of box + 0.5 happens in the boxes' own precision: a float64 box may truncate differently
        raise TypeError("boxes must be float32 (the drivers' final_boxes / scale), got %s" % boxes.dtype)
    return np.ascontiguousarray(boxes.reshape(-1, 4))


def _im_shape(im_shape):
    if len(im_shape) != 2:
        raise ValueError("im_shape must be (H, W), got %r" % (im_shape,))
    return int(im_shape[0]), int(im_shape[1])


class MaskEncoder:
    """One b2_masks encoder: a device's grow-only workspaces and stream, reused across calls."""

    def __init__(self, device: int = 0):
        self.lib = _lib.load()
        self.device = int(device)
        self._h = c_void_p(0)
        _lib.check(self.lib.b2_masks_create(ctypes.byref(self._h), self.device), "b2_masks_create")
        self._bytes = np.empty(1 << 16, np.uint8)    # grow-only host buffer for the strings

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self.lib.b2_masks_destroy(self._h)
            self._h = c_void_p(0)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _masks(self, masks, n: int):
        """(pointer, on_device, keep-alive) of [n, 28, 28] float32 masks; the shape check is the library's."""
        if hasattr(masks, "is_cuda") and masks.is_cuda:
            import torch
            if masks.dtype != torch.float32:
                raise TypeError("masks must be float32, got %s" % masks.dtype)
            if masks.device.index != self.device:
                raise ValueError("masks are on cuda:%d, the encoder on cuda:%d" % (masks.device.index, self.device))
            m = masks.contiguous()
            torch.cuda.current_stream(m.device).synchronize()   # the encoder reads them on its own stream
            return _lib.ptr(m), 1, m, tuple(m.shape)
        if hasattr(masks, "detach"):
            masks = masks.detach().numpy()
        m = np.ascontiguousarray(masks, dtype=np.float32)
        return _lib.ptr(m), 0, m, m.shape

    @staticmethod
    def _mask_hw(shape, n: int):
        if len(shape) != 3 or shape[0] != n:
            raise ValueError("masks must be [R, 28, 28] with one per box, got %s for %d boxes" % (tuple(shape), n))
        return int(shape[1]), int(shape[2])

    def fill_full_masks(self, boxes, masks, im_shape) -> np.ndarray:
        boxes = _boxes(boxes)
        n = len(boxes)
        H, W = _im_shape(im_shape)
        p, on_dev, keep, shape = self._masks(masks, n)
        mh, mw = self._mask_hw(shape, n)
        out = np.empty((n, H, W), np.uint8)
        _check(self.lib.b2_masks_paste(self._h, _lib.ptr(boxes), p, on_dev, n, mh, mw, H, W, _lib.ptr(out), out.nbytes),
               "b2_masks_paste")
        del keep
        return out

    def _strings(self, n: int, H: int, W: int, call) -> list:
        offs = np.empty(n + 1, np.int64)
        _check(call(_lib.ptr(offs), _lib.ptr(self._bytes), self._bytes.nbytes), "mask RLE")
        total = int(offs[-1])
        if total > self._bytes.nbytes:
            self._bytes = np.empty(max(total, 2 * self._bytes.nbytes), np.uint8)
            _lib.check(self.lib.b2_masks_fetch(self._h, _lib.ptr(self._bytes), self._bytes.nbytes), "b2_masks_fetch")
        raw = self._bytes[:total].tobytes()
        return [{"size": [H, W], "counts": raw[offs[i]:offs[i + 1]].decode("ascii")} for i in range(n)]

    def encode(self, boxes, masks, im_shape) -> list:
        boxes = _boxes(boxes)
        n = len(boxes)
        H, W = _im_shape(im_shape)
        p, on_dev, keep, shape = self._masks(masks, n)
        mh, mw = self._mask_hw(shape, n)
        out = self._strings(n, H, W, lambda offs, b, cap: self.lib.b2_masks_encode(self._h, _lib.ptr(boxes), p, on_dev, n,
                                                                                    mh, mw, H, W, offs, b, cap))
        del keep
        return out

    def encode_engine(self, ctx, image: int, boxes, im_shape) -> list:
        """The RLE of final_masks rows of `image` of an engine context's last pass (Detector.encode_masks)."""
        boxes = _boxes(boxes)
        n = len(boxes)
        H, W = _im_shape(im_shape)
        return self._strings(n, H, W, lambda offs, b, cap: self.lib.b2_encode_masks(ctx, self._h, int(image),
                                                                                     _lib.ptr(boxes), n, H, W, offs, b,
                                                                                     cap))


_encoders = {}


def _encoder(masks) -> MaskEncoder:
    dev = masks.device.index if (hasattr(masks, "is_cuda") and masks.is_cuda) else 0
    if dev not in _encoders:
        _encoders[dev] = MaskEncoder(dev)
    return _encoders[dev]


def fill_full_masks(boxes, masks, im_shape) -> np.ndarray:
    """[R, H, W] uint8: fill_full_mask of every (box, mask) pair."""
    return _encoder(masks).fill_full_masks(boxes, masks, im_shape)


def fill_full_mask(box, mask, im_shape) -> np.ndarray:
    """Drop-in for nn.fill_full_mask (nn.py:1565-1584): box float32 [4], mask float32 [28, 28] -> [H, W] uint8."""
    return fill_full_masks(_boxes(box), mask[None], im_shape)[0]


def encode_masks(boxes, masks, im_shape) -> list:
    """The drivers' RLE dicts ({"size": [H, W], "counts": str}) of fill_full_mask of every (box, mask) pair."""
    return _encoder(masks).encode(boxes, masks, im_shape)
