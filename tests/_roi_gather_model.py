"""ctypes access to tests/roi_gather_model.c, the host restatement of the RoIAlign backward gather (compiled on first use into a private
temporary directory, so the tree may be read-only)."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "roi_gather_model.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="mdt_roi_gather_model_"), "libroi_gather_model.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-o", out, SRC, "-lm"])
        _lib = ctypes.CDLL(out)
        _lib.model_sample_coord.restype = ctypes.c_float
        _lib.model_sample_coord.argtypes = [ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def taps(lo, hi, crop, size):
    """(lo[crop], hi[crop], lerp[crop]) of one axis, as the kernels compute them"""
    tlo, thi, lerp = np.empty(crop, np.int32), np.empty(crop, np.int32), np.empty(crop, np.float32)
    lib().model_taps(ctypes.c_float(lo), ctypes.c_float(hi), crop, size, _p(tlo), _p(thi), _p(lerp))
    return tlo, thi, lerp


def footprint(lo, hi, crop, size):
    """the gather kernel's footprint of one axis: (min, max) over the taps of the first and the last bin"""
    a, b = ctypes.c_int(), ctypes.c_int()
    lib().model_footprint(ctypes.c_float(lo), ctypes.c_float(hi), crop, size, ctypes.byref(a), ctypes.byref(b))
    return a.value, b.value


def gather_backward(grads, gs, boxes, box_ind, image, is5, shape, crop, zero_init, roi_level=None, level=0, nlevels=1):
    """the specified backward into `image` (flat float32 numpy buffer, modified in place; element strides is5 of the logical image shape
    [B, C, *spatial]).  grads: flat float32 buffer with element strides gs (5 entries, 2D: z stride 0) of a logical [n, C, *crop]; returns image"""
    dim = len(crop)
    boxes = np.ascontiguousarray(boxes, np.float32)
    box_ind = np.ascontiguousarray(box_ind, np.int32)
    grads = np.ascontiguousarray(grads, np.float32)
    assert image.dtype == np.float32 and image.flags.c_contiguous
    lv = None if roi_level is None else np.ascontiguousarray(roi_level, np.int32)
    B, C, H, W = (int(v) for v in shape[:4])
    Z = int(shape[4]) if dim == 3 else 1
    n = boxes.shape[0]
    gs = np.array(list(gs) + [0] * (5 - len(gs)), np.int64)
    is_ = np.array(list(is5) + [0] * (5 - len(is5)), np.int64)
    cz = crop[2] if dim == 3 else 1
    lib().model_gather_backward(dim, _p(grads), _p(gs), _p(boxes), _p(box_ind), None if lv is None else _p(lv), level, nlevels, n, B, H, W, Z,
                                crop[0], crop[1], cz, C, _p(image), _p(is_), int(zero_init))
    return image
