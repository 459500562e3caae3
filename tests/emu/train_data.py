"""Test-only host build + ctypes driver of the training-data emulation (tests/emu/train_data_emu.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libcsnet_train_data_emu.so")
# nvcc contracts a * b + c into one fused multiply-add in the kernels; the emulation lets g++ contract the same expressions, so its
# float64 lerps round like the device's before the single rounding to fp32.
FLAGS = ["-O2", "-shared", "-fPIC", "-std=c++17", "-mfma", "-ffp-contract=fast"]
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(HERE, "train_data_emu.cpp")
        deps = [src, os.path.join(HERE, "..", "..", "sod100k_b200", "csrc", "image_io.cuh"),
                os.path.join(HERE, "..", "..", "include", "csnet_b200.h"), os.path.abspath(__file__)]
        if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
            subprocess.run(["g++", *FLAGS, "-o", LIB, src], check=True)
        _lib = C.CDLL(LIB)
        _lib.csnet_emu_train_sample.restype = None
        _lib.csnet_emu_train_sample.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int] * 8 + [C.c_void_p] * 4
        _lib.csnet_emu_val_mae.restype = C.c_double
        _lib.csnet_emu_val_mae.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
    return _lib


def train_sample(img: np.ndarray, mask: np.ndarray, params, size, mean, std):
    """One sample as train_batch_u8_kernel builds it: img uint8 [h, w, 3] (gray [h, w] repeated, as SalImages packs it), mask uint8
    [h, w], params (y0, x0, ch, cw, flip) -> (fp32 [3, H, W], fp32 [1, H, W])."""
    if img.ndim == 2:
        img = np.repeat(img[:, :, None], 3, 2)
    img, mask = np.ascontiguousarray(img, np.uint8), np.ascontiguousarray(mask, np.uint8)
    H, W = size
    x, t = np.empty((3, H, W), np.float32), np.empty((1, H, W), np.float32)
    m, s = np.asarray(mean, np.float32), np.asarray(std, np.float32)
    y0, x0, ch, cw, flip = (int(v) for v in params)
    lib().csnet_emu_train_sample(img.ctypes.data, mask.ctypes.data, img.shape[1], y0, x0, ch, cw, flip, H, W, m.ctypes.data,
                                 s.ctypes.data, x.ctypes.data, t.ctypes.data)
    return x, t


def val_mae(logits: np.ndarray, gt: np.ndarray) -> float:
    """One image's validation MAE as val_mae_u8_kernel computes it (up to the order of the float64 sum): logits fp32 [H, W],
    gt uint8 [h, w]."""
    z, g = np.ascontiguousarray(logits, np.float32), np.ascontiguousarray(gt, np.uint8)
    return lib().csnet_emu_val_mae(z.ctypes.data, z.shape[0], z.shape[1], g.ctypes.data, g.shape[0], g.shape[1])
