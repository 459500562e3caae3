"""Test-only host build + ctypes driver of the resize emulation (tests/emu/image_io_emu.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libcsnet_image_io_emu.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(HERE, "image_io_emu.cpp")
        deps = [src, os.path.join(HERE, "..", "..", "sod100k_b200", "csrc", "image_io.cuh"),
                os.path.join(HERE, "..", "..", "include", "csnet_b200.h")]
        if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
            subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-o", LIB, src], check=True)
        _lib = C.CDLL(LIB)
        _lib.csnet_emu_resize_in.restype = None
        _lib.csnet_emu_resize_out.restype = None
        _lib.csnet_emu_sigmoid.restype = None
        _lib.csnet_emu_sigmoid.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
    return _lib


def resize_in(img: np.ndarray, size, mean, std) -> np.ndarray:
    """uint8 [h, w, 3] -> fp32 [3, H, W] network input, as resize_in_u8_kernel computes it."""
    img = np.ascontiguousarray(img, np.uint8)
    H, W = size
    out = np.empty((3, H, W), np.float32)
    m, s = np.asarray(mean, np.float32), np.asarray(std, np.float32)
    lib().csnet_emu_resize_in(img.ctypes.data_as(C.c_void_p), C.c_int(img.shape[0]), C.c_int(img.shape[1]), C.c_int(H), C.c_int(W),
                              m.ctypes.data_as(C.c_void_p), s.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
    return out


def resize_out(logits: np.ndarray, shape) -> np.ndarray:
    """fp32 logits [H, W] -> uint8 map of `shape` (h, w), as resize_out_u8_kernel computes it."""
    z = np.ascontiguousarray(logits, np.float32)
    h, w = shape
    out = np.empty((h, w), np.uint8)
    lib().csnet_emu_resize_out(z.ctypes.data_as(C.c_void_p), C.c_int(z.shape[0]), C.c_int(z.shape[1]), C.c_int(h), C.c_int(w),
                               out.ctypes.data_as(C.c_void_p))
    return out


def sigmoid(logits: np.ndarray) -> np.ndarray:
    """The kernels' fp32 sigmoid, elementwise."""
    z = np.ascontiguousarray(logits, np.float32)
    s = np.empty_like(z)
    lib().csnet_emu_sigmoid(z.ctypes.data, z.size, s.ctypes.data)
    return s
