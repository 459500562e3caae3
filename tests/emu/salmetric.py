"""Test-only host build + ctypes driver of the SalMetric counting emulation (tests/emu/salmetric_emu.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libcsnet_salmetric_emu.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(HERE, "salmetric_emu.cpp")
        deps = [src, os.path.join(HERE, "..", "..", "sod100k_b200", "csrc", "image_io.cuh"),
                os.path.join(HERE, "..", "..", "include", "csnet_b200.h")]
        if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
            subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-o", LIB, src], check=True)
        _lib = C.CDLL(LIB)
        _lib.csnet_emu_salmetric_image.restype = None
        _lib.csnet_emu_salmetric_image.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                                   C.c_void_p, C.c_void_p]
    return _lib


def salmetric_image(logits: np.ndarray, gt: np.ndarray):
    """fp32 logits [H, W] and uint8 GT [h, w] -> (hist_all [256], hist_pos [256], abs_sum, uint8 map [h, w]) as
    salmetric_images_u8_kernel counts them."""
    z = np.ascontiguousarray(logits, np.float32)
    g = np.ascontiguousarray(gt, np.uint8)
    ha, hp = np.empty(256, np.uint32), np.empty(256, np.uint32)
    ad = np.empty(1, np.uint64)
    m = np.empty(g.shape, np.uint8)
    lib().csnet_emu_salmetric_image(z.ctypes.data, z.shape[0], z.shape[1], g.ctypes.data, g.shape[0], g.shape[1], ha.ctypes.data,
                                    hp.ctypes.data, ad.ctypes.data, m.ctypes.data)
    return ha, hp, int(ad[0]), m
