"""Test-only host build + ctypes driver of the emulation of programs with RESIZE ops (tests/emu/resize_emu.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from sod100k_b200 import ir

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..", "..")
LIB = os.path.join(HERE, "libcsnet_resize_emu.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(HERE, "resize_emu.cpp")
        deps = [src, os.path.join(HERE, "emu.cpp"), os.path.join(ROOT, "sod100k_b200", "csrc", "generic_ops.cuh"),
                os.path.join(ROOT, "sod100k_b200", "csrc", "resize.cuh"), os.path.join(ROOT, "sod100k_b200", "csrc", "image_io.cuh"),
                os.path.join(ROOT, "include", "csnet_b200.h")]
        if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
            subprocess.run(["g++", "-O2", "-fopenmp", "-shared", "-fPIC", "-std=c++17", "-o", LIB, src], check=True)
        _lib = C.CDLL(LIB)
        _lib.csnet_emu_run_resize.restype = C.c_int
    return _lib


def run_ext(prog: ir.Program, ext_arrays, N: int, taps=()):
    """tests/emu.run_ext for programs that may hold RESIZE ops: `ext_arrays[i]` (float32 numpy arrays, outputs written in place) is
    bound to external i; returns {tap name: array} (compile with reuse_arena=False when taps are wanted)."""
    arena = np.zeros(prog.arena_bytes_per_image * N + 256, np.uint8)
    ext = (C.c_void_p * len(ext_arrays))(*[a.ctypes.data for a in ext_arrays])
    blob = np.ascontiguousarray(prog.blob, np.float32)
    rc = lib().csnet_emu_run_resize(prog.tensor_array(), len(prog.tensors), prog.op_array(), len(prog.ops),
                                    blob.ctypes.data_as(C.POINTER(C.c_float)), N, ext, arena.ctypes.data_as(C.c_char_p))
    if rc != 0:
        raise RuntimeError(f"emu failed rc={rc}")
    got = {}
    for name in taps:
        t = prog.tensors[prog.taps[name]]
        off = N * t.arena_offset
        got[name] = arena[off:off + N * t.bytes_per_image].view(np.float32).reshape(N, t.C, t.H, t.W).copy()
    return got
