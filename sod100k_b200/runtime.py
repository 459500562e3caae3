"""ctypes binding of libcsnet_b200.so (include/csnet_b200.h).  PyTorch is only plumbing here: it owns the
device buffers and the stream; every kernel that runs is ours.  There is no CPU or library fallback — a
missing library or a missing GPU raises."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

from . import ir

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcsnet_b200.so")
ABI_VERSION = 14
PARAM_EPOCH = 0      # bumped by in-place parameter updates that bypass torch's version counters (FusedAdam)
_lib = None

# every symbol include/csnet_b200.h declares (tests check the library exports exactly these)
SYMBOLS = ("csnet_abi_version", "csnet_last_error", "csnet_device_count", "csnet_plan_create",
           "csnet_plan_set_blob", "csnet_plan_run", "csnet_plan_profile", "csnet_plan_tensor_ptr", "csnet_plan_read_tensor", "csnet_plan_op_kernel", "csnet_plan_launches",
           "csnet_plan_arena_bytes", "csnet_plan_destroy", "csnet_plan_run_host", "csnet_plan_run_host_u8",
           "csnet_resize_u8_to_input", "csnet_resize_logits_to_u8", "csnet_salmetric_images_u8", "csnet_plan_run_host_images_u8",
           "csnet_train_batch_u8", "csnet_val_mae_u8", "csnet_train_last_error", "csnet_train_bn_stats", "csnet_train_bn_prelu_fwd", "csnet_train_bn_prelu_bwd",
           "csnet_train_dw_conv", "csnet_train_dw_wgrad", "csnet_train_dw_bwd", "csnet_train_mix_fwd", "csnet_train_mix_dgrad",
           "csnet_train_mix_wgrad", "csnet_train_pool_fwd", "csnet_train_pool_bwd", "csnet_slim_gather", "csnet_train_bce", "csnet_train_adam", "csnet_salmetric_hist",
           "csnet_train_conv_plan", "csnet_train_conv_fwd", "csnet_train_conv_dgrad", "csnet_train_conv_wgrad", "csnet_train_bias_grad",
           "csnet_train_gn_stats", "csnet_train_gn_prelu_fwd", "csnet_train_gn_prelu_bwd", "csnet_train_resize_fwd", "csnet_train_resize_bwd",
           "csnet_csf_input_u8", "csnet_csf_maps_u8", "csnet_salmetric_csf_u8", "csnet_csf_train_batch_u8", "csnet_train_bce_sum",
           "csnet_train_bn_stats_bf16", "csnet_train_bn_prelu_fwd_bf16", "csnet_train_bn_prelu_bwd_bf16", "csnet_train_dw_conv_bf16",
           "csnet_train_dw_wgrad_bf16", "csnet_train_dw_bwd_bf16", "csnet_train_mix_fwd_bf16", "csnet_train_mix_dgrad_bf16",
           "csnet_train_mix_wgrad_bf16", "csnet_train_pool_fwd_bf16", "csnet_train_pool_bwd_bf16", "csnet_train_cast_bf16",
           "csnet_train_conv_plan_bf16", "csnet_train_conv_fwd_bf16", "csnet_train_conv_dgrad_bf16", "csnet_train_conv_wgrad_bf16",
           "csnet_train_gn_stats_bf16", "csnet_train_gn_prelu_fwd_bf16", "csnet_train_gn_prelu_bwd_bf16", "csnet_train_resize_fwd_bf16",
           "csnet_train_resize_bwd_bf16", "csnet_train_bn_sync_partial", "csnet_train_bn_sync_merge", "csnet_train_bn_sync_bwd_reduce",
           "csnet_train_bn_sync_bwd_apply")


class EngineError(RuntimeError):
    pass


class ImageGeom(C.Structure):
    """csnet_image_geom: image i of a ragged batch is uint8 [h][w][3] at byte src_off of the packed input; its map is uint8 [h][w]
    at byte dst_off of the packed output."""
    _fields_ = [("src_off", C.c_int64), ("dst_off", C.c_int64), ("h", C.c_int32), ("w", C.c_int32)]


assert C.sizeof(ImageGeom) == 24
GEOM_DTYPE = np.dtype(ImageGeom)


class TrainSample(C.Structure):
    """csnet_train_sample: crop image `image` of the packed set to [y0:y0+h, x0:x0+w], then flip it (0 none, 1 'lr', 2 'ud')."""
    _fields_ = [("image", C.c_int32), ("y0", C.c_int32), ("x0", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("flip", C.c_int32)]


assert C.sizeof(TrainSample) == 24
SAMPLE_DTYPE = np.dtype(TrainSample)


def image_geometry(sizes) -> np.ndarray:
    """Geometry (GEOM_DTYPE [N]) of images of the given (h, w) sizes packed back to back in order, input and output alike."""
    hw = np.array([(int(h), int(w)) for h, w in sizes], np.int64).reshape(-1, 2)
    n = hw[:, 0] * hw[:, 1]
    g = np.zeros(len(n), GEOM_DTYPE)
    g["dst_off"][1:] = np.cumsum(n)[:-1]
    g["src_off"] = 3 * g["dst_off"]
    g["h"], g["w"] = hw[:, 0], hw[:, 1]
    return g


def load_library(path: Optional[str] = None):
    """dlopen the engine.  Raises EngineError (never falls back) if it is missing or has the wrong ABI."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise EngineError(f"{path} not found — build it with `python -m sod100k_b200.build` "
                          "(__graft_entry__.build()); there is no CPU fallback")
    lib = C.CDLL(path)
    lib.csnet_abi_version.restype = C.c_int
    lib.csnet_last_error.restype = C.c_char_p
    lib.csnet_device_count.restype = C.c_int
    lib.csnet_plan_create.restype = C.c_int
    lib.csnet_plan_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(ir.TensorDesc), C.c_int32,
                                      C.POINTER(ir.OpDesc), C.c_int32, C.c_int64, C.c_int32, C.c_int32]
    lib.csnet_plan_set_blob.restype = C.c_int
    lib.csnet_plan_set_blob.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    lib.csnet_plan_run.restype = C.c_int
    lib.csnet_plan_run.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.c_int32, C.c_void_p]
    lib.csnet_plan_profile.restype = C.c_int
    lib.csnet_plan_profile.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.c_int32, C.c_void_p,
                                       C.POINTER(C.c_float), C.c_int32]
    lib.csnet_plan_tensor_ptr.restype = C.c_void_p
    lib.csnet_plan_tensor_ptr.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    lib.csnet_plan_read_tensor.restype = C.c_int
    lib.csnet_plan_read_tensor.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    lib.csnet_plan_op_kernel.restype = C.c_char_p
    lib.csnet_plan_op_kernel.argtypes = [C.c_void_p, C.c_int32]
    lib.csnet_plan_launches.restype = C.c_int32
    lib.csnet_plan_launches.argtypes = [C.c_void_p]
    lib.csnet_plan_arena_bytes.restype = C.c_int64
    lib.csnet_plan_arena_bytes.argtypes = [C.c_void_p]
    lib.csnet_plan_destroy.restype = None
    lib.csnet_plan_destroy.argtypes = [C.c_void_p]
    lib.csnet_plan_run_host.restype = C.c_int
    lib.csnet_plan_run_host.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.csnet_plan_run_host_u8.restype = C.c_int
    lib.csnet_plan_run_host_u8.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_void_p]
    lib.csnet_resize_u8_to_input.restype = C.c_int
    lib.csnet_resize_u8_to_input.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_float),
                                             C.POINTER(C.c_float), C.c_void_p, C.c_void_p]
    lib.csnet_resize_logits_to_u8.restype = C.c_int
    lib.csnet_resize_logits_to_u8.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.csnet_salmetric_images_u8.restype = C.c_int
    lib.csnet_salmetric_images_u8.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p]
    lib.csnet_plan_run_host_images_u8.restype = C.c_int
    lib.csnet_plan_run_host_images_u8.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                                  C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_void_p]
    lib.csnet_train_batch_u8.restype = C.c_int
    lib.csnet_train_batch_u8.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                         C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.csnet_val_mae_u8.restype = C.c_int
    lib.csnet_val_mae_u8.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.csnet_csf_input_u8.restype = C.c_int
    lib.csnet_csf_input_u8.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_double),
                                       C.POINTER(C.c_double), C.c_void_p, C.c_void_p]
    lib.csnet_csf_train_batch_u8.restype = C.c_int
    lib.csnet_csf_train_batch_u8.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                             C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.csnet_train_bce_sum.restype = C.c_int
    lib.csnet_train_bce_sum.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]
    lib.csnet_csf_maps_u8.restype = C.c_int
    lib.csnet_csf_maps_u8.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.csnet_salmetric_csf_u8.restype = C.c_int
    lib.csnet_salmetric_csf_u8.argtypes = lib.csnet_salmetric_images_u8.argtypes
    lib.csnet_slim_gather.restype = C.c_int
    lib.csnet_slim_gather.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
    lib.csnet_train_last_error.restype = C.c_char_p
    if lib.csnet_abi_version() != ABI_VERSION:
        raise EngineError(f"{path}: ABI {lib.csnet_abi_version()} != expected {ABI_VERSION}; rebuild")
    if path == LIB_PATH:
        _lib = lib
    return lib


def _check(lib, rc: int, what: str):
    if rc != 0:
        raise EngineError(f"{what} failed ({rc}): {lib.csnet_last_error().decode()}")


def resize_u8_to_input(x_packed_ptr: int, geom_dev_ptr: int, N: int, H: int, W: int, mean, std, x_nchw_ptr: int, stream: int = 0):
    """Device to device: packed uint8 images (geometry on the device) -> fp32 [N,3,H,W] network input (csnet_resize_u8_to_input)."""
    lib = load_library()
    m, s_ = (C.c_float * 3)(*mean), (C.c_float * 3)(*std)
    _check(lib, lib.csnet_resize_u8_to_input(x_packed_ptr, geom_dev_ptr, int(N), int(H), int(W), m, s_, x_nchw_ptr, stream),
           "csnet_resize_u8_to_input")


def resize_logits_to_u8(logits_ptr: int, N: int, H: int, W: int, geom_dev_ptr: int, y_packed_ptr: int, stream: int = 0):
    """Device to device: fp32 logits [N,1,H,W] -> each image's uint8 map at its dst_off (csnet_resize_logits_to_u8)."""
    lib = load_library()
    _check(lib, lib.csnet_resize_logits_to_u8(logits_ptr, int(N), int(H), int(W), geom_dev_ptr, y_packed_ptr, stream),
           "csnet_resize_logits_to_u8")


def salmetric_images_u8(logits_ptr: int, N: int, H: int, W: int, geom_dev_ptr: int, m_packed_ptr: int, y_packed_ptr: int,
                        hist_all_ptr: int, hist_pos_ptr: int, abs_sum_ptr: int, stream: int = 0):
    """Device to device: fp32 logits [N,1,H,W] and each image's uint8 GT -> SalMetric counts of the maps resize_logits_to_u8 would
    write (uint32 [N,256] twice, uint64 [N]); the maps too when y_packed_ptr is non-zero (csnet_salmetric_images_u8)."""
    lib = load_library()
    _check(lib, lib.csnet_salmetric_images_u8(logits_ptr, int(N), int(H), int(W), geom_dev_ptr, m_packed_ptr, y_packed_ptr or None,
                                              hist_all_ptr, hist_pos_ptr, abs_sum_ptr, stream), "csnet_salmetric_images_u8")


def csf_input_u8(x_packed_ptr: int, geom_dev_ptr: int, N: int, H: int, W: int, mean, std, x_nchw_ptr: int, stream: int = 0):
    """Device to device: N packed uint8 images of size H x W -> fp32 [N,3,H,W] as CSF+Res2Net's load_image_test computes it, mean /
    std taken as doubles (csnet_csf_input_u8)."""
    lib = load_library()
    m, s_ = (C.c_double * 3)(*mean), (C.c_double * 3)(*std)
    _check(lib, lib.csnet_csf_input_u8(x_packed_ptr, geom_dev_ptr, int(N), int(H), int(W), m, s_, x_nchw_ptr, stream), "csnet_csf_input_u8")


def csf_train_batch_u8(x_packed_ptr: int, m_packed_ptr: int, geom_dev_ptr: int, samples_dev_ptr: int, N: int, H: int, W: int, mean,
                       std, x_nchw_ptr: int, target_ptr: int, stream: int = 0):
    """Device to device: N packed uint8 images and masks of size H x W, each flipped along W when its sample's flip is 1 -> fp32 input
    [N,3,H,W] and target [N,1,H,W] as CSF+Res2Net's ImageDataTrain computes them, mean / std taken as doubles
    (csnet_csf_train_batch_u8)."""
    lib = load_library()
    m, s_ = (C.c_double * 3)(*mean), (C.c_double * 3)(*std)
    _check(lib, lib.csnet_csf_train_batch_u8(x_packed_ptr, m_packed_ptr, geom_dev_ptr, samples_dev_ptr, int(N), int(H), int(W), m, s_,
                                             x_nchw_ptr, target_ptr, stream), "csnet_csf_train_batch_u8")


def train_bce_sum(logits_ptr: int, target_ptr: int, dlogits_ptr: int, loss_ptr: int, n: int, divisor: int, stream: int = 0):
    """Device to device: loss = BCE-with-logits summed over n elements / divisor, dlogits = (sigmoid(z) - t) * f32(1 / divisor)
    (csnet_train_bce_sum; dlogits_ptr may be 0)."""
    lib = load_library()
    rc = lib.csnet_train_bce_sum(logits_ptr, target_ptr, dlogits_ptr or None, loss_ptr, int(n), int(divisor), stream)
    if rc != 0:
        raise EngineError(f"csnet_train_bce_sum failed ({rc}): {lib.csnet_train_last_error().decode()}")


def csf_maps_u8(logits_ptr: int, N: int, H: int, W: int, geom_dev_ptr: int, y_packed_ptr: int, stream: int = 0):
    """Device to device: fp32 logits [N,1,H,W] at the images' own size -> each image's uint8 map at its dst_off, rounded as
    CSF+Res2Net's solver.test writes it (csnet_csf_maps_u8)."""
    lib = load_library()
    _check(lib, lib.csnet_csf_maps_u8(logits_ptr, int(N), int(H), int(W), geom_dev_ptr, y_packed_ptr, stream), "csnet_csf_maps_u8")


def salmetric_csf_u8(logits_ptr: int, N: int, H: int, W: int, geom_dev_ptr: int, m_packed_ptr: int, y_packed_ptr: int,
                     hist_all_ptr: int, hist_pos_ptr: int, abs_sum_ptr: int, stream: int = 0):
    """salmetric_images_u8 for the maps csf_maps_u8 writes (csnet_salmetric_csf_u8)."""
    lib = load_library()
    _check(lib, lib.csnet_salmetric_csf_u8(logits_ptr, int(N), int(H), int(W), geom_dev_ptr, m_packed_ptr, y_packed_ptr or None,
                                           hist_all_ptr, hist_pos_ptr, abs_sum_ptr, stream), "csnet_salmetric_csf_u8")


def train_batch_u8(x_packed_ptr: int, m_packed_ptr: int, geom_dev_ptr: int, samples_dev_ptr: int, N: int, H: int, W: int, mean, std,
                   x_nchw_ptr: int, target_ptr: int, stream: int = 0):
    """Device to device: packed uint8 images and masks, a crop / flip per sample -> fp32 input [N,3,H,W] and target [N,1,H,W]
    (csnet_train_batch_u8)."""
    lib = load_library()
    m, s_ = (C.c_float * 3)(*mean), (C.c_float * 3)(*std)
    _check(lib, lib.csnet_train_batch_u8(x_packed_ptr, m_packed_ptr, geom_dev_ptr, samples_dev_ptr, int(N), int(H), int(W), m, s_,
                                         x_nchw_ptr, target_ptr, stream), "csnet_train_batch_u8")


def val_mae_u8(logits_ptr: int, N: int, H: int, W: int, m_packed_ptr: int, geom_dev_ptr: int, mae_ptr: int, stream: int = 0):
    """Device to device: fp32 logits [N,1,H,W] and each image's uint8 GT -> float64 MAE [N] (csnet_val_mae_u8)."""
    lib = load_library()
    _check(lib, lib.csnet_val_mae_u8(logits_ptr, int(N), int(H), int(W), m_packed_ptr, geom_dev_ptr, mae_ptr, stream), "csnet_val_mae_u8")


class Plan:
    """One compiled program resident on one GPU."""

    def __init__(self, prog: ir.Program, max_batch: int, device: int = 0):
        self.lib = load_library()
        n = self.lib.csnet_device_count()
        if n <= 0:
            raise EngineError("no CUDA device visible: the CSNet engine runs on the GPU only "
                              f"({self.lib.csnet_last_error().decode()})")
        self.prog = prog
        self.max_batch = int(max_batch)
        self.device = int(device)
        self._h = C.c_void_p()
        self._tensors, self._ops = prog.tensor_array(), prog.op_array()
        _check(self.lib, self.lib.csnet_plan_create(C.byref(self._h), self._tensors, len(prog.tensors), self._ops,
                                                    len(prog.ops), int(prog.blob.size), self.max_batch, self.device),
               "csnet_plan_create")
        self.set_blob(prog.blob)

    def set_blob(self, blob: np.ndarray, stream: int = 0):
        blob = np.ascontiguousarray(blob, np.float32)
        _check(self.lib, self.lib.csnet_plan_set_blob(self._h, blob.ctypes.data, blob.size, stream), "csnet_plan_set_blob")

    def run(self, N: int, ext_ptrs, stream: int = 0):
        arr = (C.c_void_p * len(ext_ptrs))(*[int(p) for p in ext_ptrs])
        _check(self.lib, self.lib.csnet_plan_run(self._h, int(N), arr, len(ext_ptrs), stream), "csnet_plan_run")

    def profile(self, N: int, ext_ptrs, stream: int = 0):
        """Per-op device milliseconds of one run (CUDA events around every launch)."""
        arr = (C.c_void_p * len(ext_ptrs))(*[int(p) for p in ext_ptrs])
        ms = (C.c_float * len(self.prog.ops))()
        _check(self.lib, self.lib.csnet_plan_profile(self._h, int(N), arr, len(ext_ptrs), stream, ms, len(self.prog.ops)),
               "csnet_plan_profile")
        return list(ms)

    def run_host(self, N: int, x_host_ptr: int, y_host_ptr: int, stream: int = 0):
        _check(self.lib, self.lib.csnet_plan_run_host(self._h, int(N), x_host_ptr, y_host_ptr, stream), "csnet_plan_run_host")

    def run_host_u8(self, N: int, x_host_ptr: int, y_host_ptr: int, mean, std, stream: int = 0):
        m, s_ = (C.c_float * 3)(*mean), (C.c_float * 3)(*std)
        _check(self.lib, self.lib.csnet_plan_run_host_u8(self._h, int(N), x_host_ptr, y_host_ptr, m, s_, stream), "csnet_plan_run_host_u8")

    def run_host_images_u8(self, N: int, x_host_ptr: int, x_bytes: int, geom: np.ndarray, y_host_ptr: int, y_bytes: int, mean, std,
                           stream: int = 0):
        """Ragged uint8 images (host, packed, `geom`: GEOM_DTYPE [N] on the host) -> uint8 maps at each image's size, synchronised."""
        geom = np.ascontiguousarray(geom, GEOM_DTYPE)
        if geom.shape != (int(N),):
            raise ValueError(f"geometry for {geom.shape} images, batch of {N}")
        m, s_ = (C.c_float * 3)(*mean), (C.c_float * 3)(*std)
        _check(self.lib, self.lib.csnet_plan_run_host_images_u8(self._h, int(N), x_host_ptr, int(x_bytes), geom.ctypes.data, y_host_ptr,
                                                                int(y_bytes), m, s_, stream), "csnet_plan_run_host_images_u8")

    def tensor_ptr(self, tensor: int, N: int) -> int:
        return int(self.lib.csnet_plan_tensor_ptr(self._h, tensor, N) or 0)

    def op_kernel(self, i: int) -> str:
        """Kernel (family) that runs op i of this plan."""
        return (self.lib.csnet_plan_op_kernel(self._h, int(i)) or b"").decode()

    @property
    def launches(self) -> int:
        return int(self.lib.csnet_plan_launches(self._h))

    @property
    def arena_bytes(self) -> int:
        return int(self.lib.csnet_plan_arena_bytes(self._h))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self.lib.csnet_plan_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- torch plumbing ---------------------------------------------------------------------------
    def forward(self, x):
        """x: CUDA float32 [N,3,H,W] contiguous -> float32 logits [N,1,H,W] on the current stream."""
        import torch

        if not x.is_cuda:
            raise EngineError("input must be a CUDA tensor: the engine has no CPU path")
        if x.dtype != torch.float32:
            x = x.float()
        x = x.contiguous()
        t_in, t_out = self.prog.tensors[self.prog.input], self.prog.tensors[self.prog.output]
        if tuple(x.shape[1:]) != (t_in.C, t_in.H, t_in.W):
            raise EngineError(f"plan compiled for {(t_in.C, t_in.H, t_in.W)}, got {tuple(x.shape[1:])}")
        N = x.shape[0]
        y = torch.empty((N, t_out.C, t_out.H, t_out.W), dtype=torch.float32, device=x.device)
        self.run(N, [x.data_ptr(), y.data_ptr()], torch.cuda.current_stream(x.device).cuda_stream)
        return y

    def read_tensor(self, tensor: int, N: int):
        """Copy an arena tensor of the last run (batch N) into a float32 torch tensor (tests / taps)."""
        import torch

        t = self.prog.tensors[tensor]
        tdt = {ir.F32: torch.float32, ir.F16: torch.float16, ir.BF16: torch.bfloat16}[t.dtype]
        out = torch.empty((N, t.C, t.H, t.W), dtype=tdt, device=f"cuda:{self.device}")
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _check(self.lib, self.lib.csnet_plan_read_tensor(self._h, tensor, N, out.data_ptr(), stream), "csnet_plan_read_tensor")
        return out.float()
