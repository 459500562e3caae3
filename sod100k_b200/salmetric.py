"""SalMetric (max-F / mean-F / MAE) with the per-pixel counting on the device — SURVEY.md §8 f1.

The reference evaluates by writing png files and shelling out to a C++ binary (CSNet/eval.py:59-69,
CSNet_training/SalMetric/src/sal_metric.cpp); it declares `do_evaluation_gpu` (sal_metric.hpp:40) but never implements it.
Here the O(pixels x 256 thresholds) part — for th in 0..255: |sal > th|, |sal > th and gt > 128| (:99-120) and the MAE sum
(:86-97) — is one kernel producing two 256-bin histograms per image (`csnet_salmetric_hist`); the 256-element suffix sums,
the per-image precision / recall, their average over images and F = 1.3 P R / (0.3 P + R) (:164-185) stay on the host.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import runtime

EPSILON = np.float32(1e-4)          # sal_metric.hpp:50-52
BETA = np.float32(0.3)

_bound = False


def _lib():
    global _bound
    lib = runtime.load_library()
    if not _bound:
        lib.csnet_train_last_error.restype = C.c_char_p
        lib.csnet_salmetric_hist.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _bound = True
    return lib


def image_scores(hist_all: np.ndarray, hist_pos: np.ndarray, abs_sum: np.ndarray, hw):
    """Per image, from the device counts (host arrays hist_all / hist_pos [n, 256], abs_sum [n] as csnet_salmetric_hist and
    csnet_salmetric_images_u8 produce them; hw the pixels per image, one number or [n]): precision and recall [n, 256] in float32
    (sal_metric.cpp:99-120) and the MAE [n] in float64 (:86-97)."""
    ha = np.asarray(hist_all).astype(np.int64)
    hp = np.asarray(hist_pos).astype(np.int64)
    # a = sal > th: pixels strictly above th = suffix sum from th + 1
    a_sum = (ha[:, ::-1].cumsum(1)[:, ::-1] - ha).astype(np.float32)
    ab = (hp[:, ::-1].cumsum(1)[:, ::-1] - hp).astype(np.float32)
    b_sum = hp.sum(1).astype(np.float32)[:, None]
    mae = np.asarray(abs_sum).astype(np.float64) / (255.0 * np.asarray(hw))
    return (ab + EPSILON) / (a_sum + EPSILON), (ab + EPSILON) / (b_sum + EPSILON), mae


class SalMetric:
    """Streaming evaluator: `update(prob, gt)` per batch (CUDA tensors), `compute()` at the end."""

    def __init__(self):
        self._prec = np.zeros(256, np.float64)
        self._rec = np.zeros(256, np.float64)
        self._mae = 0.0
        self._n = 0

    def update(self, prob: torch.Tensor, gt: torch.Tensor) -> None:
        """prob: float32 CUDA [N,1,H,W] or [N,H,W] saliency in [0,1] (sigmoid of the logits); gt: uint8 CUDA, same pixels."""
        if not (prob.is_cuda and gt.is_cuda):
            raise runtime.EngineError("SalMetric.update needs CUDA tensors (there is no CPU path)")
        if prob.dtype != torch.float32 or gt.dtype != torch.uint8:
            raise TypeError("prob must be float32 and gt uint8")
        n = prob.shape[0]
        p, g = prob.reshape(n, -1).contiguous(), gt.reshape(n, -1).contiguous()
        if p.shape != g.shape:
            raise ValueError(f"prob {tuple(prob.shape)} and gt {tuple(gt.shape)} cover different pixels")
        hw = p.shape[1]
        hist_all = torch.empty(n, 256, dtype=torch.int32, device=p.device)
        hist_pos = torch.empty(n, 256, dtype=torch.int32, device=p.device)
        abs_sum = torch.empty(n, dtype=torch.int64, device=p.device)
        lib = _lib()
        rc = lib.csnet_salmetric_hist(p.data_ptr(), g.data_ptr(), n, hw, hist_all.data_ptr(), hist_pos.data_ptr(), abs_sum.data_ptr(),
                                      torch.cuda.current_stream(p.device).cuda_stream)
        if rc != 0:
            raise runtime.EngineError(f"csnet_salmetric_hist failed ({rc}): {lib.csnet_train_last_error().decode()}")
        prec, rec, mae = image_scores(hist_all.cpu().numpy(), hist_pos.cpu().numpy(), abs_sum.cpu().numpy(), hw)
        self._prec += prec.sum(0)
        self._rec += rec.sum(0)
        self._mae += float(mae.sum())
        self._n += n

    def add_images(self, hist_all: np.ndarray, hist_pos: np.ndarray, abs_sum: np.ndarray, hw) -> None:
        """Add n images from their device counts (host arrays, see image_scores) one after another, as sal_metric.cpp adds them:
        running float64 sums in image order, so the scores equal oracle/salmetric.py's on the same maps."""
        prec, rec, mae = image_scores(hist_all, hist_pos, abs_sum, hw)
        self._prec += np.cumsum(prec, 0, dtype=np.float64)[-1]
        self._rec += np.cumsum(rec, 0, dtype=np.float64)[-1]
        self._mae += float(np.cumsum(mae)[-1])
        self._n += len(mae)

    def compute(self) -> dict:
        if self._n == 0:
            raise ValueError("no images were added")
        p, r, m = self._prec / self._n, self._rec / self._n, self._mae / self._n
        f = ((1 + BETA) * p * r) / (BETA * p + r)
        k = int(np.argmax(f))
        return dict(max_f=float(f[k]), mean_f=float(f.mean()), precision=float(p[k]), recall=float(r[k]),
                    mean_precision=float(p.mean()), mean_recall=float(r.mean()), mae=float(m), argmax=k)
