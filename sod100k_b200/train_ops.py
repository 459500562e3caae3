"""Training primitives: ctypes bindings of the `csnet_train_*` C ABI wrapped as torch.autograd.Function s.

torch is plumbing here (tensor storage, the autograd tape, tiny parameter reshapes); every kernel that touches an
activation is ours.  fp32 activations (the parity configuration); see DESIGN.md for the bf16 plan.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import runtime

BN_EPS = 1e-5


class TrainPath(C.Structure):
    _fields_ = [("src", C.c_void_p), ("w", C.c_void_p), ("C", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
                ("c0", C.c_int32), ("cin", C.c_int32), ("pre_avg", C.c_int32), ("pool", C.c_int32), ("ksize", C.c_int32),
                ("dil", C.c_int32), ("stride", C.c_int32), ("pad", C.c_int32), ("up", C.c_int32), ("cout0", C.c_int32),
                ("cout", C.c_int32)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        l = runtime.load_library()
        l.csnet_train_last_error.restype = C.c_char_p
        f32p, vp, i32, i64, f = C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_float
        l.csnet_train_bn_stats.argtypes = [f32p, i32, i32, i32, f32p, f32p, vp]
        l.csnet_train_bn_prelu_fwd.argtypes = [f32p, f32p, i32, i32, i32, f32p, f32p, f32p, f32p, f32p, f, f32p, vp]
        l.csnet_train_bn_prelu_bwd.argtypes = [f32p, f32p, f32p, i32, i32, i32, f32p, f32p, f32p, f32p, f32p, f, f32p, f32p, f32p, i32, vp]
        l.csnet_train_dw_conv.argtypes = [f32p, f32p, f32p, i32, i32, i32, i32, f, i32, vp]
        l.csnet_train_dw_wgrad.argtypes = [f32p, f32p, f32p, i32, i32, i32, i32, f, vp]
        l.csnet_train_dw_bwd.argtypes = [f32p, f32p, f32p, f32p, f32p, i32, i32, i32, i32, f, vp]
        l.csnet_train_mix_fwd.argtypes = [f32p, i32, i32, i32, i32, C.POINTER(TrainPath), i32, vp]
        l.csnet_train_mix_dgrad.argtypes = [f32p, i32, i32, i32, i32, C.POINTER(TrainPath), f32p, vp]
        l.csnet_train_mix_wgrad.argtypes = [f32p, i32, i32, i32, i32, C.POINTER(TrainPath), f32p, vp]
        l.csnet_train_pool_fwd.argtypes = [f32p, i32, i32, i32, i32, i32, i32, i32, i32, f32p, vp, vp]
        l.csnet_train_pool_bwd.argtypes = [f32p, vp, i32, i32, i32, i32, i32, i32, f32p, vp]
        l.csnet_train_bce.argtypes = [f32p, f32p, f32p, f32p, i64, f, vp]
        l.csnet_train_adam.argtypes = [vp, i32, f, f, f, f, i32, f, vp]
        _lib = l
    return _lib


# True while a checkpointed ILBlock is being re-run in the backward pass (modular.csnet_forward with recompute): the second run must
# not update BatchNorm running statistics or the dynamic-weight-decay accumulator again
RECOMPUTING = False


class recomputing:
    def __enter__(self):
        global RECOMPUTING
        self._old, RECOMPUTING = RECOMPUTING, True

    def __exit__(self, *exc):
        global RECOMPUTING
        RECOMPUTING = self._old


# kernels launched through this module since import (bench.py reports the count of a timed region): kernels per entry point
LAUNCHES = 0
_KERNELS = {"csnet_train_bn_prelu_bwd": 2, "csnet_train_mix_wgrad": 2, "csnet_train_dw_wgrad": 2, "csnet_train_dw_bwd": 2}


def _ck(rc, what):
    global LAUNCHES
    if rc != 0:
        raise runtime.EngineError(f"{what} failed ({rc}): {lib().csnet_train_last_error().decode()}")
    LAUNCHES += _KERNELS.get(what, 1)


def _stream(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def _f32(t: torch.Tensor) -> torch.Tensor:
    if not t.is_cuda:
        raise runtime.EngineError("training runs on the GPU only: got a CPU tensor")
    return t.contiguous().float()


# ---- raw conv mix ------------------------------------------------------------------------------------------------
@dataclass
class PathSpec:
    src: int                 # index into the Function's tensor inputs
    w: Optional[int]         # index of the packed weight [cin][k*k][cout]; None for resample-add paths
    cin: int
    cout: int
    cout0: int = 0
    c0: int = 0
    pre_avg: int = 0
    pool: int = 1
    ksize: int = 1
    dil: int = 1
    stride: int = 1
    pad: int = 0
    up: int = 1


def _cpath(ps: PathSpec, tensors: Sequence[torch.Tensor]) -> TrainPath:
    s = tensors[ps.src]
    return TrainPath(s.data_ptr(), tensors[ps.w].data_ptr() if ps.w is not None else None, s.shape[1], s.shape[2], s.shape[3],
                     ps.c0, ps.cin, ps.pre_avg, ps.pool, ps.ksize, ps.dil, ps.stride, ps.pad, ps.up, ps.cout0, ps.cout)


class MixFn(torch.autograd.Function):
    """dst[N, C, H, W] = sum of paths (gOctaveConv.forward for one output branch, csnet.py:664-726).

    The down-sampling of a path (2x2 average of a stride-2 conv, max-pool of a high -> low path) is materialised once by
    csnet_train_pool_fwd, with the arg-max; the convolution kernels then see dense stride-1 paths only, the backward routes the
    pooled gradient with csnet_train_pool_bwd, and the full-resolution source is not kept for this Function."""

    @staticmethod
    def forward(ctx, spec, *tensors):
        out_c, out_h, out_w, paths = spec
        tensors = [_f32(t) for t in tensors]
        n = tensors[paths[0].src].shape[0]
        dev = tensors[0].device
        st = torch.cuda.current_stream(dev).cuda_stream
        saved = list(tensors)
        dense, pooled = [], {}
        for k, p in enumerate(paths):
            if p.ksize > 0 and (p.pre_avg or p.pool > 1):
                s = tensors[p.src]
                f = (2 if p.pre_avg else 1) * p.pool
                xp = torch.empty((n, p.cin, s.shape[2] // f, s.shape[3] // f), dtype=torch.float32, device=dev)
                idx = torch.empty(xp.shape, dtype=torch.uint8, device=dev) if p.pool > 1 else None
                _ck(lib().csnet_train_pool_fwd(s.data_ptr(), n, s.shape[1], p.c0, p.cin, s.shape[2], s.shape[3], p.pre_avg, p.pool,
                                               xp.data_ptr(), idx.data_ptr() if idx is not None else None, st), "csnet_train_pool_fwd")
                saved += [xp, idx]
                pooled[k] = (len(saved) - 2, len(saved) - 1, tuple(s.shape))
                dense.append(PathSpec(len(saved) - 2, p.w, p.cin, p.cout, cout0=p.cout0, ksize=p.ksize, dil=p.dil, stride=p.stride, pad=p.pad))
            else:
                dense.append(p)
        dst = torch.empty((n, out_c, out_h, out_w), dtype=torch.float32, device=dev)
        arr = (TrainPath * len(dense))(*[_cpath(p, saved) for p in dense])
        _ck(lib().csnet_train_mix_fwd(dst.data_ptr(), n, out_c, out_h, out_w, arr, len(dense), st), "csnet_train_mix_fwd")
        # a source used only through its pooled copy is not kept
        direct = {p.src for k, p in enumerate(paths) if k not in pooled}
        shapes = [tuple(t.shape) for t in tensors]
        for k, p in enumerate(paths):
            if k in pooled and p.src not in direct:
                saved[p.src] = None
        ctx.spec, ctx.dense, ctx.pooled, ctx.shapes, ctx.n_in = spec, dense, pooled, shapes, len(tensors)
        ctx.save_for_backward(*saved)
        return dst

    @staticmethod
    def backward(ctx, ddst):
        out_c, out_h, out_w, paths = ctx.spec
        saved = ctx.saved_tensors
        ddst = _f32(ddst)
        n = ddst.shape[0]
        grads: List[Optional[torch.Tensor]] = [None] * ctx.n_in
        st = _stream(ddst)
        for k, (p, q) in enumerate(zip(paths, ctx.dense)):
            cp = _cpath(q, saved)
            shp = ctx.shapes[p.src]
            if ctx.needs_input_grad[1 + p.src]:
                xs = saved[q.src].shape
                d = torch.empty((n, p.cin, xs[2], xs[3]), dtype=torch.float32, device=ddst.device)
                _ck(lib().csnet_train_mix_dgrad(ddst.data_ptr(), n, out_c, out_h, out_w, C.byref(cp), d.data_ptr(), st), "csnet_train_mix_dgrad")
                if k in ctx.pooled:
                    idx = saved[ctx.pooled[k][1]]
                    full = torch.empty((n, p.cin, shp[2], shp[3]), dtype=torch.float32, device=ddst.device)
                    _ck(lib().csnet_train_pool_bwd(d.data_ptr(), idx.data_ptr() if idx is not None else None, n, p.cin, shp[2], shp[3],
                                                   p.pre_avg, p.pool, full.data_ptr(), st), "csnet_train_pool_bwd")
                    d = full
                if p.c0 != 0 or p.cin != shp[1]:
                    full = torch.zeros(shp, dtype=torch.float32, device=ddst.device)
                    full[:, p.c0:p.c0 + p.cin] = d
                    d = full
                grads[p.src] = d if grads[p.src] is None else grads[p.src] + d
            if p.w is not None and ctx.needs_input_grad[1 + p.w]:
                dw = torch.empty_like(saved[p.w])
                _ck(lib().csnet_train_mix_wgrad(ddst.data_ptr(), n, out_c, out_h, out_w, C.byref(cp), dw.data_ptr(), st), "csnet_train_mix_wgrad")
                grads[p.w] = dw if grads[p.w] is None else grads[p.w] + dw
        return (None, *grads)


def pack_conv_weight(w: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    """[cout, cin, k, k] (a slice of a reference parameter) -> kernel layout [cin, k*k, cout]; differentiable."""
    co, ci, kh, kw = w.shape
    w = w * scale if scale != 1.0 else w
    return w.permute(1, 2, 3, 0).reshape(ci, kh * kw, co).contiguous()


# ---- train-mode BatchNorm + PReLU ----------------------------------------------------------------------------------
class BnPreluFn(torch.autograd.Function):
    """PReLU(BatchNorm2d(z)) with batch statistics (csnet.py:786,791,846-847,148); also returns the batch mean /
    biased variance (for the running-stat update) and the per-image channel means of the output (Oct_bn_hook's GAP)."""

    @staticmethod
    def forward(ctx, z, gamma, beta, slope, frozen_mean=None, frozen_var=None):
        z = _f32(z)
        n, c, h, w = z.shape
        y = torch.empty_like(z)
        gap = torch.empty((n, c), dtype=torch.float32, device=z.device)
        st = _stream(z)
        g, b, a = _f32(gamma.detach()), _f32(beta.detach()), _f32(slope.detach())
        ctx.frozen = frozen_mean is not None
        if ctx.frozen:                                   # eval-mode BN: running statistics, treated as constants
            mean, var = _f32(frozen_mean.detach()).clone(), _f32(frozen_var.detach()).clone()
        else:
            mean = torch.empty(c, dtype=torch.float32, device=z.device)
            var = torch.empty_like(mean)
            _ck(lib().csnet_train_bn_stats(z.data_ptr(), n, c, h * w, mean.data_ptr(), var.data_ptr(), st), "csnet_train_bn_stats")
        _ck(lib().csnet_train_bn_prelu_fwd(z.data_ptr(), y.data_ptr(), n, c, h * w, mean.data_ptr(), var.data_ptr(), g.data_ptr(),
                                           b.data_ptr(), a.data_ptr(), BN_EPS, gap.data_ptr(), st), "csnet_train_bn_prelu_fwd")
        ctx.save_for_backward(z, mean, var, g, b, a)
        ctx.mark_non_differentiable(mean, var, gap)
        return y, mean, var, gap

    @staticmethod
    def backward(ctx, dy, _dm, _dv, _dg):
        z, mean, var, g, b, a = ctx.saved_tensors
        dy = _f32(dy)
        n, c, h, w = z.shape
        dz = torch.empty_like(z)
        dgamma, dbeta, dslope = (torch.empty(c, dtype=torch.float32, device=z.device) for _ in range(3))
        _ck(lib().csnet_train_bn_prelu_bwd(z.data_ptr(), dy.data_ptr(), dz.data_ptr(), n, c, h * w, mean.data_ptr(), var.data_ptr(),
                                           g.data_ptr(), b.data_ptr(), a.data_ptr(), BN_EPS, dgamma.data_ptr(), dbeta.data_ptr(),
                                           dslope.data_ptr(), int(ctx.frozen), _stream(z)), "csnet_train_bn_prelu_bwd")
        return dz, dgamma, dbeta, dslope, None, None


def bn_prelu_train(z, bn: torch.nn.BatchNorm2d, prelu: torch.nn.PReLU):
    """Apply + update running statistics the way nn.BatchNorm2d does in train mode (momentum 0.1, unbiased variance)."""
    if not bn.training:                                  # frozen statistics (module left in eval mode)
        y, _, _, gap = BnPreluFn.apply(z, bn.weight, bn.bias, prelu.weight, bn.running_mean, bn.running_var)
        return y, gap
    y, mean, var, gap = BnPreluFn.apply(z, bn.weight, bn.bias, prelu.weight)
    if bn.track_running_stats and not RECOMPUTING:
        with torch.no_grad():
            m = z.shape[0] * z.shape[2] * z.shape[3]
            mom = 0.1 if bn.momentum is None else bn.momentum
            bn.running_mean.mul_(1 - mom).add_(mean, alpha=mom)
            bn.running_var.mul_(1 - mom).add_(var * (m / max(m - 1, 1)), alpha=mom)
            bn.num_batches_tracked += 1
    return y, gap


# ---- depthwise 3x3 (Conv2dX100 groups=C) ----------------------------------------------------------------------------
class DwFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, scale):
        x, wf = _f32(x), _f32(w.detach()).reshape(-1, 9)
        n, c, h, ww = x.shape
        y = torch.empty_like(x)
        _ck(lib().csnet_train_dw_conv(x.data_ptr(), wf.data_ptr(), y.data_ptr(), n, c, h, ww, scale, 0, _stream(x)), "csnet_train_dw_conv")
        ctx.save_for_backward(x, wf)
        ctx.scale, ctx.wshape = scale, w.shape
        return y

    @staticmethod
    def backward(ctx, dy):
        x, wf = ctx.saved_tensors
        dy = _f32(dy)
        n, c, h, ww = x.shape
        dx = dw = None
        if ctx.needs_input_grad[0] and ctx.needs_input_grad[1]:          # the usual case: one pass over dy for both gradients
            dx, dw = torch.empty_like(x), torch.empty_like(wf)
            _ck(lib().csnet_train_dw_bwd(x.data_ptr(), dy.data_ptr(), wf.data_ptr(), dx.data_ptr(), dw.data_ptr(), n, c, h, ww, ctx.scale,
                                         _stream(x)), "csnet_train_dw_bwd")
            return dx, dw.reshape(ctx.wshape), None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            _ck(lib().csnet_train_dw_conv(dy.data_ptr(), wf.data_ptr(), dx.data_ptr(), n, c, h, ww, ctx.scale, 1, _stream(x)), "csnet_train_dw_conv(T)")
        if ctx.needs_input_grad[1]:
            dw = torch.empty_like(wf)
            _ck(lib().csnet_train_dw_wgrad(x.data_ptr(), dy.data_ptr(), dw.data_ptr(), n, c, h, ww, ctx.scale, _stream(x)), "csnet_train_dw_wgrad")
            dw = dw.reshape(ctx.wshape)
        return dx, dw, None


# ---- loss / optimiser ------------------------------------------------------------------------------------------------
class BceFn(torch.autograd.Function):
    """F.binary_cross_entropy_with_logits(logits, target) with mean reduction (train.py:209)."""

    @staticmethod
    def forward(ctx, logits, target):
        logits, target = _f32(logits), _f32(target)
        loss = torch.zeros(1, dtype=torch.float32, device=logits.device)
        dl = torch.empty_like(logits)
        _ck(lib().csnet_train_bce(logits.data_ptr(), target.data_ptr(), dl.data_ptr(), loss.data_ptr(), logits.numel(), 1.0,
                                  _stream(logits)), "csnet_train_bce")
        ctx.save_for_backward(dl)
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        (dl,) = ctx.saved_tensors
        return dl * g, None


class BceSumFn(torch.autograd.Function):
    """F.binary_cross_entropy_with_logits(logits, target, reduction='sum') / divisor (CSF+Res2Net/solver.py:101-102), the sum
    reduced in a fixed order (csnet_train_bce_sum): the same bits on every run."""

    @staticmethod
    def forward(ctx, logits, target, divisor: int):
        logits, target = _f32(logits), _f32(target)
        if target.shape != logits.shape:
            raise ValueError(f"target {tuple(target.shape)} differs from logits {tuple(logits.shape)}")
        loss = torch.empty(1, dtype=torch.float32, device=logits.device)
        dl = torch.empty_like(logits)
        runtime.train_bce_sum(logits.data_ptr(), target.data_ptr(), dl.data_ptr(), loss.data_ptr(), logits.numel(), int(divisor),
                              _stream(logits))
        ctx.save_for_backward(dl)
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        (dl,) = ctx.saved_tensors
        return dl * g, None, None


class FusedAdam:
    """torch.optim.Adam semantics (L2 weight decay added to the gradient, bias-corrected) in ONE launch over all
    parameters; `groups` = [(params, weight_decay), ...] like the two groups of train.py:97-123."""
    CHUNK = 2048

    def __init__(self, groups, lr=1e-4, betas=(0.9, 0.99), eps=1e-8):
        self.lr, self.betas, self.eps, self.step_count = lr, betas, eps, 0
        self.params = [(p, wd) for ps, wd in groups for p in ps]
        self.m = [torch.zeros_like(p, dtype=torch.float32) for p, _ in self.params]
        self.v = [torch.zeros_like(p, dtype=torch.float32) for p, _ in self.params]
        self._table = None
        self._ptrs = None

    def _build(self):
        rec = np.dtype([("p", "<u8"), ("g", "<u8"), ("m", "<u8"), ("v", "<u8"), ("n", "<i4"), ("wd", "<f4")])
        rows = []
        for (p, wd), m, v in zip(self.params, self.m, self.v):
            if p.grad is None:
                p.grad = torch.zeros_like(p)
            if not (p.is_contiguous() and p.grad.is_contiguous() and p.dtype == torch.float32):
                raise runtime.EngineError("FusedAdam needs contiguous fp32 parameters and gradients")
            for o in range(0, p.numel(), self.CHUNK):
                k = min(self.CHUNK, p.numel() - o)
                rows.append((p.data_ptr() + 4 * o, p.grad.data_ptr() + 4 * o, m.data_ptr() + 4 * o, v.data_ptr() + 4 * o, k, wd))
        tab = np.array(rows, dtype=rec)
        self._table = torch.from_numpy(tab.view(np.uint8).copy()).to(self.params[0][0].device)
        self._n = len(rows)
        self._ptrs = [(p.data_ptr(), p.grad.data_ptr()) for p, _ in self.params]

    def step(self, grad_scale: float = 1.0):
        if self._table is None or self._ptrs != [(p.data_ptr(), p.grad.data_ptr() if p.grad is not None else 0) for p, _ in self.params]:
            self._build()
        self.step_count += 1
        dev = self.params[0][0].device
        _ck(lib().csnet_train_adam(self._table.data_ptr(), self._n, self.lr, self.betas[0], self.betas[1], self.eps, self.step_count,
                                   grad_scale, torch.cuda.current_stream(dev).cuda_stream), "csnet_train_adam")
        runtime.PARAM_EPOCH += 1     # parameters changed behind autograd's back: invalidate folded inference programs
        return self

    def zero_grad(self):
        for p, _ in self.params:
            if p.grad is not None:
                p.grad.zero_()
