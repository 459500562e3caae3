"""Training path of the CSF+Res2Net head: autograd Functions over the `csnet_train_conv_*`, `_gn_*` and `_resize_*` kernels, and the
head's forward restated on them in the reference's order.

`CSFNet.forward` runs this whenever autograd records (the backbone stays on torch autograd, cuDNN).  The order follows
networks/gOctConv.py:60-114 and csf_res2net.py:205-259:
  * gOctaveConv, output branch j: the down paths (i < j) resize the input to branch j's size and convolve it, the same-size path
    convolves; these are one GEMM call with a K segment per path.  Each up path (i > j) convolves at branch i's size and is
    resize-added to the sum, in ascending i (the reference's `sum(ysets[j])`).
  * GroupNorm(32) + PReLU per branch; MSBlock's five dilated 3x3 convs write their channel slices of one tensor; cls_layer with
    bias; the final bilinear resize to the input size.
torch is plumbing here (storage, the tape); every kernel that touches an activation or a gradient is ours.

Activation storage (`net.train_storage`, set by CSFTrainer(storage=...)): "fp32" (default) or "bf16".  Each Function follows the dtype of
the activations it receives: fp32 runs the fp32 kernels above; bf16 (the backbone's features under autocast) runs their `_bf16` twins,
with the convolutions on the tensor-core GEMM.  In bf16 the activations and their gradients are bf16; parameters, their gradients,
GroupNorm statistics, cls_layer's 1-channel map and the logits stay fp32.  A step rounds each weight to bf16 once, in the forward, and
the data gradient reads the same rounded copy.
"""
from __future__ import annotations

import ctypes as C
from typing import List, NamedTuple, Optional, Sequence

import torch

from . import runtime, splits
from . import train_ops as T

GN_EPS = 1e-5
GN_GROUPS = 32


class ConvSeg(C.Structure):
    _fields_ = [("src", C.c_void_p), ("w", C.c_void_p), ("C", C.c_int32), ("c0", C.c_int32), ("cin", C.c_int32),
                ("cout0", C.c_int32), ("cout", C.c_int32), ("ksize", C.c_int32), ("dil", C.c_int32), ("ldw", C.c_int32)]


assert C.sizeof(ConvSeg) == 48

_lib = None


def lib():
    global _lib
    if _lib is None:
        l = runtime.load_library()
        vp, i32, i64, f = C.c_void_p, C.c_int32, C.c_int64, C.c_float
        segp = C.POINTER(ConvSeg)
        l.csnet_train_last_error.restype = C.c_char_p
        l.csnet_train_conv_plan.argtypes = [i32, i32, i32, i32, segp, i32, i32, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i64)]
        l.csnet_train_conv_fwd.argtypes = [vp, i32, i32, i32, i32, segp, i32, vp, i32, i32, i32, vp, i64, vp]
        l.csnet_train_conv_dgrad.argtypes = [vp, i32, i32, i32, i32, i32, i32, segp, i32, i32, i32, i32, vp, i64, vp]
        l.csnet_train_conv_wgrad.argtypes = [vp, i32, i32, i32, i32, segp, vp, i32, i32, i32, vp, i64, vp]
        l.csnet_train_bias_grad.argtypes = [vp, i32, i32, i32, i32, i32, vp, vp]
        l.csnet_train_gn_stats.argtypes = [vp, i32, i32, i32, i32, vp, vp, vp]
        l.csnet_train_gn_prelu_fwd.argtypes = [vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, f, vp]
        l.csnet_train_gn_prelu_bwd.argtypes = [vp, vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, f, vp, vp, vp, vp, vp]
        l.csnet_train_resize_fwd.argtypes = [vp, i32, i32, i32, i32, vp, i32, i32, i32, vp]
        l.csnet_train_resize_bwd.argtypes = [vp, i32, i32, i32, i32, vp, i32, i32, vp]
        l.csnet_train_cast_bf16.argtypes = [vp, vp, i64, vp]
        l.csnet_train_conv_plan_bf16.argtypes = [i32, i32, i32, i32, segp, i32, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i64)]
        l.csnet_train_conv_fwd_bf16.argtypes = [vp, i32, i32, i32, i32, i32, segp, i32, vp, i32, i32, vp, i64, vp]
        l.csnet_train_conv_dgrad_bf16.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, segp, i32, i32, i32, vp, i64, vp]
        l.csnet_train_conv_wgrad_bf16.argtypes = [vp, i32, i32, i32, i32, segp, vp, i32, i32, vp, i64, vp]
        l.csnet_train_gn_stats_bf16.argtypes = l.csnet_train_gn_stats.argtypes
        l.csnet_train_gn_prelu_fwd_bf16.argtypes = l.csnet_train_gn_prelu_fwd.argtypes
        l.csnet_train_gn_prelu_bwd_bf16.argtypes = l.csnet_train_gn_prelu_bwd.argtypes
        l.csnet_train_resize_fwd_bf16.argtypes = l.csnet_train_resize_fwd.argtypes
        l.csnet_train_resize_bwd_bf16.argtypes = l.csnet_train_resize_bwd.argtypes
        _lib = l
    return _lib


def _ck(rc, what):
    if rc != 0:
        raise runtime.EngineError(f"{what} failed ({rc}): {lib().csnet_train_last_error().decode()}")


def _st(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def _f32(t: torch.Tensor) -> torch.Tensor:
    if not t.is_cuda:
        raise runtime.EngineError("CSF+Res2Net training runs on the GPU only: got a CPU tensor")
    if t.dtype != torch.float32:
        raise runtime.EngineError(f"CSF+Res2Net training is fp32: got {t.dtype}")
    return t.contiguous()


def _act(t: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """An activation or gradient of the given storage dtype, contiguous."""
    if not t.is_cuda:
        raise runtime.EngineError("CSF+Res2Net training runs on the GPU only: got a CPU tensor")
    if t.dtype != dtype:
        raise runtime.EngineError(f"CSF+Res2Net training with {dtype} storage: got a {t.dtype} activation")
    return t.contiguous()


def _storage(t: torch.Tensor) -> torch.dtype:
    """The storage dtype a Function runs in: that of the activation it receives."""
    if t.dtype not in (torch.float32, torch.bfloat16):
        raise runtime.EngineError(f"CSF+Res2Net training stores fp32 or bf16 activations: got {t.dtype}")
    return t.dtype


def train_dtype(net) -> torch.dtype:
    """The activation dtype of `net`'s training forward (net.train_storage); any value but "fp32" / "bf16" raises ValueError."""
    storage = getattr(net, "train_storage", "fp32")
    if storage not in T.STORAGES:
        raise ValueError(f"train_storage must be one of {sorted(T.STORAGES)}, got {storage!r}")
    return T.STORAGES[storage]


def cast_bf16(t: torch.Tensor) -> torch.Tensor:
    """fp32 -> bf16, round to nearest even (csnet_train_cast_bf16)."""
    t = _f32(t)
    out = torch.empty(t.shape, dtype=torch.bfloat16, device=t.device)
    _ck(lib().csnet_train_cast_bf16(t.data_ptr(), out.data_ptr(), t.numel(), _st(t)), "csnet_train_cast_bf16")
    return out


# ---- raw kernel calls ------------------------------------------------------------------------------------------------
def seg(src: torch.Tensor, w: torch.Tensor, co0: int, co1: int, ci0: int, ci1: int, c0: int = 0, cout0: int = 0, dil: int = 1) -> ConvSeg:
    """Segment of the conv with weight slice w[co0:co1, ci0:ci1] (w: a full OIHW parameter, contiguous).  fwd / wgrad: `src` is the
    input, read from channel c0; dgrad: pass the output's gradient as `src`, its slice starting at cout0."""
    k = w.shape[2]
    ldw = w.shape[1] * k * k
    wp = w.data_ptr() + w.element_size() * (co0 * ldw + ci0 * k * k)
    return ConvSeg(src.data_ptr(), wp, src.shape[1], c0, ci1 - ci0, cout0, co1 - co0, k, dil, ldw)


def conv_plan(form: int, N: int, H: int, W: int, segs: Sequence[ConvSeg], splits_: int = 0, tile: int = 0):
    """(splits, chain, workspace bytes) the call would use."""
    arr = (ConvSeg * len(segs))(*segs)
    s, ch, ws = C.c_int32(), C.c_int32(), C.c_int64()
    _ck(lib().csnet_train_conv_plan(form, N, H, W, arr, len(segs), splits_, tile, C.byref(s), C.byref(ch), C.byref(ws)), "csnet_train_conv_plan")
    return s.value, ch.value, ws.value


def _ws(form, N, H, W, segs, splits_, tile, dev):
    _, _, nb = conv_plan(form, N, H, W, segs, splits_, tile)
    return torch.empty(max(nb // 4, 1), dtype=torch.float32, device=dev), nb


def conv_fwd(dst: torch.Tensor, segs: Sequence[ConvSeg], bias: Optional[int] = None, accumulate=False, splits_=0, tile=0):
    N, Cd, H, W = dst.shape
    ws, nb = _ws(0, N, H, W, segs, splits_, tile, dst.device)
    arr = (ConvSeg * len(segs))(*segs)
    _ck(lib().csnet_train_conv_fwd(dst.data_ptr(), N, Cd, H, W, arr, len(segs), bias, int(accumulate), splits_, tile, ws.data_ptr(), nb,
                                   _st(dst)), "csnet_train_conv_fwd")


def conv_dgrad(dsrc: torch.Tensor, c0: int, cin: int, segs: Sequence[ConvSeg], accumulate=False, splits_=0, tile=0):
    N, Cs, H, W = dsrc.shape
    ws, nb = _ws(1, N, H, W, segs, splits_, tile, dsrc.device)
    arr = (ConvSeg * len(segs))(*segs)
    _ck(lib().csnet_train_conv_dgrad(dsrc.data_ptr(), N, Cs, H, W, c0, cin, arr, len(segs), int(accumulate), splits_, tile, ws.data_ptr(), nb,
                                     _st(dsrc)), "csnet_train_conv_dgrad")


def conv_wgrad(ddst: torch.Tensor, s: ConvSeg, dw_ptr: int, accumulate=False, splits_=0, tile=0):
    N, Cd, H, W = ddst.shape
    ws, nb = _ws(2, N, H, W, [s], splits_, tile, ddst.device)
    _ck(lib().csnet_train_conv_wgrad(ddst.data_ptr(), N, Cd, H, W, C.byref(s), dw_ptr, int(accumulate), splits_, tile, ws.data_ptr(), nb,
                                     _st(ddst)), "csnet_train_conv_wgrad")


_DT = {torch.float32: 0, torch.bfloat16: 2}        # CSNET_F32, CSNET_BF16


def conv_plan_bf16(form: int, N: int, H: int, W: int, segs: Sequence[ConvSeg], splits_: int = 0):
    """(splits, chain, workspace bytes) of a tensor-core (bf16) conv call."""
    arr = (ConvSeg * len(segs))(*segs)
    s, ch, ws = C.c_int32(), C.c_int32(), C.c_int64()
    _ck(lib().csnet_train_conv_plan_bf16(form, N, H, W, arr, len(segs), splits_, C.byref(s), C.byref(ch), C.byref(ws)),
        "csnet_train_conv_plan_bf16")
    return s.value, ch.value, ws.value


def _ws_bf16(form, N, H, W, segs, splits_, dev):
    _, _, nb = conv_plan_bf16(form, N, H, W, segs, splits_)
    return torch.empty(max(nb // 4, 1), dtype=torch.float32, device=dev), nb


def conv_fwd_bf16(dst: torch.Tensor, segs: Sequence[ConvSeg], bias: Optional[int] = None, accumulate=False, splits_=0):
    """conv_fwd on bf16 sources and weights (tensor cores); dst bf16 or fp32."""
    N, Cd, H, W = dst.shape
    ws, nb = _ws_bf16(0, N, H, W, segs, splits_, dst.device)
    arr = (ConvSeg * len(segs))(*segs)
    _ck(lib().csnet_train_conv_fwd_bf16(dst.data_ptr(), _DT[dst.dtype], N, Cd, H, W, arr, len(segs), bias, int(accumulate), splits_,
                                        ws.data_ptr(), nb, _st(dst)), "csnet_train_conv_fwd_bf16")


def conv_dgrad_bf16(dsrc: torch.Tensor, c0: int, cin: int, segs: Sequence[ConvSeg], accumulate=False, splits_=0):
    N, Cs, H, W = dsrc.shape
    ws, nb = _ws_bf16(1, N, H, W, segs, splits_, dsrc.device)
    arr = (ConvSeg * len(segs))(*segs)
    _ck(lib().csnet_train_conv_dgrad_bf16(dsrc.data_ptr(), _DT[dsrc.dtype], N, Cs, H, W, c0, cin, arr, len(segs), int(accumulate), splits_,
                                          ws.data_ptr(), nb, _st(dsrc)), "csnet_train_conv_dgrad_bf16")


def conv_wgrad_bf16(ddst: torch.Tensor, s: ConvSeg, dw_ptr: int, accumulate=False, splits_=0):
    N, Cd, H, W = ddst.shape
    ws, nb = _ws_bf16(2, N, H, W, [s], splits_, ddst.device)
    _ck(lib().csnet_train_conv_wgrad_bf16(ddst.data_ptr(), N, Cd, H, W, C.byref(s), dw_ptr, int(accumulate), splits_, ws.data_ptr(), nb,
                                          _st(ddst)), "csnet_train_conv_wgrad_bf16")


def resize_fwd(src: torch.Tensor, size, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """F.interpolate(src, size, mode='bilinear', align_corners=False); with `out`, added to it in place."""
    N, Cs, Hs, Ws = src.shape
    acc = out is not None
    if out is None:
        out = torch.empty((N, Cs, int(size[0]), int(size[1])), dtype=src.dtype, device=src.device)
    if out.dtype != src.dtype:
        raise runtime.EngineError(f"resize: {src.dtype} source, {out.dtype} destination")
    fn = lib().csnet_train_resize_fwd_bf16 if src.dtype == torch.bfloat16 else lib().csnet_train_resize_fwd
    _ck(fn(src.data_ptr(), N, Cs, Hs, Ws, out.data_ptr(), out.shape[2], out.shape[3], int(acc), _st(src)), "csnet_train_resize_fwd")
    return out


def resize_bwd(ddst: torch.Tensor, src_hw) -> torch.Tensor:
    N, Cd, Hd, Wd = ddst.shape
    d = torch.empty((N, Cd, int(src_hw[0]), int(src_hw[1])), dtype=ddst.dtype, device=ddst.device)
    fn = lib().csnet_train_resize_bwd_bf16 if ddst.dtype == torch.bfloat16 else lib().csnet_train_resize_bwd
    _ck(fn(ddst.data_ptr(), N, Cd, Hd, Wd, d.data_ptr(), d.shape[2], d.shape[3], _st(ddst)), "csnet_train_resize_bwd")
    return d


# ---- autograd Functions ----------------------------------------------------------------------------------------------
class Path(NamedTuple):
    src: int                 # index of the input tensor
    w: int                   # index of the OIHW weight parameter
    co0: int                 # weight slice [co0:co1, ci0:ci1]
    co1: int
    ci0: int
    ci1: int
    cout0: int = 0           # first output channel written
    dil: int = 1


class Out(NamedTuple):
    C: int
    H: int
    W: int
    paths: tuple
    bias: Optional[int] = None   # index of a bias [C] added once
    f32: bool = False            # with bf16 storage, an fp32 destination (cls_layer's 1-channel map)


class ConvFn(torch.autograd.Function):
    """Several outputs, each the sum of stride-1 convolutions of its paths (1x1, or 3x3 with dilation d and padding d).  Paths
    writing the same channel slice of an output are one GEMM call (a K segment each); the backward gives each source one data
    gradient call over every path it feeds, and each weight slice its own weight-gradient call."""

    @staticmethod
    def forward(ctx, outs, *tensors):
        if _storage(tensors[outs[0].paths[0].src]) == torch.bfloat16:
            return _conv_fwd_bf16(ctx, outs, tensors)
        ctx.bf16 = False
        tensors = [_f32(t.detach()) for t in tensors]
        n = tensors[outs[0].paths[0].src].shape[0]
        dev = tensors[0].device
        res = []
        for o in outs:
            dst = torch.empty((n, o.C, o.H, o.W), dtype=torch.float32, device=dev)
            slices = {}
            for p in o.paths:
                slices.setdefault(p.cout0, []).append(p)
            for c0, ps in slices.items():
                segs = [seg(tensors[p.src], tensors[p.w], p.co0, p.co1, p.ci0, p.ci1, cout0=p.cout0, dil=p.dil) for p in ps]
                b = tensors[o.bias].data_ptr() + 4 * c0 if o.bias is not None else None
                conv_fwd(dst, segs, bias=b)
            res.append(dst)
        ctx.outs = outs
        ctx.save_for_backward(*tensors)
        return tuple(res)

    @staticmethod
    def backward(ctx, *douts):
        if ctx.bf16:
            return _conv_bwd_bf16(ctx, douts)
        outs = ctx.outs
        t = ctx.saved_tensors
        dev = t[0].device
        douts = [_f32(d) if d is not None else None for d in douts]
        n = t[outs[0].paths[0].src].shape[0]
        for k, o in enumerate(outs):
            if douts[k] is None:
                douts[k] = torch.zeros((n, o.C, o.H, o.W), dtype=torch.float32, device=dev)
        grads: List[Optional[torch.Tensor]] = [None] * len(t)
        by_src = {}
        for k, o in enumerate(outs):
            for p in o.paths:
                by_src.setdefault(p.src, []).append((k, p))
        for s, kps in by_src.items():
            if not ctx.needs_input_grad[1 + s]:
                continue
            x = t[s]
            d = torch.empty_like(x)
            segs = [seg(douts[k], t[p.w], p.co0, p.co1, p.ci0, p.ci1, cout0=p.cout0, dil=p.dil) for k, p in kps]
            for i in range(0, len(segs), 8):                    # up to 8 K segments per call
                conv_dgrad(d, 0, x.shape[1], segs[i:i + 8], accumulate=i > 0)
            grads[s] = d
        seen = {}
        for k, o in enumerate(outs):
            for p in o.paths:
                if not ctx.needs_input_grad[1 + p.w]:
                    continue
                w = t[p.w]
                if grads[p.w] is None:
                    grads[p.w] = torch.zeros_like(w)
                key = (p.w, p.co0, p.ci0)
                s_ = seg(t[p.src], grads[p.w], p.co0, p.co1, p.ci0, p.ci1, cout0=p.cout0, dil=p.dil)
                conv_wgrad(douts[k], s_, s_.w, accumulate=key in seen)
                seen[key] = True
            if o.bias is not None and ctx.needs_input_grad[1 + o.bias]:
                db = torch.empty(o.C, dtype=torch.float32, device=dev)
                dd = douts[k]
                _ck(lib().csnet_train_bias_grad(dd.data_ptr(), n, o.C, o.H * o.W, 0, o.C, db.data_ptr(), _st(dd)), "csnet_train_bias_grad")
                grads[o.bias] = db if grads[o.bias] is None else grads[o.bias] + db
        return (None, *grads)


def _weights(outs) -> set:
    return {p.w for o in outs for p in o.paths}


def _conv_fwd_bf16(ctx, outs, tensors):
    """ConvFn.forward with bf16 storage: activations bf16, each weight rounded once to bf16 (kept for the data gradient), bias fp32."""
    wi, bi = _weights(outs), {o.bias for o in outs if o.bias is not None}
    t = [cast_bf16(v.detach()) if i in wi else (_f32(v.detach()) if i in bi else _act(v.detach(), torch.bfloat16))
         for i, v in enumerate(tensors)]
    n = t[outs[0].paths[0].src].shape[0]
    dev = t[0].device
    res = []
    for o in outs:
        dst = torch.empty((n, o.C, o.H, o.W), dtype=torch.float32 if o.f32 else torch.bfloat16, device=dev)
        slices = {}
        for p in o.paths:
            slices.setdefault(p.cout0, []).append(p)
        for c0, ps in slices.items():
            segs = [seg(t[p.src], t[p.w], p.co0, p.co1, p.ci0, p.ci1, cout0=p.cout0, dil=p.dil) for p in ps]
            b = t[o.bias].data_ptr() + 4 * c0 if o.bias is not None else None
            conv_fwd_bf16(dst, segs, bias=b)
        res.append(dst)
    ctx.bf16 = True
    ctx.outs = outs
    ctx.wshape = {i: tuple(tensors[i].shape) for i in wi}
    ctx.save_for_backward(*t)
    return tuple(res)


def _conv_bwd_bf16(ctx, douts):
    """ConvFn.backward with bf16 storage: data gradients bf16 on the rounded weights, weight gradients fp32.  An fp32 output gradient
    (cls_layer's map) is rounded to bf16 for the GEMMs; the bias gradient reduces it in fp32."""
    outs = ctx.outs
    t = ctx.saved_tensors
    dev = t[0].device
    n = t[outs[0].paths[0].src].shape[0]
    raw = list(douts)
    dq = []
    for k, o in enumerate(outs):
        d = raw[k]
        if d is None:
            d = torch.zeros((n, o.C, o.H, o.W), dtype=torch.bfloat16, device=dev)
        elif o.f32:
            d = cast_bf16(d)
        else:
            d = _act(d, torch.bfloat16)
        dq.append(d)
    grads: List[Optional[torch.Tensor]] = [None] * len(t)
    by_src = {}
    for k, o in enumerate(outs):
        for p in o.paths:
            by_src.setdefault(p.src, []).append((k, p))
    for s, kps in by_src.items():
        if not ctx.needs_input_grad[1 + s]:
            continue
        x = t[s]
        d = torch.empty_like(x)
        segs = [seg(dq[k], t[p.w], p.co0, p.co1, p.ci0, p.ci1, cout0=p.cout0, dil=p.dil) for k, p in kps]
        for i in range(0, len(segs), 8):                        # up to 8 K segments per call
            conv_dgrad_bf16(d, 0, x.shape[1], segs[i:i + 8], accumulate=i > 0)
        grads[s] = d
    seen = {}
    for k, o in enumerate(outs):
        for p in o.paths:
            if not ctx.needs_input_grad[1 + p.w]:
                continue
            if grads[p.w] is None:
                grads[p.w] = torch.zeros(ctx.wshape[p.w], dtype=torch.float32, device=dev)
            key = (p.w, p.co0, p.ci0)
            s_ = seg(t[p.src], grads[p.w], p.co0, p.co1, p.ci0, p.ci1, cout0=p.cout0, dil=p.dil)
            conv_wgrad_bf16(dq[k], s_, s_.w, accumulate=key in seen)
            seen[key] = True
        if o.bias is not None and ctx.needs_input_grad[1 + o.bias]:
            if not o.f32 or raw[k] is None:
                raise runtime.EngineError("bf16 storage: a bias gradient is reduced from an fp32 output gradient only")
            dd = _f32(raw[k])
            db = torch.empty(o.C, dtype=torch.float32, device=dev)
            _ck(lib().csnet_train_bias_grad(dd.data_ptr(), n, o.C, o.H * o.W, 0, o.C, db.data_ptr(), _st(dd)), "csnet_train_bias_grad")
            grads[o.bias] = db if grads[o.bias] is None else grads[o.bias] + db
    return (None, *grads)


class ResizeFn(torch.autograd.Function):
    """F.interpolate(src, size, mode='bilinear', align_corners=False), or `base + that` written into `base` (resize-add)."""

    @staticmethod
    def forward(ctx, src, size, base=None):
        src = _act(src.detach(), _storage(src))
        ctx.src_hw = tuple(src.shape[2:])
        if base is not None:
            if not base.is_contiguous():
                raise runtime.EngineError("resize-add needs a contiguous destination")
            ctx.mark_dirty(base)
            return resize_fwd(src, size, base)
        return resize_fwd(src, size)

    @staticmethod
    def backward(ctx, dout):
        dout = _act(dout, _storage(dout))
        dsrc = resize_bwd(dout, ctx.src_hw) if ctx.needs_input_grad[0] else None
        has_base = len(ctx.needs_input_grad) > 2 and ctx.needs_input_grad[2]
        return dsrc, None, dout if has_base else None


class GnPreluFn(torch.autograd.Function):
    """F.prelu(F.group_norm(z, 32, gamma, beta, 1e-5), slope)."""

    @staticmethod
    def forward(ctx, z, gamma, beta, slope):
        z = _act(z.detach(), _storage(z))
        g, b, a = (_f32(v.detach()) for v in (gamma, beta, slope))
        n, c, h, w = z.shape
        mean = torch.empty(n * GN_GROUPS, dtype=torch.float32, device=z.device)
        var = torch.empty_like(mean)
        y = torch.empty_like(z)
        bf = z.dtype == torch.bfloat16
        stats = lib().csnet_train_gn_stats_bf16 if bf else lib().csnet_train_gn_stats
        fwd = lib().csnet_train_gn_prelu_fwd_bf16 if bf else lib().csnet_train_gn_prelu_fwd
        _ck(stats(z.data_ptr(), n, c, h * w, GN_GROUPS, mean.data_ptr(), var.data_ptr(), _st(z)), "csnet_train_gn_stats")
        _ck(fwd(z.data_ptr(), y.data_ptr(), n, c, h * w, GN_GROUPS, mean.data_ptr(), var.data_ptr(), g.data_ptr(),
                                           b.data_ptr(), a.data_ptr(), GN_EPS, _st(z)), "csnet_train_gn_prelu_fwd")
        ctx.save_for_backward(z, mean, var, g, b, a)
        return y

    @staticmethod
    def backward(ctx, dy):
        z, mean, var, g, b, a = ctx.saved_tensors
        dy = _act(dy, z.dtype)
        n, c, h, w = z.shape
        dz = torch.empty_like(z)
        dg, db, da = (torch.empty(c, dtype=torch.float32, device=z.device) for _ in range(3))
        ws = torch.empty(3 * n * c, dtype=torch.float32, device=z.device)
        bwd = lib().csnet_train_gn_prelu_bwd_bf16 if z.dtype == torch.bfloat16 else lib().csnet_train_gn_prelu_bwd
        _ck(bwd(z.data_ptr(), dy.data_ptr(), dz.data_ptr(), n, c, h * w, GN_GROUPS, mean.data_ptr(), var.data_ptr(),
                                           g.data_ptr(), b.data_ptr(), a.data_ptr(), GN_EPS, dg.data_ptr(), db.data_ptr(), da.data_ptr(),
                                           ws.data_ptr(), _st(z)), "csnet_train_gn_prelu_bwd")
        return dz, dg, db, da


# ---- the head, in the reference's order ------------------------------------------------------------------------------
def goct_conv_1x1(xs: Sequence[torch.Tensor], weight: torch.Tensor, alpha_in, alpha_out) -> List[torch.Tensor]:
    """gOctaveConv.forward (gOctConv.py:60-114) with 1x1 kernels, stride 1, no bias: branch j's output has xs[j]'s size."""
    ci, co = splits.cuts(weight.shape[1], alpha_in), splits.cuts(weight.shape[0], alpha_out)
    sizes = [tuple(x.shape[2:]) for x in xs]
    inputs: List[torch.Tensor] = list(xs) + [weight]
    wi = len(xs)
    outs = []
    for j in range(len(alpha_out)):
        cj = co[j + 1] - co[j]
        if cj == 0:
            continue
        paths = []
        for i in range(len(alpha_in)):
            if ci[i] == ci[i + 1]:
                continue
            if i < j:                                              # resize the input down, then convolve (:101-103)
                inputs.append(ResizeFn.apply(xs[i], sizes[j]))
                paths.append(Path(len(inputs) - 1, wi, co[j], co[j + 1], ci[i], ci[i + 1]))
            elif i == j:
                paths.append(Path(i, wi, co[j], co[j + 1], ci[i], ci[i + 1]))
            else:                                                  # convolve at branch i's size, resize the output up (:98-100)
                outs.append(("low", j, i, Out(cj, *sizes[i], (Path(i, wi, co[j], co[j + 1], ci[i], ci[i + 1]),))))
        outs.append(("raw", j, None, Out(cj, *sizes[j], tuple(paths))))
    res = ConvFn.apply(tuple(o[3] for o in outs), *inputs)
    raw = {o[1]: r for o, r in zip(outs, res) if o[0] == "raw"}
    low = {(o[1], o[2]): r for o, r in zip(outs, res) if o[0] == "low"}
    ys = []
    for j in range(len(alpha_out)):
        if j not in raw:
            ys.append(None)
            continue
        z = raw[j]
        for i in range(j + 1, len(alpha_in)):                     # sum(ysets[j]) in ascending i
            if (j, i) in low:
                z = ResizeFn.apply(low[(j, i)], sizes[j], z)
        ys.append(z)
    return ys


def gn_prelu(z, gn: torch.nn.GroupNorm, prelu: torch.nn.PReLU):
    return GnPreluFn.apply(z, gn.weight, gn.bias, prelu.weight)


def msblock(x, block) -> torch.Tensor:
    """MSBlock.forward (csf_res2net.py:218-225): five dilated 3x3 convs into one tensor's channel slices, GroupNorm, PReLU."""
    paths, c = [], 0
    ws = [m.weight for m in block.msconv]
    for d, (w, dil) in enumerate(zip(ws, block.dilations)):
        paths.append(Path(0, 1 + d, 0, w.shape[0], 0, w.shape[1], cout0=c, dil=dil))
        c += w.shape[0]
    (raw,) = ConvFn.apply((Out(c, x.shape[2], x.shape[3], tuple(paths)),), x, *ws)
    return gn_prelu(raw, block.bn, block.prelu)


def csf_head(net, feats: Sequence[torch.Tensor], size) -> torch.Tensor:
    """CSFNet.forward after the backbone (csf_res2net.py:253-258) on `net`'s parameters: fp32 logits [N, 1, H, W] at `size`.  The
    features' dtype (fp32, or bf16 with bf16 storage) is the head's activation storage; cls_layer writes its map in fp32."""
    fuse = net.fuse
    y = goct_conv_1x1(feats, fuse.conv.weights, fuse.alpha_in, fuse.alpha_out)
    y = [gn_prelu(t, fuse.bns[j], fuse.prelus[j]) if t is not None else None for j, t in enumerate(y)]
    z = [msblock(t, net.ms.convs[b]) for b, t in enumerate(y)]
    f1 = net.fuse1x1
    f = goct_conv_1x1(z, f1.conv.weights, f1.alpha_in, f1.alpha_out)
    f0 = gn_prelu(f[0], f1.bns[0], f1.prelus[0])
    cl = net.cls_layer
    (out,) = ConvFn.apply((Out(cl.weight.shape[0], f0.shape[2], f0.shape[3], (Path(0, 1, 0, cl.weight.shape[0], 0, cl.weight.shape[1]),),
                               bias=2, f32=True),), f0, cl.weight, cl.bias)
    return ResizeFn.apply(out, tuple(size))
