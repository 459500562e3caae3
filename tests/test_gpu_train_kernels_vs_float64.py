"""Every training kernel (sod100k_b200/csrc/train_ops.cu, train_fast.cuh) against the float64 reference of tests/trainref.py
with its per-element error bound.

(a) One case per launch form, calling the C ABI directly through train_ops.lib().  Each output lies inside a larger buffer
    whose 256-byte guard bands (and the output itself) start as a NaN pattern, so an element the kernel never writes fails
    the check and a write outside the output changes a guard.  Every element is checked (q = max |got - ref| / bound <= 1)
    and every case runs twice and must give bit-identical outputs, except the generic weight-gradient kernel
    (tr_mix_wgrad_kernel merges its image splits with atomicAdd) and the BCE loss value (an atomicAdd over blocks).
(b) Coverage: the CUDA kernels each case launches are recorded with torch.profiler (CUDA activity only); each case asserts
    the kernels it targets, and one test asserts that every __global__ instantiation of the two sources is reached.
(c) One Trainer.step of csnet-L-x2 with every MixFn / DwFn / BnPreluFn / BceFn call and FusedAdam.step certified op by op on
    that call's own inputs, at the bench configuration (batch 256, 224^2) and at batch 2, 64^2.  Every gradient MixFn returns
    is checked: the sum of its paths' data gradients (pooled paths routed through pool_bwd) or weight gradients; a gradient
    that could not be attributed is counted as skipped and fails the test.
(d) Whole-net gradients with frozen BatchNorm (the net in eval mode, frozen_bn_training) against float64 autograd, also with
    parameters frozen so that both single-gradient depthwise forms run inside the graph.

Every check prints `TRAINREF_Q <kernel> <case> <q>` (pytest -s)."""
import collections
import ctypes as C
import os
import re
import zlib
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from tests import trainref as R

pytestmark = pytest.mark.gpu

GUARD = 256
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCES = [os.path.join(ROOT, "sod100k_b200", "csrc", f) for f in ("train_ops.cu", "train_fast.cuh")]
# covered by their own suites: channel slimming (tests/test_gpu_slim.py) and SalMetric counting (tests/test_gpu_salmetric.py)
EXEMPT = {"slim_gather_kernel": "tests/test_gpu_slim.py", "salmetric_hist_kernel": "tests/test_gpu_salmetric.py"}


def _note(kernel, case, q):
    print(f"TRAINREF_Q {kernel} {case} {q:.4f}")


# ---- inputs ------------------------------------------------------------------------------------------------------------
def _gen(case_id):
    return torch.Generator().manual_seed(zlib.crc32(case_id.encode()))


def biased(g, shape, mean=0.5):
    """Normal values with a nonzero mean (a dropped image or partial then shows in every sum) and exact zeros."""
    x = torch.randn(shape, generator=g, dtype=torch.float64) + mean
    flat = x.reshape(-1)
    k = flat.numel()
    flat[torch.randint(0, k, (max(1, k // 16),), generator=g)] = 0.0
    return x.float()


@dataclass
class Case:
    id: str
    kind: str                    # mix | dw | bn | pool | bce | adam
    p: dict
    targets: tuple               # kernels the case must launch


def mix(cid, N, C, H, W, srcs, paths, targets):
    return Case(cid, "mix", dict(N=N, C=C, H=H, W=W, srcs=srcs, paths=paths), tuple(targets))


def cp(src, cin, cout, k=1, dil=1, stride=1, pad=None, c0=0, cout0=0, up=1):
    return dict(src=src, cin=cin, cout=cout, ksize=k, dil=dil, stride=stride, pad=dil * (k // 2) if pad is None else pad, c0=c0,
                cout0=cout0, up=up)


def rs(src, c, up, c0=0, cout0=0):
    return dict(src=src, cin=c, cout=c, ksize=0, dil=1, stride=1, pad=0, c0=c0, cout0=cout0, up=up)


CASES = [
    # ---- 1x1 mixes: the direct kernel's four forms (forward and transposed data gradient), conv_wgrad_kernel<1> ----------
    mix("c1_narrow", 2, 18, 16, 20, [(14, 16, 20)], [cp(0, 12, 18, c0=2)], ["conv1x1_narrow_kernel", "conv_wgrad_kernel<1>"]),
    mix("c1_wide_vec4", 2, 40, 12, 24, [(20, 12, 24)], [cp(0, 20, 40)], ["conv1x1_kernel<4,true>"]),
    mix("c1_w14", 3, 33, 14, 14, [(9, 14, 14)], [cp(0, 9, 33)], ["conv1x1_kernel<2,true>"]),
    mix("c1_w30", 2, 20, 10, 30, [(12, 10, 30)], [cp(0, 12, 20)], ["conv1x1_kernel<2,true>"]),
    mix("c1_w7", 3, 26, 7, 7, [(7, 7, 7)], [cp(0, 7, 26)], ["conv1x1_kernel<4,false>"]),
    mix("c1_w13_slices", 2, 30, 9, 13, [(11, 9, 13), (8, 9, 13)], [cp(0, 7, 20, c0=3, cout0=4), cp(1, 8, 10, cout0=20)],
        ["conv1x1_kernel<4,false>"]),
    mix("c1_with_resample", 2, 21, 24, 40, [(9, 24, 40), (21, 12, 20)], [cp(0, 9, 21), rs(1, 21, 2)],
        ["conv1x1_narrow_kernel", "resample_bwd_kernel<2>"]),
    mix("c1_tiles_over_256", 2, 72, 8, 12, [(72, 8, 12)], [cp(0, 72, 72)], ["conv_wgrad_kernel<1>"]),
    # ---- mixes the register-tiled kernels do not take: the generic tr_mix_* kernels --------------------------------------------
    mix("gen_w_tile_96k", 2, 128, 8, 8, [(200, 8, 8)], [cp(0, 200, 128)], ["tr_mix_fwd_kernel", "tr_mix_dgrad_kernel"]),
    mix("gen_w_over_1024", 1, 6, 2, 1030, [(4, 2, 1030)], [cp(0, 4, 6)], ["tr_mix_fwd_kernel", "tr_mix_dgrad_kernel"]),
    mix("gen_mixed_k", 2, 12, 10, 12, [(5, 10, 12)], [cp(0, 5, 6), cp(0, 5, 6, k=3, cout0=6)], ["tr_mix_fwd_kernel"]),
    mix("gen_6_conv_paths", 2, 18, 8, 8, [(4, 8, 8)], [cp(0, 4, 3, cout0=3 * i) for i in range(6)], ["tr_mix_fwd_kernel"]),
    mix("gen_4_resample", 2, 8, 16, 16, [(2, 8, 8), (2, 4, 4), (3, 2, 2)],
        [rs(0, 2, 2), rs(1, 2, 4, cout0=2), rs(2, 2, 8, c0=1, cout0=4), rs(0, 2, 2, cout0=6)], ["tr_mix_fwd_kernel", "tr_mix_dgrad_kernel"]),
    mix("resample_only", 2, 10, 8, 12, [(5, 4, 6), (4, 2, 3)], [rs(0, 4, 2, c0=1, cout0=1), rs(1, 4, 4, cout0=6)],
        ["conv1x1_narrow_kernel", "resample_bwd_kernel<2>", "resample_bwd_kernel<4>"]),
    mix("k5", 2, 10, 12, 16, [(6, 12, 16)], [cp(0, 6, 10, k=5)], ["conv_fwd_kernel<0>", "tr_mix_wgrad_kernel"]),
    mix("stride2", 2, 8, 8, 10, [(6, 16, 20)], [cp(0, 6, 8, k=3, stride=2)], ["tr_mix_fwd_kernel", "tr_mix_dgrad_kernel", "tr_mix_wgrad_kernel"]),
    mix("stride2_odd", 2, 5, 7, 5, [(3, 13, 9)], [cp(0, 3, 5, k=3, stride=2)], ["tr_mix_fwd_kernel", "tr_mix_wgrad_kernel"]),
    mix("k1_dil2_wgrad", 2, 6, 10, 12, [(5, 10, 12)], [cp(0, 5, 6, dil=2)], ["tr_mix_wgrad_kernel"]),
    mix("resample_up8", 2, 3, 24, 40, [(3, 3, 5)], [rs(0, 3, 8)], ["tr_mix_dgrad_kernel"]),
    mix("resample_hs1_odd", 2, 10, 2, 14, [(6, 1, 7)], [rs(0, 5, 2, c0=1, cout0=3)], ["resample_bwd_kernel<2>"]),
    mix("resample_up4_ws1", 2, 9, 20, 4, [(4, 5, 1)], [rs(0, 4, 4, cout0=2)], ["resample_bwd_kernel<4>"]),
    # ---- 3x3 / dilated: conv_fwd_kernel<3> / <0> (forward and transposed), conv_wgrad_kernel<3> / <0> ----------------------------
    mix("k3_ipb_14", 9, 5, 14, 14, [(7, 14, 14)], [cp(0, 7, 5, k=3)], ["conv_fwd_kernel<3>", "conv_wgrad_kernel<3>"]),
    mix("k3_ipb_7", 5, 20, 7, 7, [(6, 7, 7)], [cp(0, 6, 20, k=3)], ["conv_fwd_kernel<3>"]),
    mix("k3_band_37", 2, 6, 37, 40, [(4, 37, 40)], [cp(0, 4, 6, k=3)], ["conv_fwd_kernel<3>", "conv_wgrad_kernel<3>"]),
    mix("k3_chunk_lt_cin", 2, 8, 28, 28, [(96, 28, 28)], [cp(0, 96, 8, k=3)], ["conv_fwd_kernel<3>", "conv_wgrad_kernel<3>"]),
    mix("k3_wgrad_r0", 2, 8, 28, 28, [(128, 28, 28)], [cp(0, 128, 8, k=3)], ["conv_fwd_kernel<3>", "tr_mix_wgrad_kernel"]),
    mix("k3_tiles_over_256", 2, 40, 12, 16, [(40, 12, 16)], [cp(0, 40, 40, k=3)], ["conv_wgrad_kernel<3>"]),
    mix("k3_r_smem", 2, 32, 28, 56, [(32, 28, 56)], [cp(0, 32, 32, k=3)], ["conv_wgrad_kernel<3>"]),
    mix("k3_tiny_tiles_w30", 3, 5, 10, 30, [(6, 10, 30)], [cp(0, 6, 5, k=3)], ["conv_wgrad_kernel<3>"]),
    mix("dil_wide_plane", 1, 3, 4, 700, [(2, 4, 700)], [cp(0, 2, 3, k=3, dil=16)], ["tr_mix_fwd_kernel", "conv_wgrad_kernel<0>"]),
    mix("msblock_14", 2, 15, 14, 14, [(8, 14, 14)], [cp(0, 8, 3, k=3, dil=d, cout0=3 * i) for i, d in enumerate((1, 2, 4, 8, 16))],
        ["conv_fwd_kernel<0>", "conv_wgrad_kernel<0>", "conv_wgrad_kernel<3>"]),
    mix("dil8_7x7", 3, 4, 7, 7, [(5, 7, 7)], [cp(0, 5, 4, k=3, dil=8)], ["conv_fwd_kernel<0>", "conv_wgrad_kernel<0>"]),
    # ---- depthwise 3x3 -----------------------------------------------------------------------------------------------------------
    Case("dw_h5", "dw", dict(N=3, C=6, H=5, W=12), ("dw3_kernel", "dw3_wgrad_kernel", "dw3_bwd_kernel", "reduce_partials_kernel")),
    Case("dw_h13_w1", "dw", dict(N=2, C=5, H=13, W=1), ("dw3_kernel",)),
    Case("dw_w2", "dw", dict(N=2, C=4, H=9, W=2), ("dw3_kernel",)),
    Case("dw_w3", "dw", dict(N=2, C=4, H=16, W=3), ("dw3_kernel",)),
    Case("dw_w5", "dw", dict(N=2, C=4, H=11, W=5), ("dw3_kernel",)),
    Case("dw_cap_binds", "dw", dict(N=8, C=200, H=64, W=64), ("dw3_wgrad_kernel", "dw3_bwd_kernel")),
    Case("dw_c_over_8sms", "dw", dict(N=2, C=1100, H=8, W=8), ("dw3_wgrad_kernel", "dw3_bwd_kernel")),
    # ---- BatchNorm + PReLU ----------------------------------------------------------------------------------------------------------
    Case("bn_s1", "bn", dict(N=4, C=8, H=16, W=16, mode="normal"), ("bn_stats_kernel", "bn_prelu_fwd_kernel", "bn_prelu_bwd_reduce_kernel",
                                                                      "bn_prelu_bwd_apply_kernel")),
    Case("bn_segments_scalar", "bn", dict(N=2, C=4, H=130, W=130, mode="normal"), ("bn_stats_kernel",)),
    Case("bn_mean_1e4", "bn", dict(N=2, C=3, H=32, W=32, mode="big_mean"), ("bn_stats_kernel",)),
    Case("bn_const_channel", "bn", dict(N=2, C=5, H=12, W=20, mode="const"), ("bn_stats_kernel",)),
    Case("bn_n1", "bn", dict(N=1, C=5, H=64, W=64, mode="normal"), ("bn_stats_kernel",)),
    # ---- pooling -----------------------------------------------------------------------------------------------------------------------
    Case("pool2_vec", "pool", dict(N=2, Cs=5, c0=1, cin=3, Hs=8, Ws=16, pre_avg=0, pool=2, ints=True), ("pool2_fwd_kernel", "pool_bwd4_kernel")),
    Case("pool2_ws18", "pool", dict(N=2, Cs=4, c0=0, cin=4, Hs=8, Ws=18, pre_avg=0, pool=2, ints=True), ("pool_fwd_kernel", "pool_bwd_kernel")),
    Case("pool4_ragged", "pool", dict(N=2, Cs=6, c0=2, cin=3, Hs=19, Ws=21, pre_avg=0, pool=4, ints=True), ("pool_fwd_kernel", "pool_bwd_kernel")),
    Case("pool8_avg", "pool", dict(N=2, Cs=3, c0=0, cin=3, Hs=35, Ws=48, pre_avg=1, pool=8, ints=True), ("pool_fwd_kernel", "pool_bwd4_kernel")),
    Case("pool2_avg_real", "pool", dict(N=2, Cs=4, c0=1, cin=2, Hs=18, Ws=20, pre_avg=1, pool=2, ints=False), ("pool_fwd_kernel", "pool_bwd4_kernel")),
    Case("avg_only", "pool", dict(N=2, Cs=3, c0=0, cin=3, Hs=11, Ws=13, pre_avg=1, pool=1, ints=False), ("pool_fwd_kernel", "pool_bwd_kernel")),
    # ---- loss, optimiser ----------------------------------------------------------------------------------------------------------------
    Case("bce_small", "bce", dict(n=200, gs=1.0, zmax=100.0), ("bce_kernel",)),
    Case("bce_ragged", "bce", dict(n=5000, gs=0.37, zmax=8.0), ("bce_kernel",)),
    Case("bce_over_cap", "bce", dict(n=1184 * 2048 + 4133, gs=3.0, zmax=100.0), ("bce_kernel",)),
    Case("adam_5_steps", "adam", dict(sizes=(1, 2 * 2048 + 37, 300, 5000), wds=(5e-3, 0.0, 5e-3, 0.0), gs=(1.0, 0.5, 2.0, 1.0, 0.25)),
         ("adam_kernel",)),
]
BY_ID = {c.id: c for c in CASES}


def make_inputs(case):
    """CPU float32 inputs of a case (deterministic per case id)."""
    g = _gen(case.id)
    p = case.p
    if case.kind == "mix":
        srcs = [biased(g, (p["N"],) + tuple(s)) for s in p["srcs"]]
        ws = []
        for q in p["paths"]:
            k = q["ksize"]
            s = 1.0 / np.sqrt(max(1, q["cin"] * k * k))
            ws.append(((torch.rand((q["cin"], k * k, q["cout"]), generator=g, dtype=torch.float64) * 2 - 1) * s).float() if k else None)
        return dict(srcs=srcs, ws=ws, ddst=biased(g, (p["N"], p["C"], p["H"], p["W"])))
    if case.kind == "dw":
        shape = (p["N"], p["C"], p["H"], p["W"])
        return dict(x=biased(g, shape), dy=biased(g, shape), w=(0.01 * torch.randn((p["C"], 9), generator=g)).float(), scale=100.0)
    if case.kind == "bn":
        N, Cc, H, W = p["N"], p["C"], p["H"], p["W"]
        z = 2.0 * torch.randn((N, Cc, H, W), generator=g, dtype=torch.float64) + 0.3
        if p["mode"] == "big_mean":
            z = z * 0.5 + 1e4
        if p["mode"] == "const":
            z[:, 1] = 0.7
        slope = torch.tensor([-0.5, 1.5, 0.25, 0.0, 0.1, -1.2, 2.0, 0.3][:Cc] + [0.25] * max(0, Cc - 8), dtype=torch.float64)
        return dict(z=z.float(), dy=biased(g, (N, Cc, H, W), 0.2), gamma=(torch.rand(Cc, generator=g) + 0.5).float(),
                    beta=torch.randn(Cc, generator=g).float(), slope=slope.float(), eps=1e-5)
    if case.kind == "pool":
        shape = (p["N"], p["Cs"], p["Hs"], p["Ws"])
        if p["ints"]:
            src = torch.randint(-2, 3, shape, generator=g).float()
            src[:, :, : p["Hs"] // 2, : p["Ws"] // 3] = 0.0                 # a zero plateau
        else:
            src = biased(g, shape)
        f = (2 if p["pre_avg"] else 1) * p["pool"]
        return dict(src=src, dpool=biased(g, (p["N"], p["cin"], p["Hs"] // f, p["Ws"] // f)))
    if case.kind == "bce":
        n = p["n"]
        z = (torch.rand(n, generator=g, dtype=torch.float64) * 2 - 1) * p["zmax"]
        t = torch.rand(n, generator=g, dtype=torch.float64)
        t[: n // 3] = (t[: n // 3] > 0.5).double()                             # binary targets and fractional ones
        return dict(z=z.float(), t=t.float(), gs=p["gs"])
    if case.kind == "adam":
        params = [(0.1 * torch.randn(s, generator=g)).float() for s in p["sizes"]]
        grads = []
        for _ in p["gs"]:
            gl = []
            for s in p["sizes"]:
                v = (1e-3 * torch.randn(s, generator=g)).float()
                v[torch.rand(s, generator=g) < 0.1] = 0.0                      # zero-gradient elements
                gl.append(v)
            grads.append(gl)
        return dict(params=params, grads=grads)
    raise ValueError(case.kind)


def _paths(case, inp, dev=None):
    mv = (lambda t: t.to(dev)) if dev is not None else (lambda t: t)
    return [R.Path(src=mv(inp["srcs"][q["src"]]), w=mv(inp["ws"][i]) if inp["ws"][i] is not None else None, cin=q["cin"], cout=q["cout"],
                   c0=q["c0"], cout0=q["cout0"], ksize=q["ksize"], dil=q["dil"], stride=q["stride"], pad=q["pad"], up=q["up"])
            for i, q in enumerate(case.p["paths"])]


LR, BETAS, EPS = float(np.float32(1e-3)), (float(np.float32(0.9)), float(np.float32(0.99))), float(np.float32(1e-8))


def reference(case, inp, got=None, defect=None, sms=R.SMS):
    """{output name: (ref, bound)} of a case; `got` supplies the kernel outputs that later calls read (BatchNorm mean / var,
    the pool arg-max); without it the fp32-rounded references stand in."""
    p = case.p
    out = {}
    if case.kind == "mix":
        paths = _paths(case, inp)
        out["dst"] = R.mix_fwd(paths, p["C"], p["H"], p["W"], defect=defect)["dst"]
        for i, q in enumerate(paths):
            out[f"dsrc{i}"] = R.mix_dgrad(inp["ddst"], q, defect=defect)["dsrc"]
            if q.ksize:
                out[f"dw{i}"] = R.mix_wgrad(inp["ddst"], q, sms=sms, defect=defect)["dw"]
        return out
    if case.kind == "dw":
        out["y"] = R.dw_conv(inp["x"], inp["w"], inp["scale"], 0, defect=defect)["y"]
        out["dxT"] = R.dw_conv(inp["dy"], inp["w"], inp["scale"], 1, defect=defect)["y"]
        out["dw"] = R.dw_wgrad(inp["x"], inp["dy"], inp["scale"], sms=sms, defect=defect)["dw"]
        b = R.dw_bwd(inp["x"], inp["dy"], inp["w"], inp["scale"], sms=sms, defect=defect)
        out["bwd_dx"], out["bwd_dw"] = b["dx"], b["dw"]
        return out
    if case.kind == "bn":
        st = R.bn_stats(inp["z"], defect=defect)
        out["mean"], out["var"] = st["mean"], st["var"]
        mean = got["mean"] if got is not None else st["mean"][0].float()
        var = got["var"] if got is not None else st["var"][0].float()
        a = (inp["z"], mean, var, inp["gamma"], inp["beta"], inp["slope"], inp["eps"])
        f = R.bn_prelu_fwd(*a, defect=defect)
        out["y"], out["gap"] = f["y"], f["gap"]
        for fr in (0, 1):
            b = R.bn_prelu_bwd(inp["z"], inp["dy"], *a[1:], frozen=fr, defect=defect)
            for k, v in b.items():
                out[f"{k}{fr}"] = v
        return out
    if case.kind == "pool":
        r = R.pool_fwd(inp["src"], p["c0"], p["cin"], p["pre_avg"], p["pool"], defect=defect)
        out["dst"] = r["dst"]
        if p["pool"] > 1:
            out["idx"] = r["idx"]
        idx = got["idx"] if got is not None and p["pool"] > 1 else (r["idx"][0] if p["pool"] > 1 else None)
        out["dsrc"] = R.pool_bwd(inp["dpool"], idx, p["Hs"], p["Ws"], p["pre_avg"], p["pool"], defect=defect)["dsrc"]
        return out
    if case.kind == "bce":
        r = R.bce(inp["z"], inp["t"], inp["gs"], defect=defect)
        return {"loss": r["loss"], "dl": r["dlogits"]}
    if case.kind == "adam":
        res = R.adam(inp["params"], inp["grads"], p["wds"], LR, BETAS, EPS, p["gs"], defect=defect)
        return {f"p{i}": v for i, v in enumerate(res)}
    raise ValueError(case.kind)


# ---- running the C ABI -------------------------------------------------------------------------------------------------------
KRE = re.compile(r"(\w+_kernel)\s*(<[^>(]*>)?")


def kernel_names(events):
    out = set()
    for e in events:
        m = KRE.search(e.name)
        if m:
            out.add(m.group(1) + (m.group(2) or "").replace(" ", ""))
    return out


class Runner:
    """Guarded outputs and ABI calls."""

    def __init__(self):
        from sod100k_b200 import train_ops as T
        self.T, self.lib = T, T.lib()
        self.bufs, self.outs, self.kernels, self.no_repeat = [], {}, set(), set()

    def out(self, name, shape, dtype=torch.float32):
        n = int(np.prod(shape)) * torch.tensor([], dtype=dtype).element_size()
        buf = torch.full((GUARD + n + GUARD,), 0xFF, dtype=torch.uint8, device="cuda")
        self.bufs.append(buf)
        t = buf[GUARD:GUARD + n].view(dtype).view(shape)
        self.outs[name] = t
        return t

    def call(self, label, fn, *args):
        rc = getattr(self.lib, fn)(*args, torch.cuda.current_stream().cuda_stream)
        assert rc == 0, (label, fn, rc, self.lib.csnet_train_last_error().decode())

    def guards_intact(self):
        return all(bool((b[:GUARD] == 0xFF).all()) and bool((b[-GUARD:] == 0xFF).all()) for b in self.bufs)


def _ptr(t):
    return t.data_ptr() if t is not None else None


def launch(case, inp, trace):
    """Run a case's ABI calls on the GPU; returns the Runner (outputs, guards and, with `trace`, the kernels launched)."""
    rn = Runner()
    if not trace:
        _calls(rn, case, inp)
        torch.cuda.synchronize()
        return rn
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        _calls(rn, case, inp)
        torch.cuda.synchronize()
    rn.kernels = kernel_names(prof.events())
    if "tr_mix_wgrad_kernel" in rn.kernels:         # atomicAdd over image splits: its weight gradients are not bit-reproducible
        rn.no_repeat |= {k for k in rn.outs if k.startswith("dw")}
    return rn


def _calls(rn, case, inp):
    T = rn.T
    p = case.p
    cu = lambda t: t.cuda().contiguous()
    if case.kind == "mix":
        N, Cc, H, W = p["N"], p["C"], p["H"], p["W"]
        srcs = [cu(s) for s in inp["srcs"]]
        ws = [cu(w) if w is not None else None for w in inp["ws"]]
        ddst = cu(inp["ddst"])
        tp = [T.TrainPath(srcs[q["src"]].data_ptr(), _ptr(ws[i]), *srcs[q["src"]].shape[1:], q["c0"], q["cin"], 0, 1, q["ksize"], q["dil"],
                          q["stride"], q["pad"], q["up"], q["cout0"], q["cout"]) for i, q in enumerate(p["paths"])]
        dst = rn.out("dst", (N, Cc, H, W))
        rn.call("fwd", "csnet_train_mix_fwd", dst.data_ptr(), N, Cc, H, W, (T.TrainPath * len(tp))(*tp), len(tp))
        for i, q in enumerate(p["paths"]):
            s = srcs[q["src"]]
            d = rn.out(f"dsrc{i}", (N, q["cin"], s.shape[2], s.shape[3]))
            rn.call(f"dsrc{i}", "csnet_train_mix_dgrad", ddst.data_ptr(), N, Cc, H, W, C.byref(tp[i]), d.data_ptr())
            if q["ksize"]:
                dw = rn.out(f"dw{i}", tuple(ws[i].shape))
                rn.call(f"dw{i}", "csnet_train_mix_wgrad", ddst.data_ptr(), N, Cc, H, W, C.byref(tp[i]), dw.data_ptr())
    elif case.kind == "dw":
        N, Cc, H, W = p["N"], p["C"], p["H"], p["W"]
        x, dy, w, sc = cu(inp["x"]), cu(inp["dy"]), cu(inp["w"]), inp["scale"]
        y = rn.out("y", x.shape)
        rn.call("y", "csnet_train_dw_conv", x.data_ptr(), w.data_ptr(), y.data_ptr(), N, Cc, H, W, sc, 0)
        dxt = rn.out("dxT", x.shape)
        rn.call("dxT", "csnet_train_dw_conv", dy.data_ptr(), w.data_ptr(), dxt.data_ptr(), N, Cc, H, W, sc, 1)
        dw = rn.out("dw", (Cc, 9))
        rn.call("dw", "csnet_train_dw_wgrad", x.data_ptr(), dy.data_ptr(), dw.data_ptr(), N, Cc, H, W, sc)
        bdx, bdw = rn.out("bwd_dx", x.shape), rn.out("bwd_dw", (Cc, 9))
        rn.call("bwd", "csnet_train_dw_bwd", x.data_ptr(), dy.data_ptr(), w.data_ptr(), bdx.data_ptr(), bdw.data_ptr(), N, Cc, H, W, sc)
    elif case.kind == "bn":
        N, Cc, H, W = p["N"], p["C"], p["H"], p["W"]
        z, dy = cu(inp["z"]), cu(inp["dy"])
        g, b, a = cu(inp["gamma"]), cu(inp["beta"]), cu(inp["slope"])
        mean, var = rn.out("mean", (Cc,)), rn.out("var", (Cc,))
        rn.call("stats", "csnet_train_bn_stats", z.data_ptr(), N, Cc, H * W, mean.data_ptr(), var.data_ptr())
        y, gap = rn.out("y", z.shape), rn.out("gap", (N, Cc))
        rn.call("fwd", "csnet_train_bn_prelu_fwd", z.data_ptr(), y.data_ptr(), N, Cc, H * W, mean.data_ptr(), var.data_ptr(), g.data_ptr(),
                b.data_ptr(), a.data_ptr(), C.c_float(inp["eps"]), gap.data_ptr())
        for fr in (0, 1):
            dz = rn.out(f"dz{fr}", z.shape)
            dg, db, ds = (rn.out(f"{k}{fr}", (Cc,)) for k in ("dgamma", "dbeta", "dslope"))
            rn.call(f"bwd{fr}", "csnet_train_bn_prelu_bwd", z.data_ptr(), dy.data_ptr(), dz.data_ptr(), N, Cc, H * W, mean.data_ptr(),
                    var.data_ptr(), g.data_ptr(), b.data_ptr(), a.data_ptr(), C.c_float(inp["eps"]), dg.data_ptr(), db.data_ptr(), ds.data_ptr(), fr)
    elif case.kind == "pool":
        src, dpool = cu(inp["src"]), cu(inp["dpool"])
        f = (2 if p["pre_avg"] else 1) * p["pool"]
        shp = (p["N"], p["cin"], p["Hs"] // f, p["Ws"] // f)
        dst = rn.out("dst", shp)
        idx = rn.out("idx", shp, torch.uint8) if p["pool"] > 1 else None
        rn.call("fwd", "csnet_train_pool_fwd", src.data_ptr(), p["N"], p["Cs"], p["c0"], p["cin"], p["Hs"], p["Ws"], p["pre_avg"], p["pool"],
                dst.data_ptr(), _ptr(idx))
        dsrc = rn.out("dsrc", (p["N"], p["cin"], p["Hs"], p["Ws"]))
        rn.call("bwd", "csnet_train_pool_bwd", dpool.data_ptr(), _ptr(idx), p["N"], p["cin"], p["Hs"], p["Ws"], p["pre_avg"], p["pool"],
                dsrc.data_ptr())
    elif case.kind == "bce":
        z, t = cu(inp["z"]), cu(inp["t"])
        loss, dl = rn.out("loss", ()), rn.out("dl", z.shape)
        rn.call("bce", "csnet_train_bce", z.data_ptr(), t.data_ptr(), dl.data_ptr(), loss.data_ptr(), z.numel(), C.c_float(inp["gs"]))
        rn.no_repeat.add("loss")                       # atomicAdd over blocks
    elif case.kind == "adam":
        ps = [rn.out(f"p{i}", tuple(q.shape)) for i, q in enumerate(inp["params"])]
        for q, src in zip(ps, inp["params"]):
            q.copy_(src)
        gs = [torch.zeros_like(q) for q in ps]
        ms = [torch.zeros_like(q) for q in ps]
        vs = [torch.zeros_like(q) for q in ps]
        rec = np.dtype([("p", "<u8"), ("g", "<u8"), ("m", "<u8"), ("v", "<u8"), ("n", "<i4"), ("wd", "<f4")])
        rows = []
        for q, g_, m_, v_, wd in zip(ps, gs, ms, vs, p["wds"]):
            for o in range(0, q.numel(), 2048):
                k = min(2048, q.numel() - o)
                rows.append((q.data_ptr() + 4 * o, g_.data_ptr() + 4 * o, m_.data_ptr() + 4 * o, v_.data_ptr() + 4 * o, k, wd))
        tab = torch.from_numpy(np.array(rows, dtype=rec).view(np.uint8).copy()).cuda()
        for s, scale in enumerate(p["gs"]):
            for g_, src in zip(gs, inp["grads"][s]):
                g_.copy_(src)
            rn.call(f"step{s + 1}", "csnet_train_adam", tab.data_ptr(), len(rows), C.c_float(LR), C.c_float(BETAS[0]), C.c_float(BETAS[1]),
                    C.c_float(EPS), s + 1, C.c_float(scale))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


_KERNELS_SEEN = {}


def run_case(case):
    inp = make_inputs(case)
    for _ in range(3):                           # a trace can come back without its kernels' activity records: trace again
        a = launch(case, inp, trace=True)
        if set(case.targets) <= a.kernels:
            break
    b = launch(case, inp, trace=False)
    _KERNELS_SEEN[case.id] = a.kernels
    for k in case.targets:
        assert k in a.kernels, (case.id, k, sorted(a.kernels))
    assert a.guards_intact() and b.guards_intact(), (case.id, "guard band overwritten")
    for name, t in a.outs.items():
        if name in a.no_repeat:
            continue
        u, v = t.view(torch.uint8), b.outs[name].view(torch.uint8)
        assert torch.equal(u, v), (case.id, name, "not bit-identical across two runs")
    got = {k: v.cpu() for k, v in a.outs.items()}
    refs = reference(case, inp, got=got, sms=_sms())
    label = "+".join(sorted(case.targets))
    worst = 0.0
    for name, rb in refs.items():
        if name == "idx":
            bad = R.check_idx(got["idx"], *rb)
            _note(label, f"{case.id}/idx", float(bad))
            assert bad == 0, (case.id, "arg-max not the first admissible maximum in", bad, "windows")
            continue
        q, msg = R.check(got[name], *rb)
        _note(label, f"{case.id}/{name}", q)
        assert q <= 1.0, (case.id, name, msg)
        worst = max(worst, q)
    return worst


# ---- (a) ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case_id", list(BY_ID))
def test_training_kernel_matches_float64(case_id):
    run_case(BY_ID[case_id])


# ---- (b) ---------------------------------------------------------------------------------------------------------------------
def source_kernels():
    """Every kernel instantiation the two sources launch (`name<args><<<`), and every __global__ they define."""
    launched, defined = set(), set()
    for path in SOURCES:
        src = open(path).read()
        for m in re.finditer(r"(\w+_kernel)\s*(<[^<>]*>)?\s*<<<", src):
            launched.add(m.group(1) + (m.group(2) or "").replace(" ", ""))
        for m in re.finditer(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(", src):
            defined.add(m.group(1))
    return launched, defined


def test_every_training_kernel_is_reached():
    launched, defined = source_kernels()
    assert defined <= {k.split("<")[0] for k in launched}, sorted(defined - {k.split("<")[0] for k in launched})
    seen = set()
    for c in CASES:
        if c.id not in _KERNELS_SEEN:
            run_case(c)
        seen |= _KERNELS_SEEN[c.id]
    missing = sorted(k for k in launched if k not in seen and k not in EXEMPT)
    print("training kernels reached:", sorted(k for k in launched if k in seen))
    assert not missing, missing


# ---- (c) the bench step, op by op ----------------------------------------------------------------------------------------------
class Certifier:
    """Checks every wrapped call against trainref on that call's own inputs; keeps the worst q per entry point."""

    def __init__(self, sms):
        self.sms, self.worst = sms, collections.defaultdict(float)
        self.calls, self.skipped = collections.Counter(), collections.Counter()

    def check(self, entry, got, ref, bound, count=True):
        """count: the first piece of a call checked in pieces (images or channels) counts the call."""
        q, msg = R.check(got, ref, bound)
        self.worst[entry] = max(self.worst[entry], q)
        self.calls[entry] += int(count)
        assert q <= 1.0, (entry, msg)


def _install(monkeypatch, cert):
    from sod100k_b200 import train_ops as T

    mix_f, mix_b = T.MixFn.forward, T.MixFn.backward
    dw_f, dw_b = T.DwFn.forward, T.DwFn.backward
    bn_f, bn_b = T.BnPreluFn.forward, T.BnPreluFn.backward
    bce_f, bce_b = T.BceFn.forward, T.BceFn.backward
    adam_step = T.FusedAdam.step

    def rpath(q, tensors, shape_src=None):
        return R.Path(src=tensors[q.src], w=tensors[q.w] if q.w is not None else None, cin=q.cin, cout=q.cout, c0=q.c0, cout0=q.cout0,
                      ksize=q.ksize, dil=q.dil, stride=q.stride, pad=q.pad, up=q.up)

    def pooled(p, s):
        """The pooled source a path reads (recomputed with the same kernel: deterministic) and its certification."""
        n = s.shape[0]
        f = (2 if p.pre_avg else 1) * p.pool
        xp = torch.empty((n, p.cin, s.shape[2] // f, s.shape[3] // f), dtype=torch.float32, device=s.device)
        idx = torch.empty(xp.shape, dtype=torch.uint8, device=s.device) if p.pool > 1 else None
        st = torch.cuda.current_stream().cuda_stream
        assert T.lib().csnet_train_pool_fwd(s.data_ptr(), n, s.shape[1], p.c0, p.cin, s.shape[2], s.shape[3], p.pre_avg, p.pool, xp.data_ptr(),
                                            _ptr(idx), st) == 0
        r = R.pool_fwd(s, p.c0, p.cin, p.pre_avg, p.pool)
        cert.check("pool_fwd", xp, *r["dst"])
        if idx is not None:
            bad = R.idx_violations(idx, *r["idx"])
            assert bad == (0, 0), ("pool_fwd idx (not admissible, after the first maximum)", bad, tuple(s.shape), p.pre_avg, p.pool)
        return xp, idx

    def mix_forward(ctx, spec, *tensors):
        dst = mix_f(ctx, spec, *tensors)
        with torch.no_grad():
            out_c, out_h, out_w, paths = spec
            ts = [t.detach().float().contiguous() for t in tensors]
            rp = []
            for p in paths:
                if p.ksize > 0 and (p.pre_avg or p.pool > 1):
                    xp, _ = pooled(p, ts[p.src])
                    q = rpath(p, ts)
                    q.src, q.c0 = xp, 0
                    rp.append(q)
                else:
                    rp.append(rpath(p, ts))
            cert.check("mix_fwd", dst, *R.mix_fwd(rp, out_c, out_h, out_w)["dst"])
        return dst

    def dgrad_ref(ctx, saved, dd, ks, j, a, b):
        """Reference of the gradient MixFn returns for its tensor input j, images [a, b): the sum over the paths ks reading it
        of each path's data gradient (a pooled path's routed through pool_bwd with the saved arg-max), placed at its channel
        slice; the bounds add, plus u |partial sum| for each fp32 add of the backward's accumulation."""
        paths = ctx.spec[3]
        shp = ctx.shapes[j]
        v = torch.zeros((b - a,) + tuple(shp[1:]), dtype=torch.float64, device=dd.device)
        bnd, mag = torch.zeros_like(v), torch.zeros_like(v)
        for k in ks:
            p, q = paths[k], ctx.dense[k]
            rq = rpath(q, saved)
            rq.src = rq.src[a:b]
            rv, rb = R.mix_dgrad(dd[a:b], rq)["dsrc"]
            if k in ctx.pooled:
                idx = saved[ctx.pooled[k][1]]
                idx = idx[a:b] if idx is not None else None
                route = lambda t: R.pool_bwd(t, idx, shp[2], shp[3], p.pre_avg, p.pool)["dsrc"][0]
                rv, rb = route(rv), route(rb) + R.TINY
            sl = slice(p.c0, p.c0 + p.cin)
            v[:, sl] += rv
            bnd[:, sl] += rb
            mag[:, sl] += rv.abs() + rb
        return v, bnd + (len(ks) - 1) * R.U * mag

    def mix_backward(ctx, ddst):
        grads = mix_b(ctx, ddst)
        with torch.no_grad():
            paths = ctx.spec[3]
            saved = ctx.saved_tensors
            dd = ddst.float().contiguous()
            N = dd.shape[0]
            for j in range(ctx.n_in):
                g = grads[1 + j]
                if g is None:
                    continue
                srcs = [k for k, p in enumerate(paths) if p.src == j]
                wts = [k for k, p in enumerate(paths) if p.w == j]
                if srcs:
                    entry = "mix_dgrad+pool_bwd" if any(k in ctx.pooled for k in srcs) else "mix_dgrad"
                    per = max(1, (1 << 24) // max(1, int(np.prod(ctx.shapes[j][1:]))))      # images per reference chunk
                    for a in range(0, N, per):
                        b = min(N, a + per)
                        cert.check(entry, g[a:b], *dgrad_ref(ctx, saved, dd, srcs, j, a, b), count=a == 0)
                elif wts:
                    v = bnd = mag = 0.0
                    for k in wts:
                        rv, rb = R.mix_wgrad(dd, rpath(ctx.dense[k], saved), sms=cert.sms)["dw"]
                        v, bnd, mag = v + rv, bnd + rb, mag + rv.abs() + rb
                    cert.check("mix_wgrad", g, v, bnd + (len(wts) - 1) * R.U * mag)
                else:
                    cert.skipped["MixFn.backward"] += 1
        return grads

    def dw_forward(ctx, x, w, scale):
        y = dw_f(ctx, x, w, scale)
        with torch.no_grad():
            cert.check("dw_conv", y, *R.dw_conv(x, w.reshape(-1, 9), scale, 0)["y"])
        return y

    def dw_backward(ctx, dy):
        dx, dw, _ = dw_b(ctx, dy)
        with torch.no_grad():
            x, wf = ctx.saved_tensors
            dyf = dy.float().contiguous()
            if dx is not None and dw is not None:
                r = R.dw_bwd(x, dyf, wf, ctx.scale, sms=cert.sms)
                cert.check("dw_bwd.dx", dx, *r["dx"])
                cert.check("dw_bwd.dw", dw.reshape(-1, 9), *r["dw"])
            elif dx is not None:
                cert.check("dw_conv(T)", dx, *R.dw_conv(dyf, wf, ctx.scale, 1)["y"])
            elif dw is not None:
                cert.check("dw_wgrad", dw.reshape(-1, 9), *R.dw_wgrad(x, dyf, ctx.scale, sms=cert.sms)["dw"])
        return dx, dw, None

    def channel_chunks(z):
        """BatchNorm is per channel: the references run on a few channels at a time to bound their memory at batch 256."""
        per = max(1, (1 << 25) // max(1, z.shape[0] * z[0, 0].numel()))
        return [slice(c, min(z.shape[1], c + per)) for c in range(0, z.shape[1], per)]

    def bn_forward(ctx, z, gamma, beta, slope, frozen_mean=None, frozen_var=None):
        y, mean, var, gap = bn_f(ctx, z, gamma, beta, slope, frozen_mean, frozen_var)
        with torch.no_grad():
            for c in channel_chunks(z):
                one = c.start == 0
                if frozen_mean is None:
                    st = R.bn_stats(z[:, c])
                    cert.check("bn_stats.mean", mean[c], *st["mean"], count=one)
                    cert.check("bn_stats.var", var[c], *st["var"], count=one)
                r = R.bn_prelu_fwd(z[:, c], mean[c], var[c], gamma[c], beta[c], slope[c], T.BN_EPS)
                cert.check("bn_prelu_fwd.y", y[:, c], *r["y"], count=one)
                cert.check("bn_prelu_fwd.gap", gap[:, c], *r["gap"], count=one)
        return y, mean, var, gap

    def bn_backward(ctx, dy, dm, dv, dg):
        out = bn_b(ctx, dy, dm, dv, dg)
        with torch.no_grad():
            z, mean, var, g, b, a = ctx.saved_tensors
            dyf = dy.float().contiguous()
            parts = R.bn_parts_max(z.shape[0], z.shape[1])
            tag = "bn_prelu_bwd" + ("(frozen)" if ctx.frozen else "")
            for c in channel_chunks(z):
                r = R.bn_prelu_bwd(z[:, c], dyf[:, c], mean[c], var[c], g[c], b[c], a[c], T.BN_EPS, int(ctx.frozen), parts=parts)
                cert.check(f"{tag}.dz", out[0][:, c], *r["dz"], count=c.start == 0)
                for name, got in zip(("dgamma", "dbeta", "dslope"), out[1:4]):
                    cert.check(f"{tag}.{name}", got[c], *r[name], count=c.start == 0)
        return out

    def bce_forward(ctx, logits, target):
        loss = bce_f(ctx, logits, target)
        with torch.no_grad():
            r = R.bce(logits, target, 1.0)
            cert.check("bce.loss", loss, *r["loss"])
            ctx.cert_dlogits = r["dlogits"]
        return loss

    def bce_backward(ctx, g):
        (dl,) = ctx.saved_tensors
        cert.check("bce.dlogits", dl, *ctx.cert_dlogits)
        del ctx.cert_dlogits
        return bce_b(ctx, g)

    def adam(self, grad_scale=1.0):
        assert self.step_count == 0, "the certified step starts from a fresh optimiser"
        before = [p.detach().clone() for p, _ in self.params]
        grads = [p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p) for p, _ in self.params]
        r = adam_step(self, grad_scale)
        with torch.no_grad():
            f = lambda v: float(np.float32(v))
            res = R.adam(before, [grads], [wd for _, wd in self.params], f(self.lr), (f(self.betas[0]), f(self.betas[1])), f(self.eps),
                         [grad_scale])
            for (p, _), (ref, bound) in zip(self.params, res):
                cert.check("adam", p, ref, bound)
        return r

    monkeypatch.setattr(T.MixFn, "forward", staticmethod(mix_forward))
    monkeypatch.setattr(T.MixFn, "backward", staticmethod(mix_backward))
    monkeypatch.setattr(T.DwFn, "forward", staticmethod(dw_forward))
    monkeypatch.setattr(T.DwFn, "backward", staticmethod(dw_backward))
    monkeypatch.setattr(T.BnPreluFn, "forward", staticmethod(bn_forward))
    monkeypatch.setattr(T.BnPreluFn, "backward", staticmethod(bn_backward))
    monkeypatch.setattr(T.BceFn, "forward", staticmethod(bce_forward))
    monkeypatch.setattr(T.BceFn, "backward", staticmethod(bce_backward))
    monkeypatch.setattr(T.FusedAdam, "step", adam)


@pytest.mark.parametrize("n,hw", [(256, 224), (2, 64)], ids=["bench_b256_224", "b2_64"])
def test_trainer_step_certified_op_by_op(monkeypatch, n, hw):
    from sod100k_b200 import synth
    from sod100k_b200.model import csnet
    from sod100k_b200.trainer import Trainer
    from tests import fixtures

    cfg, sd = fixtures.checkpoint("csnet-L-x2")
    m = csnet.CSNet(cfg)
    m.load_state_dict(sd)
    m.cuda().train()
    tr = Trainer(m, lr=1e-4, weight_decay=5e-3, flops_weight=3.0, flops_expand=1.0)
    x = torch.from_numpy(synth.randn_images(n, hw, hw, 81)).cuda()
    t = torch.from_numpy(synth.random_masks(n, hw, hw, 82)).cuda()
    cert = Certifier(_sms())
    _install(monkeypatch, cert)
    tr.step(x, t)
    torch.cuda.synchronize()
    for entry in sorted(cert.worst):
        _note(entry, f"trainer_step/b{n}_{hw}/calls={cert.calls[entry]}", cert.worst[entry])
    print("calls checked:", dict(cert.calls), "skipped:", dict(cert.skipped))
    assert not cert.skipped, cert.skipped
    for entry in ("mix_fwd", "mix_dgrad", "mix_dgrad+pool_bwd", "mix_wgrad", "pool_fwd", "dw_conv", "dw_bwd.dx", "dw_bwd.dw", "bn_stats.mean",
                  "bn_stats.var", "bn_prelu_fwd.y", "bn_prelu_fwd.gap", "bn_prelu_bwd.dz", "bn_prelu_bwd.dgamma", "bce.loss", "bce.dlogits",
                  "adam"):
        assert cert.calls[entry] > 0, entry


# ---- (d) whole-net frozen BatchNorm ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("freeze", [False, True], ids=["all_params", "some_frozen"])
def test_frozen_batchnorm_gradients_match_float64(freeze, monkeypatch):
    from oracle import csnet_oracle as O
    from sod100k_b200 import synth, train_ops as T
    from sod100k_b200.model import csnet
    from tests import fixtures
    from tests.test_gpu_train import _check_grads

    cfg, sd = fixtures.checkpoint("csnet-L-x2")
    m = csnet.CSNet(cfg)
    m.load_state_dict(sd)
    m.cuda().eval()
    m.frozen_bn_training = True
    frozen = set()
    if freeze:
        # the stem's 3x3 conv, BatchNorms and PReLUs frozen: the first depthwise layer's input needs no gradient (DwFn runs
        # dw_wgrad alone); every other depthwise weight frozen: those layers run the transposed dw_conv alone
        for name, p in m.named_parameters():
            if name.startswith("stage0.0.conv1x1.") or (p.dim() == 4 and p.shape[1] == 1 and not name.startswith("stage0.0.conv3x3_1.")):
                p.requires_grad_(False)
                frozen.add(name)
    stats0 = {k: v.detach().clone() for k, v in m.state_dict().items() if "running" in k or "num_batches" in k}
    seen = collections.Counter()
    dw_b, bn_b = T.DwFn.backward, T.BnPreluFn.backward

    def dw_backward(ctx, dy):
        need_x, need_w = ctx.needs_input_grad[:2]
        seen["dw_both" if need_x and need_w else ("dw_dgrad_only" if need_x else "dw_wgrad_only")] += 1
        return dw_b(ctx, dy)

    def bn_backward(ctx, *a):
        seen["bn_frozen" if ctx.frozen else "bn_batch"] += 1
        return bn_b(ctx, *a)

    monkeypatch.setattr(T.DwFn, "backward", staticmethod(dw_backward))
    monkeypatch.setattr(T.BnPreluFn, "backward", staticmethod(bn_backward))
    n, hw = 2, 64
    x = synth.randn_images(n, hw, hw, 91)
    gy = torch.from_numpy(synth.randn_images(n, hw, hw, 92)[:, :1].copy())
    out = m(torch.from_numpy(x).cuda())
    out.backward(gy.cuda())
    assert seen["bn_frozen"] > 0 and seen["bn_batch"] == 0, seen
    if freeze:
        assert seen["dw_wgrad_only"] > 0 and seen["dw_dgrad_only"] > 0, seen
    for k, v in m.state_dict().items():
        if k in stats0:
            assert torch.equal(v, stats0[k]), k
    # float64 autograd of the oracle's eval-mode forward (and the fp32 oracle, the yardstick of each tensor's conditioning)
    params = {k: v for k, v in sd.items() if k in dict(m.named_parameters())}

    def oracle_grads(dt):
        leaves = {k: v.to(dt).clone().requires_grad_(k not in frozen) for k, v in params.items()}
        sdd = {k: (v.to(dt) if v.dtype.is_floating_point else v) for k, v in sd.items()}
        sdd.update(leaves)
        y = O.csnet_forward(cfg, sdd, torch.from_numpy(x).to(dt), training=False)
        y.backward(gy.to(dt))
        return {k: (v.grad if v.grad is not None else torch.zeros_like(v)).detach() for k, v in leaves.items()}

    g64, g32 = oracle_grads(torch.float64), oracle_grads(torch.float32)

    class Trainable:                              # _check_grads walks named_parameters(); frozen tensors have no gradient
        def named_parameters(self):
            return [(k, p) for k, p in m.named_parameters() if p.requires_grad]

    for name, p in m.named_parameters():
        assert (p.grad is None) == (name in frozen), name
    _check_grads(Trainable(), g32, g64)
