"""bf16 activation storage of the CSNet training step (sod100k_b200/csrc/train_bf16.cu, Trainer(storage="bf16")) on the GPU.

1. Kernel by kernel: every `csnet_train_*_bf16` entry point runs the fp32 suite's cases (tests/test_gpu_train_kernels_vs_float64.py)
   on those cases' inputs rounded to bf16, against trainref's float64 reference on the same values, with the bounds of the
   bf16-stored outputs widened by one rounding to nearest even (tests/trainref_bf16.py).  The mixes also run with an fp32
   source side (the stem) and an fp32 destination side (cls_layer).  Outputs are guarded, every case runs twice and must give
   identical bits, and a shape the tiled kernels do not take must return CSNET_E_UNSUPPORTED.
2. Reach: every __global__ defined in train_bf16.cu is launched there, and every instance it launches is reached by (1)'s
   cases, traced together in one profiler session.
3. One Trainer(storage="bf16") step certified op by op at the bench configuration and at batch 2, 64^2.
4. Storage: what the step saves for backward is bf16 except what the policy keeps fp32, and no ATen copy converts an
   activation between bf16 and fp32.
5. Determinism and recompute: the same bits twice, and with ILBlock recompute, from less saved memory.
6. Training still works: 20 steps from the shipped checkpoint track the fp32 Trainer's loss within 1 %.

Every check prints `TRAINREF_Q <kernel> <case> <q>` (pytest -s)."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from tests import trainref as R
from tests import trainref_bf16 as RB
from tests.test_gpu_train_kernels_vs_float64 import (BY_ID, CASES, Certifier, Runner, _install, _note, _ptr, _sms, kernel_names, make_inputs,
                                                     reference)

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _release_cached_memory():
    """The step tests below reserve tens of GB (batch 256 at 224^2 with float64 references): hand the cache back after each test,
    so the tests that follow (and the profiler's own device buffers) find free memory."""
    yield
    import gc

    gc.collect()
    torch.cuda.empty_cache()

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCE = os.path.join(ROOT, "sod100k_b200", "csrc", "train_bf16.cu")
E_UNSUPPORTED = -4
F32, BF16 = 0, 2
BF = "__nv_bfloat16"
TORCH = {F32: torch.float32, BF16: torch.bfloat16}

# (source side, destination side) of a mix: both bf16; the stem's fp32 input; cls_layer's fp32 logits
IOS = {"bb": (BF16, BF16), "fb": (F32, BF16), "bf": (BF16, F32)}
MIXED_IDS = ["c1_narrow", "c1_wide_vec4", "c1_w14", "c1_w7", "k3_ipb_14", "dil8_7x7"]
# calls the tiled kernels do not take (the fp32 entry points run the generic tr_mix_* kernels there)
UNSUPPORTED = {
    "gen_w_tile_96k": {"dst", "dsrc0"}, "gen_w_over_1024": {"dst", "dsrc0"}, "gen_mixed_k": {"dst"}, "gen_6_conv_paths": {"dst"},
    "gen_4_resample": {"dst", "dsrc2"}, "stride2": {"dst", "dsrc0", "dw0"}, "stride2_odd": {"dst", "dsrc0", "dw0"},
    "k1_dil2_wgrad": {"dw0"}, "resample_up8": {"dsrc0"}, "k5": {"dw0"},
}
# an fp32 destination (cls_layer) is taken for 1x1 mixes only: the fp32-side 3x3 calls
UNSUPPORTED_MIXED = {("fb", "k3_ipb_14"): {"dsrc0"}, ("fb", "dil8_7x7"): {"dsrc0"}, ("bf", "k3_ipb_14"): {"dst"}, ("bf", "dil8_7x7"): {"dst"}}

BF16_CASES = [(c.id, "bb") for c in CASES if c.kind in ("mix", "dw", "bn", "pool")] + [(cid, io) for io in ("fb", "bf") for cid in MIXED_IDS]


def _unsupported(case_id, io):
    return (UNSUPPORTED.get(case_id, set()) if io == "bb" else set()) | UNSUPPORTED_MIXED.get((io, case_id), set())


def _to(t, dt):
    return t.to(TORCH[dt]).cuda().contiguous()


def _calls(rn, case, inp, io, refused):
    """The bf16 entry points on one case; `refused` collects the outputs whose call returned CSNET_E_UNSUPPORTED."""
    T = rn.T
    p = case.p
    st = lambda: torch.cuda.current_stream().cuda_stream

    def call(label, fn, *args, may_refuse=False):
        rc = getattr(rn.lib, fn)(*args, st())
        if rc == E_UNSUPPORTED and may_refuse:
            refused.add(label)
            return
        assert rc == 0, (case.id, io, label, fn, rc, rn.lib.csnet_train_last_error().decode())

    if case.kind == "mix":
        sd, dd_t = IOS[io]
        N, Cc, H, W = p["N"], p["C"], p["H"], p["W"]
        srcs = [_to(s, sd) for s in inp["srcs"]]
        ws = [w.cuda().contiguous() if w is not None else None for w in inp["ws"]]
        ddst = _to(inp["ddst"], dd_t)
        tp = [T.TrainPath(srcs[q["src"]].data_ptr(), _ptr(ws[i]), *srcs[q["src"]].shape[1:], q["c0"], q["cin"], 0, 1, q["ksize"], q["dil"],
                          q["stride"], q["pad"], q["up"], q["cout0"], q["cout"]) for i, q in enumerate(p["paths"])]
        dst = rn.out("dst", (N, Cc, H, W), TORCH[dd_t])
        call("dst", "csnet_train_mix_fwd_bf16", dst.data_ptr(), dd_t, N, Cc, H, W, (T.TrainPath * len(tp))(*tp), len(tp), sd, may_refuse=True)
        for i, q in enumerate(p["paths"]):
            s = srcs[q["src"]]
            d = rn.out(f"dsrc{i}", (N, q["cin"], s.shape[2], s.shape[3]), TORCH[sd])
            call(f"dsrc{i}", "csnet_train_mix_dgrad_bf16", ddst.data_ptr(), dd_t, N, Cc, H, W, C.byref(tp[i]), d.data_ptr(), sd, may_refuse=True)
            if q["ksize"]:
                dw = rn.out(f"dw{i}", tuple(ws[i].shape))
                call(f"dw{i}", "csnet_train_mix_wgrad_bf16", ddst.data_ptr(), dd_t, N, Cc, H, W, C.byref(tp[i]), dw.data_ptr(), sd, may_refuse=True)
    elif case.kind == "dw":
        N, Cc, H, W = p["N"], p["C"], p["H"], p["W"]
        x, dy, w, sc = _to(inp["x"], BF16), _to(inp["dy"], BF16), inp["w"].cuda(), inp["scale"]
        y = rn.out("y", x.shape, torch.bfloat16)
        call("y", "csnet_train_dw_conv_bf16", x.data_ptr(), w.data_ptr(), y.data_ptr(), N, Cc, H, W, C.c_float(sc), 0)
        dxt = rn.out("dxT", x.shape, torch.bfloat16)
        call("dxT", "csnet_train_dw_conv_bf16", dy.data_ptr(), w.data_ptr(), dxt.data_ptr(), N, Cc, H, W, C.c_float(sc), 1)
        dw = rn.out("dw", (Cc, 9))
        call("dw", "csnet_train_dw_wgrad_bf16", x.data_ptr(), dy.data_ptr(), dw.data_ptr(), N, Cc, H, W, C.c_float(sc))
        bdx, bdw = rn.out("bwd_dx", x.shape, torch.bfloat16), rn.out("bwd_dw", (Cc, 9))
        call("bwd", "csnet_train_dw_bwd_bf16", x.data_ptr(), dy.data_ptr(), w.data_ptr(), bdx.data_ptr(), bdw.data_ptr(), N, Cc, H, W, C.c_float(sc))
    elif case.kind == "bn":
        N, Cc, H, W = p["N"], p["C"], p["H"], p["W"]
        z, dy = _to(inp["z"], BF16), _to(inp["dy"], BF16)
        g, b, a = inp["gamma"].cuda(), inp["beta"].cuda(), inp["slope"].cuda()
        mean, var = rn.out("mean", (Cc,)), rn.out("var", (Cc,))
        call("stats", "csnet_train_bn_stats_bf16", z.data_ptr(), N, Cc, H * W, mean.data_ptr(), var.data_ptr())
        y, gap = rn.out("y", z.shape, torch.bfloat16), rn.out("gap", (N, Cc))
        call("fwd", "csnet_train_bn_prelu_fwd_bf16", z.data_ptr(), y.data_ptr(), N, Cc, H * W, mean.data_ptr(), var.data_ptr(), g.data_ptr(),
             b.data_ptr(), a.data_ptr(), C.c_float(inp["eps"]), gap.data_ptr())
        for fr in (0, 1):
            dz = rn.out(f"dz{fr}", z.shape, torch.bfloat16)
            dg, db, ds = (rn.out(f"{k}{fr}", (Cc,)) for k in ("dgamma", "dbeta", "dslope"))
            call(f"bwd{fr}", "csnet_train_bn_prelu_bwd_bf16", z.data_ptr(), dy.data_ptr(), dz.data_ptr(), N, Cc, H * W, mean.data_ptr(),
                 var.data_ptr(), g.data_ptr(), b.data_ptr(), a.data_ptr(), C.c_float(inp["eps"]), dg.data_ptr(), db.data_ptr(), ds.data_ptr(), fr)
    elif case.kind == "pool":
        src, dpool = _to(inp["src"], BF16), _to(inp["dpool"], BF16)
        f = (2 if p["pre_avg"] else 1) * p["pool"]
        shp = (p["N"], p["cin"], p["Hs"] // f, p["Ws"] // f)
        dst = rn.out("dst", shp, torch.bfloat16)
        idx = rn.out("idx", shp, torch.uint8) if p["pool"] > 1 else None
        call("fwd", "csnet_train_pool_fwd_bf16", src.data_ptr(), p["N"], p["Cs"], p["c0"], p["cin"], p["Hs"], p["Ws"], p["pre_avg"], p["pool"],
             dst.data_ptr(), _ptr(idx))
        dsrc = rn.out("dsrc", (p["N"], p["cin"], p["Hs"], p["Ws"]), torch.bfloat16)
        call("bwd", "csnet_train_pool_bwd_bf16", dpool.data_ptr(), _ptr(idx), p["N"], p["cin"], p["Hs"], p["Ws"], p["pre_avg"], p["pool"],
             dsrc.data_ptr())


def _inputs(case, io):
    sd, dd_t = IOS[io] if case.kind == "mix" else (BF16, BF16)
    sides = tuple(n for n, d in (("srcs", sd), ("ddst", dd_t)) if d == BF16)
    return RB.bf16_inputs(case.kind, make_inputs(case), sides), sd, dd_t


def _launch(case, inp, io):
    rn, refused = Runner(), set()
    _calls(rn, case, inp, io, refused)
    torch.cuda.synchronize()
    return rn, refused


def run_case(case_id, io):
    case = BY_ID[case_id]
    inp, sd, dd_t = _inputs(case, io)
    a, refused = _launch(case, inp, io)
    b, refused_b = _launch(case, inp, io)
    expect = _unsupported(case_id, io)
    assert refused == expect and refused_b == expect, (case_id, io, "CSNET_E_UNSUPPORTED from", sorted(refused), "expected", sorted(expect))
    assert a.guards_intact() and b.guards_intact(), (case_id, io, "guard band overwritten")
    for name, t in a.outs.items():
        if name in refused:
            continue
        assert torch.equal(t.view(torch.uint8), b.outs[name].view(torch.uint8)), (case_id, io, name, "not bit-identical across two runs")
    got = {k: v.cpu() for k, v in a.outs.items()}
    refs = RB.widen_refs(case.kind, reference(case, inp, got=got, sms=_sms()), bf16_dst=dd_t == BF16, bf16_src=sd == BF16)
    label = f"{case.kind}_bf16[{io}]"
    for name, rb in refs.items():
        if name in refused:
            continue
        if name == "idx":
            bad = R.check_idx(got["idx"], *rb)
            assert bad == 0, (case_id, "arg-max not the first admissible maximum in", bad, "windows")
            continue
        q, msg = R.check(got[name], *rb)
        _note(label, f"{case_id}/{name}", q)
        assert q <= 1.0, (case_id, io, name, msg)


# ---- 1 -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case_id,io", BF16_CASES, ids=[f"{c}-{io}" for c, io in BF16_CASES])
def test_bf16_kernel_matches_float64(case_id, io):
    run_case(case_id, io)


# ---- 2 -----------------------------------------------------------------------------------------------------------------------
# the (TI, TO / TD) pairs each templated launcher of train_bf16.cu is instantiated with
PAIRS = {"conv1x1_bf16_kernel": [(BF, BF), ("float", BF), (BF, "float")], "conv1x1_narrow_bf16_kernel": [(BF, BF), ("float", BF), (BF, "float")],
         "conv_fwd_bf16_kernel": [(BF, BF), ("float", BF)], "conv_wgrad_bf16_kernel": [(BF, BF), ("float", BF), (BF, "float")]}


def source_kernels():
    """Every kernel instance train_bf16.cu launches (its TI / TO / TD placeholders expanded over PAIRS) and every __global__ it defines."""
    src = open(SOURCE).read()
    launched, defined = set(), set()
    for m in re.finditer(r"(\w+_kernel)\s*(<[^<>]*>)?\s*<<<", src):
        name, args = m.group(1), (m.group(2) or "").replace(" ", "")
        if re.search(r"\bT[IOD]\b", args):
            for ti, to in PAIRS[name]:
                launched.add(name + re.sub(r"\bT[OD]\b", to, re.sub(r"\bTI\b", ti, args)))
        else:
            launched.add(name + args)
    for m in re.finditer(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(", src):
        defined.add(m.group(1))
    return launched, defined


def test_every_bf16_kernel_is_reached():
    launched, defined = source_kernels()
    assert defined <= {k.split("<")[0] for k in launched}, sorted(defined - {k.split("<")[0] for k in launched})
    assert len(launched) == 38, sorted(launched)
    # every case's launches in ONE profiler session (the outputs are checked by the cases above); a trace can come back without
    # some of its kernels' activity records, so a kernel missing from it is looked for in up to two more sessions
    seen = set()
    for _ in range(3):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for cid, io in BF16_CASES:
                _launch(BY_ID[cid], _inputs(BY_ID[cid], io)[0], io)
        seen |= kernel_names(prof.events())
        if all(k in seen for k in launched):
            break
        print("not in the trace yet:", sorted(k for k in launched if k not in seen))
    missing = sorted(k for k in launched if k not in seen)
    assert not missing, missing
    print("bf16 kernels reached:", sorted(k for k in launched if k in seen))


# ---- 3 -----------------------------------------------------------------------------------------------------------------------
class Bf16Certifier(Certifier):
    """Certifier whose bound of an output stored in bf16 is widened by its rounding (unless the caller's bound has it)."""

    def check(self, entry, got, ref, bound, count=True, complete=False):
        if got.dtype == torch.bfloat16 and not complete:
            bound = RB.widen(ref, bound)
        super().check(entry, got, ref, bound, count)


def _install_bf16(monkeypatch, cert):
    """The fp32 suite's op-by-op wrappers (they read bf16 inputs exactly and the certifier widens bf16 outputs), with MixFn's
    replaced: its pooled copies are bf16 for bf16 sources, and its summed data gradients round at every bf16 add."""
    from sod100k_b200 import train_ops as T

    mix_f, mix_b = T.MixFn.forward, T.MixFn.backward
    _install(monkeypatch, cert)

    def rpath(q, tensors):
        return R.Path(src=tensors[q.src], w=tensors[q.w] if q.w is not None else None, cin=q.cin, cout=q.cout, c0=q.c0, cout0=q.cout0,
                      ksize=q.ksize, dil=q.dil, stride=q.stride, pad=q.pad, up=q.up)

    def pooled(p, s):
        n, f = s.shape[0], (2 if p.pre_avg else 1) * p.pool
        xp = torch.empty((n, p.cin, s.shape[2] // f, s.shape[3] // f), dtype=s.dtype, device=s.device)
        idx = torch.empty(xp.shape, dtype=torch.uint8, device=s.device) if p.pool > 1 else None
        fn = "csnet_train_pool_fwd_bf16" if s.dtype == torch.bfloat16 else "csnet_train_pool_fwd"
        assert getattr(T.lib(), fn)(s.data_ptr(), n, s.shape[1], p.c0, p.cin, s.shape[2], s.shape[3], p.pre_avg, p.pool, xp.data_ptr(),
                                    _ptr(idx), torch.cuda.current_stream().cuda_stream) == 0
        r = R.pool_fwd(s, p.c0, p.cin, p.pre_avg, p.pool)
        cert.check("pool_fwd", xp, *r["dst"])
        if idx is not None:
            assert R.idx_violations(idx, *r["idx"]) == (0, 0), ("pool_fwd idx", tuple(s.shape), p.pre_avg, p.pool)
        return xp

    def mix_forward(ctx, spec, *tensors):
        dst = mix_f(ctx, spec, *tensors)
        with torch.no_grad():
            out_c, out_h, out_w, paths = spec[:4]
            ts = [t.detach().contiguous() for t in tensors]
            rp = []
            for p in paths:
                q = rpath(p, ts)
                if p.ksize > 0 and (p.pre_avg or p.pool > 1):
                    q.src, q.c0 = pooled(p, ts[p.src]), 0
                rp.append(q)
            cert.check("mix_fwd", dst, *R.mix_fwd(rp, out_c, out_h, out_w)["dst"])
        return dst

    def dgrad_ref(ctx, saved, dd, ks, j, a, b, bf):
        """The gradient MixFn returns for input j, images [a, b): each path's data gradient (stored in the sources' dtype by the
        kernel; a pooled path's routed through pool_bwd, exact in bf16 but for underflow) at its channel slice, and one rounding to
        the sources' dtype for each of the len(ks) - 1 adds."""
        paths = ctx.spec[3]
        shp = ctx.shapes[j]
        v = torch.zeros((b - a,) + tuple(shp[1:]), dtype=torch.float64, device=dd.device)
        bnd, mag = torch.zeros_like(v), torch.zeros_like(v)
        u, tiny = (RB.U_BF16, RB.TINY_BF16) if bf else (R.U, R.TINY)
        for k in ks:
            p, q = paths[k], ctx.dense[k]
            rq = rpath(q, saved)
            rq.src = rq.src[a:b]
            rv, rb = R.mix_dgrad(dd[a:b], rq)["dsrc"]
            if bf:
                rb = RB.widen(rv, rb)
            if k in ctx.pooled:
                idx = saved[ctx.pooled[k][1]]
                idx = idx[a:b] if idx is not None else None
                route = lambda t: R.pool_bwd(t, idx, shp[2], shp[3], p.pre_avg, p.pool)["dsrc"][0]
                rv, rb = route(rv), route(rb) + tiny
            sl = slice(p.c0, p.c0 + p.cin)
            v[:, sl] += rv
            bnd[:, sl] += rb
            mag[:, sl] += rv.abs() + rb
        return v, bnd + (len(ks) - 1) * (u * mag + tiny)

    def mix_backward(ctx, ddst):
        grads = mix_b(ctx, ddst)
        with torch.no_grad():
            paths = ctx.spec[3]
            saved = ctx.saved_tensors
            dd = ddst.contiguous()
            N = dd.shape[0]
            for j in range(ctx.n_in):
                g = grads[1 + j]
                if g is None:
                    continue
                srcs = [k for k, p in enumerate(paths) if p.src == j]
                wts = [k for k, p in enumerate(paths) if p.w == j]
                if srcs:
                    entry = "mix_dgrad+pool_bwd" if any(k in ctx.pooled for k in srcs) else "mix_dgrad"
                    per = max(1, (1 << 24) // max(1, int(np.prod(ctx.shapes[j][1:]))))
                    for a in range(0, N, per):
                        b = min(N, a + per)
                        cert.check(entry, g[a:b], *dgrad_ref(ctx, saved, dd, srcs, j, a, b, g.dtype == torch.bfloat16), count=a == 0, complete=True)
                elif wts:
                    v = bnd = mag = 0.0
                    for k in wts:
                        rv, rb = R.mix_wgrad(dd, rpath(ctx.dense[k], saved), sms=cert.sms)["dw"]
                        v, bnd, mag = v + rv, bnd + rb, mag + rv.abs() + rb
                    cert.check("mix_wgrad", g, v, bnd + (len(wts) - 1) * R.U * mag)
                else:
                    cert.skipped["MixFn.backward"] += 1
        return grads

    monkeypatch.setattr(T.MixFn, "forward", staticmethod(mix_forward))
    monkeypatch.setattr(T.MixFn, "backward", staticmethod(mix_backward))


def _model(tag="csnet-L-x2"):
    from sod100k_b200.model import csnet
    from tests import fixtures

    cfg, sd = fixtures.checkpoint(tag)
    m = csnet.CSNet(cfg)
    m.load_state_dict(sd)
    return m.cuda().train()


def _batch(n, hw, seed):
    from sod100k_b200 import synth

    return torch.from_numpy(synth.randn_images(n, hw, hw, seed)).cuda(), torch.from_numpy(synth.random_masks(n, hw, hw, seed + 1)).cuda()


@pytest.mark.parametrize("tag,n,hw", [("csnet-L-x2", 256, 224), ("csnet-L-x2", 2, 64), ("csnet-L-x1", 2, 64)],
                         ids=["x2_bench_b256_224", "x2_b2_64", "x1_b2_64"])
def test_bf16_trainer_step_certified_op_by_op(monkeypatch, tag, n, hw):
    from sod100k_b200.trainer import Trainer

    m = _model(tag)
    tr = Trainer(m, lr=1e-4, weight_decay=5e-3, flops_weight=3.0, flops_expand=1.0, storage="bf16")
    x, t = _batch(n, hw, 81)
    cert = Bf16Certifier(_sms())
    _install_bf16(monkeypatch, cert)
    tr.step(x, t)
    torch.cuda.synchronize()
    for entry in sorted(cert.worst):
        _note(entry, f"bf16_trainer_step/{tag}/b{n}_{hw}/calls={cert.calls[entry]}", cert.worst[entry])
    print("calls checked:", dict(cert.calls), "skipped:", dict(cert.skipped))
    assert not cert.skipped, cert.skipped
    for entry in ("mix_fwd", "mix_dgrad", "mix_dgrad+pool_bwd", "mix_wgrad", "pool_fwd", "dw_conv", "dw_bwd.dx", "dw_bwd.dw", "bn_stats.mean",
                  "bn_stats.var", "bn_prelu_fwd.y", "bn_prelu_fwd.gap", "bn_prelu_bwd.dz", "bn_prelu_bwd.dgamma", "bce.loss", "bce.dlogits",
                  "adam"):
        assert cert.calls[entry] > 0, entry


# ---- 4 -----------------------------------------------------------------------------------------------------------------------
def test_bf16_step_saves_bf16_and_converts_nothing():
    from torch.utils._python_dispatch import TorchDispatchMode

    from sod100k_b200.trainer import Trainer

    n = 7
    m = _model()
    tr = Trainer(m, flops_weight=3.0, storage="bf16")
    x, t = _batch(n, 64, 91)
    saved = []

    def pack(v):
        saved.append((v.dtype, tuple(v.shape), v.data_ptr()))
        return v

    conversions = []

    class Conversions(TorchDispatchMode):
        def __torch_dispatch__(self, func, types, args=(), kwargs=None):
            out = func(*args, **(kwargs or {}))
            if func.__name__.split(".")[0] in ("_to_copy", "copy_", "to"):
                ins = [a for a in args if isinstance(a, torch.Tensor)]
                outs = [out] if isinstance(out, torch.Tensor) else []
                dts = {v.dtype for v in ins + outs}
                if {torch.bfloat16, torch.float32} <= dts and any(v.dim() >= 3 for v in ins + outs):
                    conversions.append((func.__name__, [tuple(v.shape) for v in ins]))
            return out

    with torch.autograd.graph.saved_tensors_hooks(pack, lambda v: v), Conversions():
        tr.step(x, t)
    torch.cuda.synchronize()
    assert not conversions, conversions[:10]
    acts = [(dt, shp) for dt, shp, ptr in saved if len(shp) == 4 and shp[0] == n]
    kept_fp32 = [(dt, shp) for dt, shp, ptr in saved if len(shp) == 4 and shp[0] == n and dt != torch.bfloat16]
    # fp32 by policy: the network input and its pooled copies (the stem's sources), the 1-channel maps after cls_layer and the BCE
    # gradient; uint8 arg-max indices
    pooled_input = lambda shp: shp[1] == x.shape[1] and any(shp[2:] == (x.shape[2] >> k, x.shape[3] >> k) for k in range(1, 4))
    allowed = [(dt, shp) for dt, shp, ptr in saved if len(shp) == 4 and shp[0] == n and dt != torch.bfloat16
               and (ptr == x.data_ptr() or (dt == torch.float32 and pooled_input(shp)) or shp[1] == 1 or dt == torch.uint8)]
    print(f"saved 4-D batch tensors: {len(acts)}, bf16 {len(acts) - len(kept_fp32)}, fp32 / uint8 by policy {len(allowed)}")
    assert len(acts) > 50
    assert kept_fp32 == allowed, [v for v in kept_fp32 if v not in allowed][:10]
    gaps = [(dt, shp) for dt, shp, _ in saved if len(shp) == 2 and shp[0] == n]
    assert gaps and all(dt == torch.float32 for dt, _ in gaps)          # the Oct_bn_hook GAP [N, C] stays fp32


# ---- 5 -----------------------------------------------------------------------------------------------------------------------
def _params_after_step(storage, recompute, n=4, hw=64, measure=False):
    from sod100k_b200.trainer import Trainer

    m = _model()
    tr = Trainer(m, flops_weight=3.0, storage=storage, recompute=recompute)
    x, t = _batch(n, hw, 95)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    held = None
    if measure:                                      # memory held between the forward and the backward: what the step saved
        from sod100k_b200 import train_ops as T

        m.clear_flops()
        m.set_batchsize(n)
        loss = T.BceFn.apply(m(x), t) + 3.0 * m.get_flops()
        torch.cuda.synchronize()
        held = torch.cuda.memory_allocated() - base
        loss.backward()
        del loss
    tr.step(x, t)
    torch.cuda.synchronize()
    return [p.detach().clone() for p in m.parameters()], held


def test_bf16_step_is_deterministic_and_recompute_gives_the_same_bits():
    a, held = _params_after_step("bf16", False, measure=True)
    b, _ = _params_after_step("bf16", False, measure=True)
    c, held_rc = _params_after_step("bf16", True, measure=True)
    f32, held32 = _params_after_step("fp32", False, measure=True)
    for pa, pb, pc in zip(a, b, c):
        assert torch.equal(pa, pb)
        assert torch.equal(pa, pc)
    print(f"held between forward and backward at b4 64^2: fp32 {held32} B, bf16 {held} B, bf16 + recompute {held_rc} B")
    assert held_rc < held < held32
    assert any(not torch.equal(pa, pf) for pa, pf in zip(a, f32))     # the storage option is live


# ---- 6 -----------------------------------------------------------------------------------------------------------------------
def test_bf16_training_tracks_fp32_loss():
    """SURVEY §8d's training gate: csnet-L-x2 from the shipped checkpoint, batch 16 at 224^2, 20 steps on seeded batches.

    Gate (1 %): at every step of the fp32 Trainer's run, the loss with bf16 storage on the same parameters and batch.
    Reported: two free-running runs against the fp32 one, the bf16 Trainer's and an fp32 Trainer's started from parameters one
    ulp away.  Adam's first steps move each parameter by about lr * sign(gradient), so a small gradient difference changes the
    trajectory; the control shows how far fp32 itself drifts from such a difference."""
    from sod100k_b200 import train_ops as T
    from sod100k_b200.trainer import Trainer

    batches = [_batch(16, 224, 1000 + 2 * k) for k in range(20)]

    def run(storage, perturb=False, lockstep=False):
        m = _model()
        if perturb:
            with torch.no_grad():
                g = torch.Generator().manual_seed(7)
                for p in m.parameters():                   # every parameter one ulp up or down
                    away = torch.where(torch.rand(p.shape, generator=g) < 0.5, -torch.inf, torch.inf).cuda()
                    p.copy_(torch.nextafter(p, away))
        tr = Trainer(m, lr=1e-4, weight_decay=5e-3, flops_weight=3.0, storage=storage)
        out, same = [], []
        for x, t in batches:
            if lockstep:                                   # the bf16 loss on this step's parameters, without a step
                bufs = [b.clone() for b in m.buffers()]
                m.train_storage = "bf16"
                with torch.no_grad():
                    same.append(T.BceFn.apply(m(x), t))
                m.train_storage = storage
                with torch.no_grad():
                    for b, v in zip(m.buffers(), bufs):
                        b.copy_(v)
            out.append(tr.step(x, t))
        return torch.stack(out).cpu().double(), (torch.stack(same).cpu().double() if lockstep else None)

    ref, same = run("fp32", lockstep=True)
    bf, _ = run("bf16")
    ctl, _ = run("fp32", perturb=True)
    gap = lambda v: float(((v - ref).abs() / ref.abs()).max())
    print("fp32 losses:", [round(v, 5) for v in ref.tolist()])
    print("bf16 losses:", [round(v, 5) for v in bf.tolist()])
    print("fp32 from parameters one rounding away:", [round(v, 5) for v in ctl.tolist()])
    print(f"max relative loss gap: bf16 on the fp32 run's parameters {gap(same):.4%}, free-running bf16 {gap(bf):.4%}, "
          f"free-running fp32 control {gap(ctl):.4%}")
    assert gap(same) <= 0.01
    assert gap(bf) > 0.0 and gap(ctl) > 0.0                 # both runs are live
