"""CSF+Res2Net at input sizes that are not multiples of 32 on the GPU: the module against the reference's goldens, the head's taps, every
op of the programs against float64 bounds, the RESIZE kernel alone, its rejections, and the bounded plan cache."""
import collections
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import csf_res2net_oracle as R
from sod100k_b200 import compiler_r, ir, runtime, synth
from sod100k_b200.networks import csf_res2net
from tests import fixtures
from tests.opref import check, opref
from tests.resize_ref import resize64, resize_op_ref

pytestmark = pytest.mark.gpu

TORCH_DT = {ir.F32: torch.float32, ir.F16: torch.float16, ir.BF16: torch.bfloat16}
GUARD = 4096                                       # NaN bytes (0xFF) before and after every destination


def _golden():
    z = np.load(os.path.join(fixtures.GOLDEN, "csf_res2net_sizes.npz"))
    return z, json.loads(str(z["__meta__"]))


def _model(meta):
    m = csf_res2net.build_model()
    sd = synth.synth_state_r({k: tuple(v) for k, v in meta["shapes"].items()}, meta["seed"])
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    return m.cuda().eval(), {k: torch.from_numpy(v) for k, v in sd.items()}


def _ref(z, meta, tag, y):
    """(engine values, reference values) at the golden's logits (all of them, or its sample)."""
    if tag in meta["sampled"]:
        return y.reshape(-1)[z[f"{tag}/logits_idx"]], z[f"{tag}/logits_sample"]
    return y, z[f"{tag}/logits"]


def test_fp32_and_fp16_match_reference_goldens_at_any_size():
    z, meta = _golden()
    m, _ = _model(meta)
    for dtype in ("fp32", "fp16"):
        m.set_precision(dtype)
        for tag, (h, w, seed) in meta["cases"].items():
            with torch.no_grad():
                y = m(torch.from_numpy(synth.randn_images(1, h, w, seed)).cuda()).cpu().numpy()
            assert y.shape == (1, 1, h, w)
            got, ref = _ref(z, meta, tag, y)
            scale = max(1.0, np.abs(ref).max())
            if dtype == "fp32":
                assert np.abs(got - ref).max() <= 1e-3 * scale, (tag, np.abs(got - ref).max())
            else:                                  # fp16 backbone (cuDNN autocast) and head storage, as the existing CSF test
                assert np.abs(got - ref).max() <= 3e-2 * scale, (tag, np.abs(got - ref).max())
                sig = lambda v: 1.0 / (1.0 + np.exp(-v.astype(np.float64)))
                assert np.abs(sig(got) - sig(ref)).max() <= 2e-2, tag


@pytest.mark.parametrize("tag", ["75x100", "24x130", "400x300"])
def test_head_taps_match_the_oracle(tag):
    z, meta = _golden()
    _, sd = _model(meta)
    h, w, seed = meta["cases"][tag]
    x = torch.from_numpy(synth.randn_images(2, h, w, seed))
    taps = {}
    with torch.no_grad():
        ref = R.csfnet_forward(sd, x, taps)
    feats = [f.cuda().contiguous() for f in taps["feats"]]
    for tc in (False, True):
        prog = compiler_r.compile_csf_head(sd, [tuple(f.shape[1:]) for f in feats], h, w, "fp32", reuse_arena=False, tensor_core=tc)
        plan = runtime.Plan(prog, max_batch=2)
        try:
            y = torch.empty((2, 1, h, w), device="cuda")
            plan.run(2, [f.data_ptr() for f in feats] + [y.data_ptr()], torch.cuda.current_stream().cuda_stream)
            assert (y.cpu() - ref).abs().max().item() <= 1e-3 * max(1.0, ref.abs().max().item()), tc
            for name, r in (("fuse/0", taps["fuse"][0]), ("fuse/2", taps["fuse"][2]), ("ms/3", taps["ms"][3]),
                            ("fuse1x1/0", taps["fuse1x1"])):
                got = plan.read_tensor(prog.taps[name], 2).cpu()
                assert (got - r).abs().max().item() <= 1e-3 * max(1.0, r.abs().max().item()), (tc, name)
        finally:
            plan.close()


def _values(rng, shape, dtype):
    """Random values stored in `dtype` (the kernel reads exactly these)."""
    return torch.from_numpy(rng.standard_normal(shape)).to(TORCH_DT[dtype])


def _prefix_states(prog, max_batch, N, ext, wanted):
    """{k: {tensor id: float64 CPU values right after op k}} for the (k, tensors) in `wanted`: a plan of the program's first k + 1
    ops (same tensors, same kernels) run on the same inputs."""
    out = {}
    for k, tensors in sorted(wanted.items()):
        sub = ir.Program(tensors=prog.tensors, ops=prog.ops[:k + 1], blob=prog.blob, taps=prog.taps)
        plan = runtime.Plan(sub, max_batch=max_batch)
        try:
            plan.run(N, [a.data_ptr() for a in ext], torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            out[k] = {t: plan.read_tensor(t, N).cpu().to(torch.float64) for t in tensors}
        finally:
            plan.close()
    return out


def check_program_any(prog, max_batch, N, feats, label):
    """Every op of a head program against its float64 reference and bound (tests/opref.py for MIX / GN, tests/resize_ref.py for
    RESIZE), each on the values it read.  An op whose destination a later op accumulates into is checked on a run of the program
    cut after it; so is the old destination value an accumulating RESIZE reads.  Returns the op kernels."""
    ops = prog.ops
    writers = collections.defaultdict(list)
    for k, o in enumerate(ops):
        for t in o.dsts:
            writers[t].append(k)
    for k, o in enumerate(ops):                    # every source is final when it is read
        assert all(max(writers[q.src], default=-1) < k for q in o.paths), (label, o.name)
    wanted = {}
    for k, o in enumerate(ops):
        if any(max(writers[t]) > k for t in o.dsts):
            wanted[k] = o.dsts
    ext = [None] * (1 + max(t.external for t in prog.tensors))
    for i, x in feats.items():
        ext[i] = x.cuda().contiguous()
    for t in prog.tensors:
        if t.external >= 0 and ext[t.external] is None:
            ext[t.external] = torch.full((N, t.C, t.H, t.W), float("nan"), dtype=TORCH_DT[t.dtype], device="cuda")
    states = _prefix_states(prog, max_batch, N, ext, wanted)
    plan = runtime.Plan(prog, max_batch=max_batch)
    try:
        plan.run(N, [a.data_ptr() for a in ext], torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        final = {}

        def after(t, k):
            """Values of tensor t right after op k."""
            if k in states and t in states[k]:
                return states[k][t]
            assert max(writers[t], default=-1) <= k, (t, k)
            if t not in final:
                d = prog.tensors[t]
                final[t] = (ext[d.external].float() if d.external >= 0 else plan.read_tensor(t, N)).cpu().to(torch.float64)
            return final[t]

        kernels = []
        for k, o in enumerate(ops):
            kern = plan.op_kernel(k)
            kernels.append(kern)
            inputs = {q.src: after(q.src, k) for q in o.paths}
            if o.kind == ir.OP_RESIZE:
                refs = resize_op_ref(prog, k, inputs, after(o.dst, k - 1) if o.ext_off[0] == 1 else None)
            else:
                refs = opref(prog, k, inputs)
            for t, (ref, bound) in refs.items():
                got = after(t, k)
                if o.kind == ir.OP_RESIZE:
                    q = o.paths[0]
                    got = got[:, q.cout0:q.cout0 + q.cout]
                qv, msg = check(got, ref, bound)
                assert qv <= 1.0, (label, k, o.name, kern, msg)
        return kernels
    finally:
        plan.close()


@pytest.mark.parametrize("dtype", ["fp32", "fp16"])
@pytest.mark.parametrize("H,W", [(75, 100), (300, 400)])
def test_any_size_head_program_op_by_op(H, W, dtype):
    _, meta = _golden()
    sd = synth.synth_state_r({k: tuple(v) for k, v in meta["shapes"].items()}, meta["seed"])
    dims = [(c, h, w) for c, (h, w) in zip((256, 512, 1024, 2048), compiler_r.res2net_feat_dims(H, W))]
    prog = compiler_r.compile_csf_head(sd, dims, H, W, dtype, reuse_arena=False)
    rng = np.random.default_rng(H + W)
    dt = ir.DTYPE_NAMES[dtype]
    feats = {i: _values(rng, (1,) + d, dt).abs() * 0.5 for i, d in enumerate(dims)}      # post-ReLU backbone features
    kernels = check_program_any(prog, 1, 1, feats, f"csf_head/{dtype}/{H}x{W}")
    assert {kernels[k] for k, o in enumerate(prog.ops) if o.kind == ir.OP_RESIZE} == {"resize_kernel"}
    print("CSF_ANY_KERNELS", H, W, dtype, dict(collections.Counter(kernels)))


def _resize_prog(Cs, Hs, Ws, Cd, Hd, Wd, c0, cout0, C_, accumulate, sdt, ddt):
    """One RESIZE op from external 0 into external 1.  External 2 is bound but unused: a plan with exactly two externals replays
    small batches through staging copies of its input and output (csnet_plan_run), which do not carry the destination's old values."""
    b = ir.Builder()
    s = b.tensor(Cs, Hs, Ws, sdt, external=0, name="src")
    d = b.tensor(Cd, Hd, Wd, ddt, external=1, name="dst")
    b.tensor(1, 1, 1, ir.F32, external=2, name="unused")
    b.op(ir.OP_RESIZE, d, [ir.Path(s, C_, C_, c0=c0, cout0=cout0, ksize=0)], name="resize").ext_off = [int(accumulate)]
    return b.finish(reuse=False)


def _run_resize(plan, prog, N, src, old):
    """Run batch N with the destination inside NaN guard bands, starting from `old`; returns (dst, guards intact)."""
    d = prog.tensors[1]
    nbytes = N * d.C * d.H * d.W * ir.DTYPE_BYTES[d.dtype]
    buf = torch.full((GUARD + nbytes + GUARD,), 0xFF, dtype=torch.uint8, device="cuda")
    dst = buf[GUARD:GUARD + nbytes].view(TORCH_DT[d.dtype]).view(N, d.C, d.H, d.W)
    dst.copy_(old[:N])
    s = src[:N].cuda().contiguous()
    spare = torch.zeros(1, device="cuda")
    plan.run(N, [s.data_ptr(), dst.data_ptr(), spare.data_ptr()], torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    intact = bool((buf[:GUARD] == 0xFF).all()) and bool((buf[-GUARD:] == 0xFF).all())
    return dst.cpu(), intact


DT = (ir.F32, ir.F16, ir.BF16)
RESIZE_CASES = (
    # (Hs, Ws) -> (Hd, Wd), source / destination dtype pairs
    [((13, 17), (75, 100), s, d) for s in DT for d in DT] +
    [((75, 100), (10, 13), ir.F16, ir.F16), ((19, 25), (19, 25), ir.F32, ir.F16), ((1, 1), (7, 5), ir.F32, ir.F32),
     ((7, 9), (1, 1), ir.F16, ir.F32), ((1, 9), (5, 1), ir.BF16, ir.BF16), ((30, 40), (9, 700), ir.F32, ir.F16),
     ((38, 50), (300, 401), ir.F32, ir.F32), ((10, 13), (75, 101), ir.F32, ir.F16)])


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("case", RESIZE_CASES, ids=[f"{a[0]}x{a[1]}to{b[0]}x{b[1]}-{s}{d}" for a, b, s, d in RESIZE_CASES])
def test_resize_kernel_alone(case, accumulate):
    (Hs, Ws), (Hd, Wd), sdt, ddt = case
    Cs, Cd, c0, cout0, C_, mb = 11, 13, 2, 3, 9, 3
    prog = _resize_prog(Cs, Hs, Ws, Cd, Hd, Wd, c0, cout0, C_, accumulate, sdt, ddt)
    rng = np.random.default_rng(Hs * 7 + Wd)
    src = _values(rng, (mb, Cs, Hs, Ws), sdt)
    old = _values(rng, (mb, Cd, Hd, Wd), ddt).cuda()
    plan = runtime.Plan(prog, max_batch=mb)
    try:
        assert plan.op_kernel(0) == "resize_kernel"
        runs = {}
        for N in (1, mb):
            got, intact = _run_resize(plan, prog, N, src, old)
            assert intact, (case, N, "guard band overwritten")
            prev = old[:N].cpu().to(torch.float64)
            ref, bound = resize64(src[:N, c0:c0 + C_].to(torch.float64), Hd, Wd, prev[:, cout0:cout0 + C_] if accumulate else None, ddt)
            q, msg = check(got[:, cout0:cout0 + C_].to(torch.float64), ref, bound)
            assert q <= 1.0, (case, N, msg)
            keep = [c for c in range(Cd) if not cout0 <= c < cout0 + C_]
            assert torch.equal(got[:, keep], old[:N, keep].cpu()), "channels outside the slice changed"
            runs[N] = got
        bits = torch.int16 if runs[1].element_size() == 2 else torch.int32
        assert torch.equal(runs[1].view(bits), runs[mb][:1].contiguous().view(bits)), "image 0 differs between batch 1 and max_batch"
    finally:
        plan.close()


def _bad(field):
    prog = _resize_prog(4, 5, 6, 4, 7, 9, 0, 0, 4, False, ir.F32, ir.F32)
    op = prog.ops[0]
    q = op.paths[0]
    if field == "n_paths":
        op.paths.append(ir.Path(0, 4, 4, ksize=0))
    elif field == "ksize":
        q.ksize, q.w_off = 1, 0
    elif field == "cin_ne_cout":
        q.cin = 3
    elif field == "c0":
        q.c0 = 1
    elif field == "cout0":
        q.cout0 = 1
    elif field in ("up", "pool", "pre_avg", "stride", "dil", "pad"):
        setattr(q, field, 2)
    elif field == "w_off":
        q.w_off = 0
    elif field == "accumulate":
        op.ext_off = [2]
    elif field == "ext_off1":
        op.ext_off = [0, 0]
    elif field == "bias":
        op.bias_off = 0
    elif field == "slope":
        op.slope_off = 0
    elif field == "dst2":
        op.dst2 = 0
    elif field == "in_place":
        q.src = op.dst
    elif field == "src_range":
        q.src = 5
    return prog


BAD = ["n_paths", "ksize", "cin_ne_cout", "c0", "cout0", "up", "pool", "pre_avg", "stride", "dil", "pad", "w_off", "accumulate",
       "ext_off1", "bias", "slope", "dst2", "in_place", "src_range"]


@pytest.mark.parametrize("field", BAD)
def test_plan_creation_rejects_malformed_resize_ops(field):
    runtime.Plan(_resize_prog(4, 5, 6, 4, 7, 9, 0, 0, 4, False, ir.F32, ir.F32), max_batch=1).close()     # the well-formed op
    prog = _bad(field)
    lib = runtime.load_library()
    h = C.c_void_p()
    rc = lib.csnet_plan_create(C.byref(h), prog.tensor_array(), len(prog.tensors), prog.op_array(), len(prog.ops),
                               int(prog.blob.size), 1, 0)
    assert rc == -1 and not h.value, (field, rc)             # CSNET_E_INVALID, nothing created
    assert b"op 0" in lib.csnet_last_error(), lib.csnet_last_error()


def test_plan_cache_stays_within_the_budget():
    z, meta = _golden()
    m, _ = _model(meta)
    sizes = [(75, 100), (97, 131), (96, 100), (80, 112), (24, 130)]
    xs = {s: torch.from_numpy(synth.randn_images(1, s[0], s[1], 1500 + i)).cuda() for i, s in enumerate(sizes)}
    first = {}
    with torch.no_grad():
        m.plan_budget = 1 << 40
        for s in sizes:
            first[s] = m(xs[s]).cpu()
        arenas = {k: p.arena_bytes for k, p in m._plans.items()}
        assert len(arenas) == len(sizes)
        m.plan_budget = max(arenas.values()) + min(arenas.values())        # holds two plans, not five
        for _ in range(2):
            for s in sizes:
                y = m(xs[s]).cpu()
                assert torch.equal(y, first[s]), s                        # a rebuilt plan computes the same bits
                resident = {k: p.arena_bytes for k, p in m._plans.items()}
                assert sum(resident.values()) <= m.plan_budget and 1 <= len(resident) < len(sizes)
                assert next(reversed(m._plans))[:2] == s                  # the plan just used is the most recent
                assert set(m._plan_version) == set(m._plans)
        # new weights re-fold every cached plan, evicted ones included
        with torch.no_grad():
            m.cls_layer.bias.add_(0.25)
        for s in sizes[-2:] + sizes[:1]:
            y = m(xs[s]).cpu()
            assert (y - (first[s] + 0.25)).abs().max().item() <= 1e-4 * max(1.0, first[s].abs().max().item()), s
