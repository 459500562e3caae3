"""tests/opref.py, the float64 reference and error bound of one program op, checked without a GPU:
  * the host emulation of the generic kernels (tests/emu: the exact per-thread bodies of generic_ops.cuh) lies inside the
    bound for every MIX path kind, DW and GN;
  * an ILBLOCK op's reference equals the chained references of the same block compiled unfused (MIX + DW ops);
  * the check has power: each of a list of typical kernel mistakes, applied to the reference, is flagged on its case."""
import numpy as np
import pytest
import torch

from sod100k_b200 import compiler, ir
from tests import emu, fixtures
from tests.opref import DEFECTS, check, opref

F32, F16 = ir.F32, ir.F16


def _inputs16(rng, shape, dtype=F16):
    """Values of a 16-bit tensor: normal, with exact zeros, negatives and (fp16) subnormals mixed in."""
    x = rng.standard_normal(shape)
    flat = x.reshape(-1)
    k = flat.size
    flat[rng.integers(0, k, k // 16)] = 0.0
    if dtype == F16:
        flat[rng.integers(0, k, k // 32)] = rng.uniform(-1, 1, k // 32) * 2.0 ** -15
        return x.astype(np.float16).astype(np.float64)
    if dtype == ir.BF16:
        u = x.astype(np.float32).view(np.uint32)
        return ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32).view(np.float32).astype(np.float64)
    return x.astype(np.float32).astype(np.float64)


def single_op(srcs, dst, paths, kind=ir.OP_MIX, bias=False, slope=False, seed=0, wscale=None, ext=None, dst_dtype=None):
    """A one-op program: sources are externals 0..k-1, the destination external k.  srcs / dst: (C, H, W, dtype);
    paths: ir.Path objects without w_off (random weights are appended for conv paths)."""
    rng = np.random.default_rng(seed)
    b = ir.Builder()
    sid = [b.tensor(c, h, w, dt, external=i) for i, (c, h, w, dt) in enumerate(srcs)]
    C, H, W, dt = dst
    d = b.tensor(C, H, W, dt, external=len(srcs))
    for q in paths:
        q.src = sid[q.src]
        if q.ksize > 0:
            n = q.cin * q.ksize * q.ksize
            s = (1.0 / np.sqrt(n)) if wscale is None else wscale
            q.w_off = b.param(rng.uniform(-s, s, (q.cin, q.ksize * q.ksize, q.cout)))
    Cm = ext[2] if (ext is not None and kind == ir.OP_MIXPROJ) else C
    o = b.op(kind, d, paths, bias=rng.uniform(-0.5, 0.5, Cm) if bias else None, slope=rng.uniform(0.1, 0.4, Cm) if slope else None)
    if kind == ir.OP_MIXPROJ:
        o.ext_off = [b.param(rng.uniform(-0.3, 0.3, Cm)), b.param(rng.uniform(-0.2, 0.2, 1)), Cm]
    elif ext is not None:
        o.ext_off = [b.param(e) if isinstance(e, np.ndarray) else e for e in ext]
    return b.finish()


def dw_op(C, H, W, dtype, seed=0, bias=True, slope=True):
    rng = np.random.default_rng(seed)
    b = ir.Builder()
    s = b.tensor(C, H, W, dtype, external=0)
    d = b.tensor(C, H, W, dtype, external=1)
    w = rng.uniform(-1, 1, (C, 9)) * 100.0 / 9 * rng.uniform(0.005, 0.02)     # the folded x100 weights
    b.op(ir.OP_DW, d, [ir.Path(s, C, C, ksize=3, pad=1, w_off=b.param(w))], bias=rng.uniform(-0.5, 0.5, C) if bias else None,
         slope=rng.uniform(0.1, 0.4, C) if slope else None)
    return b.finish()


def gn_op(C, H, W, dtype, groups, seed=0, slope=True):
    rng = np.random.default_rng(seed)
    b = ir.Builder()
    s = b.tensor(C, H, W, dtype, external=0)
    d = b.tensor(C, H, W, dtype, external=1)
    o = b.op(ir.OP_GN, d, [ir.Path(s, C, C, ksize=0, up=groups)], slope=rng.uniform(0.1, 0.4, C) if slope else None)
    o.ext_off = [b.param(rng.uniform(0.5, 1.5, C)), b.param(rng.uniform(-0.3, 0.3, C))]
    return b.finish()


def make_inputs(prog, N, seed=1):
    rng = np.random.default_rng(seed)
    srcs = sorted({q.src for o in prog.ops for q in o.paths})
    return {t: _inputs16(rng, (N, prog.tensors[t].C, prog.tensors[t].H, prog.tensors[t].W), prog.tensors[t].dtype) for t in srcs}


P = ir.Path
# (name, srcs, dst, paths, kind, bias, slope) — fp32 single-op programs for the host emulation
EMU_CASES = [
    ("conv1x1_slices", [(24, 8, 12, F32)], (20, 8, 12, F32), [P(0, 9, 7, c0=5, cout0=3), P(0, 4, 10, c0=20, cout0=10)], True, True),
    ("conv3x3_pad1", [(5, 9, 11, F32)], (17, 9, 11, F32), [P(0, 5, 17, ksize=3, pad=1)], True, True),
    ("conv3x3_dil3", [(4, 10, 10, F32)], (6, 10, 10, F32), [P(0, 4, 3, ksize=3, pad=3, dil=3), P(0, 4, 3, cout0=3, ksize=3, pad=1)], True, False),
    ("conv3x3_stride2", [(6, 12, 16, F32)], (8, 6, 8, F32), [P(0, 6, 8, ksize=3, pad=1, stride=2)], False, True),
    ("pre_avg_legacy_and_pool", [(6, 16, 16, F32)], (5, 4, 4, F32), [P(0, 6, 5, pre_avg=1, pool=2, ksize=3, pad=1)], True, True),
    ("pre_avg_2_4_8", [(3, 32, 32, F32), (3, 16, 16, F32), (3, 8, 8, F32)], (4, 4, 4, F32),
     [P(2, 3, 4, pre_avg=2), P(1, 3, 4, pre_avg=4), P(0, 3, 4, pre_avg=8)], True, False),
    ("pool4", [(7, 16, 24, F32)], (9, 4, 6, F32), [P(0, 7, 9, pool=4, ksize=3, pad=1)], True, True),
    ("input_side_up", [(6, 4, 6, F32), (5, 16, 24, F32)], (11, 16, 24, F32), [P(0, 6, 11, up=4), P(1, 5, 11)], True, True),
    ("resample_bilinear", [(4, 5, 3, F32), (9, 10, 6, F32)], (9, 10, 6, F32),
     [P(0, 4, 4, c0=0, cout0=2, ksize=0, up=2), P(1, 9, 9, ksize=1)], True, True),
    ("resample_up8", [(3, 2, 3, F32)], (3, 16, 24, F32), [P(0, 3, 3, ksize=0, up=8)], False, False),
    ("resample_avg_max_copy", [(5, 16, 16, F32), (5, 8, 8, F32)], (5, 8, 8, F32),
     [P(0, 5, 5, ksize=0, pre_avg=1), P(0, 5, 5, ksize=0, pool=2), P(1, 3, 3, c0=2, cout0=1, ksize=0)], True, False),
]


@pytest.mark.parametrize("case", EMU_CASES, ids=[c[0] for c in EMU_CASES])
def test_emulated_generic_mix_kernel_lies_within_the_bound(case):
    name, srcs, dst, paths, bias, slope = case
    prog = single_op(srcs, dst, [P(**vars(p)) for p in paths], bias=bias, slope=slope, seed=len(name))
    _run_emu_and_check(prog, N=2)


@pytest.mark.parametrize("C,H,W", [(5, 7, 9), (3, 1, 4), (16, 12, 8)])
def test_emulated_generic_dw_kernel_lies_within_the_bound(C, H, W):
    _run_emu_and_check(dw_op(C, H, W, F32, seed=C), N=2)


@pytest.mark.parametrize("groups,slope", [(1, True), (4, False), (32, True)])
def test_emulated_gn_lies_within_the_bound(groups, slope):
    _run_emu_and_check(gn_op(64, 6, 10, F32, groups, seed=groups, slope=slope), N=2)


def _run_emu_and_check(prog, N):
    inputs = make_inputs(prog, N)
    ext = [None] * (1 + max(t.external for t in prog.tensors))
    for t, a in inputs.items():
        ext[prog.tensors[t].external] = np.ascontiguousarray(a, np.float32)
    d = prog.tensors[prog.ops[0].dst]
    ext[d.external] = np.zeros((N, d.C, d.H, d.W), np.float32)
    emu.run_ext(prog, ext, N)
    (ref, bound), = opref(prog, 0, inputs).values()
    q, msg = check(torch.from_numpy(ext[d.external]), ref, bound)
    assert q <= 1.0, msg
    assert float(ref.abs().max()) > 0


# ---- ILBLOCK against its unfused form -------------------------------------------------------------------------------------
def _block_programs(tag, stem):
    cfg, sd = fixtures.checkpoint(tag)
    full = compiler.compile_csnet(cfg, sd, 64, 64, "fp16", fuse=True)
    name = next(o.name for o in full.ops if o.kind == ir.OP_ILBLOCK and (o.paths[0].ksize == 3) == stem)
    fused = compiler.compile_csnet(cfg, sd, 64, 64, "fp16", reuse_arena=False, fuse={name})
    plain = compiler.compile_csnet(cfg, sd, 64, 64, "fp16", reuse_arena=False, fuse=False)
    return name, fused, plain


def _chain(prog, prefix, values):
    """Float64 references of the block's ops in program order, each fed the previous references."""
    for k, o in enumerate(prog.ops):
        if o.name.startswith(prefix + "."):
            for t, (r, _) in opref(prog, k, values).items():
                values[t] = r
    return values


@pytest.mark.parametrize("tag", ["csnet-L-x2", "csnet-L-x1"])
@pytest.mark.parametrize("stem", [False, True], ids=["1x1", "stem"])
def test_ilblock_reference_equals_the_unfused_chain(tag, stem):
    name, fused, plain = _block_programs(tag, stem)
    k = next(i for i, o in enumerate(fused.ops) if o.kind == ir.OP_ILBLOCK and o.name == name)
    op = fused.ops[k]
    inv = {t: n for n, t in fused.taps.items()}
    rng = np.random.default_rng(7)
    srcs = sorted({q.src for q in op.paths})
    inputs, plain_inputs = {}, {}
    for t in srcs:
        d = fused.tensors[t]
        a = _inputs16(rng, (2, d.C, d.H, d.W), d.dtype)
        inputs[t] = a
        plain_inputs[fused.input if t == fused.input else plain.taps[inv[t]]] = torch.from_numpy(a)
    # the fused op holds its 1x1 / stem weights as 16-bit values: give the unfused MIX ops the same (rounded) weights
    plain.blob = plain.blob.copy()
    for o in plain.ops:
        if o.name.startswith(name + ".conv1x1") and o.kind == ir.OP_MIX:
            for q in o.paths:
                if q.ksize > 0:
                    n = q.cin * q.ksize * q.ksize * q.cout
                    plain.blob[q.w_off:q.w_off + n] = plain.blob[q.w_off:q.w_off + n].astype(np.float16).astype(np.float32)
    got = opref(fused, k, inputs)
    chained = _chain(plain, name, dict(plain_inputs))
    n = 0
    for b_ in (0, 1):
        key = f"{name}/{b_}"
        if key not in fused.taps:
            continue
        ref, bound = got[fused.taps[key]]
        other = chained[plain.taps[key]]
        scale = float(ref.abs().max())
        assert scale > 0
        assert float((ref - other).abs().max()) <= 1e-12 * scale, key
        assert bool((bound > 0).all())
        n += 1
    assert n >= 1


# ---- the check has power -------------------------------------------------------------------------------------------------
def _round16(r, dtype):
    return r.to(torch.float16 if dtype == F16 else torch.bfloat16).to(torch.float64)


def _defect_case(defect):
    """(program, op index, inputs) of a 16-bit case whose data exercises the defect's edge."""
    if defect in ("replicate_pad", "row_above"):
        prog = dw_op(8, 12, 24, F16, seed=3)
    elif defect == "drop_bias":
        prog = single_op([(16, 8, 16, F16)], (12, 8, 16, F16), [P(0, 16, 12)], bias=True, slope=True, seed=4)
    elif defect == "slice_shift":
        prog = single_op([(16, 8, 16, F16)], (12, 8, 16, F16), [P(0, 9, 12, c0=3)], bias=True, seed=5)
    elif defect == "align_corners":
        prog = single_op([(6, 6, 8, ir.F32)], (6, 12, 16, F16), [P(0, 6, 6, ksize=0, up=2)], seed=6)
    elif defect == "dil_minus_1":
        prog = single_op([(16, 16, 16, F16)], (12, 16, 16, F16),
                         [P(0, 16, 3, ksize=3, pad=1), P(0, 16, 3, cout0=3, ksize=3, pad=2, dil=2),
                          P(0, 16, 3, cout0=6, ksize=3, pad=4, dil=4), P(0, 16, 3, cout0=9, ksize=3, pad=8, dil=8)],
                         bias=True, slope=True, seed=7)
    elif defect == "max_first":
        prog = single_op([(8, 16, 16, F16)], (8, 8, 8, F16), [P(0, 8, 8, pool=2)], seed=8)
    else:                                                          # t1_pre_prelu
        name, fused, _ = _block_programs("csnet-L-x2", False)
        k = next(i for i, o in enumerate(fused.ops) if o.name == name)
        return fused, k, make_inputs_for(fused, k)
    return prog, 0, make_inputs(prog, 2)


def make_inputs_for(prog, k, N=2, seed=1):
    rng = np.random.default_rng(seed)
    return {q.src: _inputs16(rng, (N,) + (prog.tensors[q.src].C, prog.tensors[q.src].H, prog.tensors[q.src].W), prog.tensors[q.src].dtype)
            for q in prog.ops[k].paths}


@pytest.mark.parametrize("defect", DEFECTS)
def test_each_defect_is_flagged(defect):
    prog, k, inputs = _defect_case(defect)
    good = opref(prog, k, inputs)
    bad = opref(prog, k, inputs, defect=defect)
    worst = 0.0
    for t, (ref, bound) in good.items():
        # the correct result, stored as a kernel would store it, passes ...
        q_ok, msg = check(_round16(ref, prog.tensors[t].dtype), ref, bound)
        assert q_ok <= 1.0, msg
        # ... the defective one does not
        q, _ = check(_round16(bad[t][0], prog.tensors[t].dtype), ref, bound)
        worst = max(worst, q)
    assert worst > 1.0, (defect, worst)
