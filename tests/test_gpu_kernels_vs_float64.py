"""Every inference kernel, op by op, against the float64 reference of tests/opref.py with its per-element error bound.

(a) One-op programs built with ir.Builder, one case per geometry branch of a kernel.  Inputs and outputs are externals; each
    output lies inside a larger buffer whose 256-byte guard bands (and the output itself) start as a NaN pattern, so an
    element the kernel never writes fails the check and a write outside the output changes a guard.  Every case asserts
    the kernel it means to test (csnet_plan_op_kernel), runs at a small batch and at max_batch, checks every element of
    both runs against the reference and checks that each image of the small run is bit-identical in the large one.
(b) The shipped programs, compiled with every tensor kept (reuse_arena=False): each op's output is checked against the
    reference evaluated on that op's stored inputs, so every op of the bench plan is certified at its real shape and
    errors do not compound.

Every check prints q = max |got - ref| / bound (pytest -s) as `OPREF_Q <kernel> <case> <q>`."""
import collections
import os

import numpy as np
import pytest
import torch

from sod100k_b200 import compiler, compiler_r, ir, runtime, synth
from tests import fixtures
from tests.opref import check, opref
from tests.test_gpu_il_stream import EXPECTED_KERNELS

pytestmark = pytest.mark.gpu

F32, F16, BF16 = ir.F32, ir.F16, ir.BF16
TORCH_DT = {F32: torch.float32, F16: torch.float16, BF16: torch.bfloat16}
GUARD = 256
P = ir.Path
SWITCHES = ("CSNET_MS", "CSNET_ILS", "CSNET_ILS_NS", "CSNET_ILS_MIN_CHUNKS")


def _note(kernel, case, q):
    print(f"OPREF_Q {kernel!r} {case} {q:.4f}")


def plan_with(prog, max_batch, env):
    """A plan created with the kernel switches in `env` (read at plan creation), the previous environment restored."""
    old = {k: os.environ.get(k) for k in SWITCHES}
    for k in SWITCHES:
        os.environ.pop(k, None)
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return runtime.Plan(prog, max_batch=max_batch)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# ---- input values and one-op programs ----------------------------------------------------------------------------------
def values(rng, shape, dtype):
    """Normal values with exact zeros, negatives and (fp16) subnormals, as a CPU tensor of the storage type."""
    x = rng.standard_normal(shape)
    f = x.reshape(-1)
    k = f.size
    f[rng.integers(0, k, max(1, k // 16))] = 0.0
    if dtype == F16:
        m = max(1, k // 32)
        f[rng.integers(0, k, m)] = rng.uniform(-1, 1, m) * 2.0 ** -15
    return torch.from_numpy(x).to(TORCH_DT[dtype])


def mix(srcs, dst, paths, kind=ir.OP_MIX, bias=True, slope=True, seed=0, proj_c=None):
    rng = np.random.default_rng(seed)
    b = ir.Builder()
    sid = [b.tensor(c, h, w, dt, external=i) for i, (c, h, w, dt) in enumerate(srcs)]
    C, H, W, dt = dst
    d = b.tensor(C, H, W, dt, external=len(srcs))
    for q in paths:
        q.src = sid[q.src]
        if q.ksize > 0:
            s = 1.0 / np.sqrt(q.cin * q.ksize * q.ksize)
            q.w_off = b.param(rng.uniform(-s, s, (q.cin, q.ksize * q.ksize, q.cout)))
    Cm = proj_c or C
    o = b.op(kind, d, paths, bias=rng.uniform(-0.5, 0.5, Cm) if bias else None, slope=rng.uniform(0.1, 0.4, Cm) if slope else None)
    if kind == ir.OP_MIXPROJ:
        o.ext_off = [b.param(rng.uniform(-0.3, 0.3, Cm)), b.param(rng.uniform(-0.2, 0.2, 1)), Cm]
    return b.finish()


def dw(C, H, W, dt, bias=True, slope=True, seed=0, src_dt=None):
    rng = np.random.default_rng(seed)
    b = ir.Builder()
    s = b.tensor(C, H, W, src_dt if src_dt is not None else dt, external=0)
    d = b.tensor(C, H, W, dt, external=1)
    w = rng.uniform(-1, 1, (C, 9)) * 100.0 / 9                 # the x100 of Conv2dX100 folded in
    b.op(ir.OP_DW, d, [P(s, C, C, ksize=3, pad=1, w_off=b.param(w))], bias=rng.uniform(-0.5, 0.5, C) if bias else None,
         slope=rng.uniform(0.1, 0.4, C) if slope else None)
    return b.finish()


def gn(C, H, W, dt, groups, slope=True, seed=0):
    rng = np.random.default_rng(seed)
    b = ir.Builder()
    s = b.tensor(C, H, W, dt, external=0)
    d = b.tensor(C, H, W, dt, external=1)
    o = b.op(ir.OP_GN, d, [P(s, C, C, ksize=0, up=groups)], slope=rng.uniform(0.1, 0.4, C) if slope else None)
    o.ext_off = [b.param(rng.uniform(0.5, 1.5, C)), b.param(rng.uniform(-0.3, 0.3, C))]
    return b.finish()


def _bits(a, dt):
    a = np.ascontiguousarray(a, np.float32)
    if dt == F16:
        return a.astype(np.float16).view(np.uint16)
    u = a.view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def ilblock(Chi, Cli, Cho, Clo, H, W, dt, stem=False, seed=0):
    """One ILBLOCK op (ext_off layout of include/csnet_b200.h) with random 16-bit GEMM weights and fp32 depthwise stages."""
    rng = np.random.default_rng(seed)
    ru = lambda v, m: (v + m - 1) // m * m
    b = ir.Builder()
    if stem:
        x = b.tensor(Chi, H, W, F32, external=0)
        K, K8, srcs = Chi * 9, 32, (x, x)
    else:
        xh, xl = b.tensor(Chi, H, W, dt, external=0), b.tensor(Cli, H // 2, W // 2, dt, external=1)
        K, K8, srcs = Chi + Cli, ru(Chi + Cli, 8), (xh, xl)
    ne = 1 if stem else 2
    yh = b.tensor(Cho, H, W, dt, external=ne)
    yl = b.tensor(Clo, H // 2, W // 2, dt, external=ne + 1) if Clo else -1
    WH, WL = np.zeros((ru(Cho, 16), K8)), np.zeros((max(ru(Clo, 16), 16), K8))
    WH[:Cho, :K] = rng.uniform(-1, 1, (Cho, K)) / np.sqrt(K)
    WL[:Clo, :K] = rng.uniform(-1, 1, (Clo, K)) / np.sqrt(K)
    vec = lambda c, lo, hi: b.param(rng.uniform(lo, hi, c))
    dwp = lambda c: [b.param(rng.uniform(-1, 1, (c, 9)) * 0.6), vec(c, -0.3, 0.3), vec(c, 0.1, 0.4)]
    none3 = [-1, -1, -1]
    ext = [b.param_bits16(_bits(WH, dt)), b.param_bits16(_bits(WL, dt)), vec(Cho, -0.3, 0.3), vec(Cho, 0.1, 0.4)]
    ext += [vec(Clo, -0.3, 0.3), vec(Clo, 0.1, 0.4)] if Clo else [-1, -1]
    ext += dwp(Cho) + (dwp(Clo) if Clo else none3) + dwp(Cho) + (dwp(Clo) if Clo else none3)
    if stem:
        paths = [P(x, Chi, Cho, ksize=3, pad=1), P(x, Chi, max(Clo, 1), ksize=3, pad=1, pool=2)]
    else:
        paths = [P(xh, Chi, Cho), P(xl, Cli, Cho)]
    o = b.op(ir.OP_ILBLOCK, yh, paths)
    o.dst2, o.ext_off = yl, ext
    return b.finish()


# ---- running one case --------------------------------------------------------------------------------------------------
def _run(plan, prog, N, inputs):
    """Run batch N with the first N images of `inputs`; returns ({out tensor id: CPU tensor}, guard intact?)."""
    ext = [None] * (1 + max(t.external for t in prog.tensors))
    for t, x in inputs.items():
        ext[prog.tensors[t].external] = x[:N].cuda().contiguous()
    outs, bufs = {}, {}
    for o in prog.ops:
        for t in o.dsts:
            d = prog.tensors[t]
            if d.external < 0:
                continue
            nbytes = N * d.C * d.H * d.W * ir.DTYPE_BYTES[d.dtype]
            buf = torch.full((GUARD + nbytes + GUARD,), 0xFF, dtype=torch.uint8, device="cuda")
            bufs[t] = buf
            outs[t] = buf[GUARD:GUARD + nbytes].view(TORCH_DT[d.dtype]).view(N, d.C, d.H, d.W)
            ext[d.external] = outs[t]
    plan.run(N, [a.data_ptr() for a in ext], torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    intact = all(bool((b[:GUARD] == 0xFF).all()) and bool((b[-GUARD:] == 0xFF).all()) for b in bufs.values())
    return {t: v.cpu() for t, v in outs.items()}, intact


def run_case(case_id, prog, max_batch, n_small, env, kernel, seed=11):
    plan = plan_with(prog, max_batch, env)
    try:
        got_kernel = plan.op_kernel(0)
        assert got_kernel.startswith(kernel), (case_id, got_kernel)
        rng = np.random.default_rng(seed)
        srcs = sorted({q.src for q in prog.ops[0].paths})
        inputs = {t: values(rng, (max_batch, prog.tensors[t].C, prog.tensors[t].H, prog.tensors[t].W), prog.tensors[t].dtype)
                  for t in srcs}
        runs = {}
        for N in sorted({n_small, max_batch}):
            outs, intact = _run(plan, prog, N, inputs)
            assert intact, (case_id, N, "guard band overwritten")
            refs = opref(prog, 0, {t: x[:N] for t, x in inputs.items()})
            for t, (ref, bound) in refs.items():
                q, msg = check(outs[t].to(torch.float64), ref, bound)
                _note(got_kernel, f"{case_id}/N{N}/t{t}", q)
                assert q <= 1.0, (case_id, N, t, msg)
            runs[N] = outs
        for t, small in runs[n_small].items():
            big = runs[max_batch][t][:n_small]
            assert torch.equal(small.view(torch.int16 if small.element_size() == 2 else torch.int32),
                               big.contiguous().view(torch.int16 if big.element_size() == 2 else torch.int32)), (case_id, t)
    finally:
        plan.close()


# ---- (a) the cases -------------------------------------------------------------------------------------------------------
ILS = {"CSNET_ILS_MIN_CHUNKS": 0}
NO_ILS = {"CSNET_ILS": 0}
NO_MS = {"CSNET_MS": 0}


def _ru(v, m):
    return (v + m - 1) // m * m


def ms_batch(prog):
    """The smallest max_batch at which mix_stream takes the op: choose_kernel() in csrc/plan.cu wants
    max_batch * (H / kMsRows) >= 2 * SMs, kMsRows = 2."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return -(-2 * sms // (prog.tensors[prog.ops[0].dst].H // 2))


# The helpers below mirror choices csnet_plan_op_kernel does not report, so that every case asserts the geometry it means
# to test.  Each one follows the plan.cu function it names line by line; a change there must be mirrored here.
def resample_kernel(prog, op):
    """"pool2" / "upsample" / "resample": the pure-resample branch of choose_kernel() in csrc/plan.cu."""
    q, D = op.paths[0], prog.tensors[op.dst]
    S = prog.tensors[q.src]
    avg2, max2 = q.pre_avg == 1 and q.pool == 1, q.pre_avg == 0 and q.pool == 2
    fast = S.dtype == D.dtype and D.dtype != F32 and D.W % 4 == 0 and op.bias_off < 0 and op.slope_off < 0
    if fast and (avg2 or max2) and q.up == 1 and q.c0 == 0:
        return "pool2"
    if fast and q.up > 1 and not q.pre_avg and q.pool == 1:
        return "upsample"
    return "resample"


def dw_kernel(prog, op):
    """"fast" (dw_fast_kernel) / "generic" (dw_generic_kernel): the last line of choose_kernel() in csrc/plan.cu."""
    S, D = prog.tensors[op.paths[0].src], prog.tensors[op.dst]
    veto = len(op.ext_off) > 23 and op.ext_off[23] == 1
    return "fast" if not veto and S.dtype == D.dtype and D.dtype != F32 and D.W % 4 == 0 else "generic"


IL_TILES = ((32, 32), (28, 32), (16, 64), (16, 32), (8, 16))      # plan_il's candidates, in its order


def il_tile(prog, op):
    """(TH, TW, chunked depthwise tail) of il_block_kernel: plan_il() in csrc/plan.cu with il_smem_bytes() of il_block.cuh."""
    Xh, Xl, Yh = prog.tensors[op.paths[0].src], prog.tensors[op.paths[1].src], prog.tensors[op.dst]
    first = op.paths[0].ksize == 3
    Chi, Cli = (Xh.C * 9, 0) if first else (Xh.C, Xl.C)
    Cho, Clo = Yh.C, (prog.tensors[op.dst2].C if op.dst2 >= 0 else 0)
    K8, MH16, ML16 = _ru(Chi + Cli, 8), _ru(Cho, 16), (_ru(Clo, 16) if Clo else 0)
    rowsAh, rowsAl = max(K8, Cho), (max(K8, Clo) if Clo else Cli)
    best = None
    for chunked in (False, True):
        for TH, TW in IL_TILES:
            t2h = 8 if chunked else Cho
            if chunked and Cho <= 8:
                continue
            NPH, NPL = ((TH + 8) | 1) * (TW + 8), ((TH // 2 + 4) | 1) * (TW // 2 + 8)
            halves = rowsAh * NPH + t2h * NPH + rowsAl * NPL + Clo * NPL + MH16 * K8 + ML16 * K8
            if halves * 2 + 512 > 227 * 1024:
                continue
            if first and Xh.C * (TH + 12) * (TW + 24) * 4 > (t2h * NPH + Clo * NPL) * 2:
                continue
            cost = -(-Yh.H // TH) * -(-Yh.W // TW) * NPH * (1.15 if chunked else 1.0)
            if best is None or cost < best[0]:
                best = (cost, (TH, TW, chunked))
    return best[1]


def _ms_rows_of_source(Hs, Ws, up, oy):
    """Source row of the top-left / bottom-left bilinear tap of destination row oy: ms_tap() of mix_stream.cuh (fp32)."""
    sy = max(np.float32((np.float32(oy) + np.float32(0.5)) * (np.float32(1.0) / np.float32(up)) - np.float32(0.5)), np.float32(0))
    y0 = int(sy)
    return y0, y0 + (1 if y0 < Hs - 1 else 0)


def ms_chunk_rows(prog, op):
    """Chunk height of mix_stream_kernel: the stage layout and the rows loop of plan_ms() in csrc/plan.cu."""
    D = prog.tensors[op.dst]
    C = op.ext_off[2] if op.kind == ir.OP_MIXPROJ else D.C
    NN, G = _ru(C, 16), D.W // 8
    conv = [q for q in op.paths if q.ksize > 0]
    rs = [q for q in op.paths if q.ksize == 0]
    k3 = conv[0].ksize == 3
    S = [_ru(q.cin, 16) + 1 for q in conv]
    r128 = lambda v: _ru(v, 128)
    wb = sum(r128((9 if k3 else 1) * NN * (s - 1) * 2) for s in S)

    def stages(rows):
        nb, cpi, off = (rows * G + 7) // 8, D.H // rows, 0
        for s in S:
            off += (3 if k3 else 1) * r128((rows + (2 if k3 else 0)) * G * s * 16)
        for q in rs:
            Sq = prog.tensors[q.src]
            r_rows = max(_ms_rows_of_source(Sq.H, Sq.W, q.up, c * rows + rows - 1)[1] - _ms_rows_of_source(Sq.H, Sq.W, q.up, c * rows)[0] + 1
                         for c in range(cpi))
            off += r128(q.cout * r_rows * Sq.W * 4)
        slack = (nb * 8 - rows * G) * max(S) * 16
        return nb, min(6, int((227 * 1024 - (wb + slack + 512 + 1280 + 128)) / off))

    for rows in range(1, 17):
        if D.H % rows == 0:
            nb, ns = stages(rows)
            if nb >= 3 and ns >= 3:
                return rows
    return 2 if stages(2)[1] >= 2 else 1


def tc_geometry(prog, op):
    """(mt, rows, kc) of mix_tc_kernel: choose_tc() in csrc/plan.cu with tc_plane_halves() of mix_tc.cuh."""
    D = prog.tensors[op.dst]
    C = op.ext_off[2] if op.kind == ir.OP_MIXPROJ else D.C
    conv = [q for q in op.paths if q.ksize > 0]
    pad, kk, cin_max = max(q.pad for q in conv), max(q.ksize ** 2 for q in conv), max(q.cin for q in conv)
    mt = 5 if C > 80 else (C + 15) // 16
    rows = (4 if mt == 1 else 2 if mt == 2 else 1) if pad >= 4 else 1
    xs = _ru((8 * rows + 2 * pad) * (32 if pad == 0 else 64), 16) + 8
    kc = next((k for k in (32, 16) if k <= _ru(cin_max, 8) and (k * xs + kk * mt * 16 * (k + 8)) * 2 <= 100 * 1024), 8)
    return mt, rows, kc


GEOMETRY = {"kernel": resample_kernel, "dw": dw_kernel, "tile": il_tile, "rows": ms_chunk_rows,
            "tc": tc_geometry}


CASES = {
    # il_stream: Cho / Clo / K / W / H / strips
    "ils_K17_Cho16_Clo9_W16_H4": (lambda: ilblock(8, 9, 16, 9, 4, 16, F16), 4, 1, ILS, "il_stream"),
    "ils_K64_Cho64_Clo64_W48_H12": (lambda: ilblock(32, 32, 64, 64, 12, 48, F16), 3, 1, ILS, "il_stream"),
    "ils_K2_Cho1_Clo0_W240_H4": (lambda: ilblock(1, 1, 1, 0, 4, 240, F16), 2, 1, ILS, "il_stream"),
    "ils_K63_Cho40_Clo1_W256_ns4": (lambda: ilblock(40, 23, 40, 1, 12, 256, F16), 2, 1, dict(ILS, CSNET_ILS_NS=4), "il_stream"),
    "ils_K17_Cho40_Clo1_W256_ns2": (lambda: ilblock(9, 8, 40, 1, 4, 256, F16), 2, 1, dict(ILS, CSNET_ILS_NS=2), "il_stream"),
    "ils_K17_Cho17_Clo64_W256_ns4": (lambda: ilblock(9, 8, 17, 64, 4, 256, F16), 3, 1, dict(ILS, CSNET_ILS_NS=4), "il_stream"),
    "ils_stem_W48_H12": (lambda: ilblock(3, 0, 16, 16, 12, 48, F16, stem=True), 3, 1, ILS, "il_stream"),
    "ils_stem_Cho40_Clo1_W256_ns2": (lambda: ilblock(3, 0, 40, 1, 4, 256, F16, stem=True), 2, 1, dict(ILS, CSNET_ILS_NS=2), "il_stream"),
    "ils_Cho72_falls_back_to_il_block": (lambda: ilblock(16, 16, 72, 16, 8, 32, F16), 2, 1, ILS, "il_block", ("tile", (8, 16, False))),
    "ils_Clo65_falls_back_to_il_block": (lambda: ilblock(16, 16, 16, 65, 8, 32, F16), 2, 1, ILS, "il_block", ("tile", (8, 16, False))),
    # il_block: partial tiles, chunked tail, bf16, stem
    "ilb_W24_H14_fp16": (lambda: ilblock(16, 8, 24, 12, 14, 24, F16), 3, 1, NO_ILS, "il_block", ("tile", (16, 32, False))),
    "ilb_W40_H30_bf16": (lambda: ilblock(24, 16, 40, 20, 30, 40, BF16), 2, 1, NO_ILS, "il_block", ("tile", (32, 32, True))),
    "ilb_W56_H14_Cho8": (lambda: ilblock(8, 8, 8, 8, 14, 56, F16), 2, 1, NO_ILS, "il_block", ("tile", (16, 64, False))),
    "ilb_W64_H32_Cho80_K64": (lambda: ilblock(32, 32, 80, 80, 32, 64, F16), 2, 1, NO_ILS, "il_block", ("tile", (8, 16, False))),
    "ilb_stem_W56_H14_bf16": (lambda: ilblock(3, 0, 16, 32, 14, 56, BF16, stem=True), 2, 1, NO_ILS, "il_block", ("tile", (16, 32, False))),
    "ilb_stem_W24_H30_fp16_no_lo": (lambda: ilblock(3, 0, 24, 0, 30, 24, F16, stem=True), 2, 1, NO_ILS, "il_block", ("tile", (32, 32, False))),
    # every (tile, chunked tail) pair plan_il can choose; (16 x 64, chunked) cannot occur: whenever the unchunked 16 x 32
    # tile fits shared memory it is cheaper, and whenever it does not fit, neither does the chunked 16 x 64 tile
    "ilb_tile28_W40_H28": (lambda: ilblock(8, 8, 16, 8, 28, 40, F16), 2, 1, NO_ILS, "il_block", ("tile", (28, 32, False))),
    "ilb_tile28_chunked_W24_H28": (lambda: ilblock(16, 8, 40, 12, 28, 24, F16), 2, 1, NO_ILS, "il_block", ("tile", (28, 32, True))),
    "ilb_stem_tile28_chunked_W40": (lambda: ilblock(3, 0, 40, 40, 28, 40, F16, stem=True), 2, 1, NO_ILS, "il_block", ("tile", (28, 32, True))),
    "ilb_tile32_W24_H30_Cho8": (lambda: ilblock(16, 16, 8, 8, 30, 24, F16), 2, 1, NO_ILS, "il_block", ("tile", (32, 32, False))),
    "ilb_tile16x32_chunked_W24_H14": (lambda: ilblock(16, 8, 64, 16, 14, 24, BF16), 2, 1, NO_ILS, "il_block", ("tile", (16, 32, True))),
    "ilb_tile8x16_chunked_Cho160_W24_H10": (lambda: ilblock(8, 8, 160, 0, 10, 24, F16), 2, 1, NO_ILS, "il_block", ("tile", (8, 16, True))),
    # mix_stream: 1x1 / 3x3, 1-3 inputs, resample paths, fp32 destination, MIXPROJ, chunk heights 1 / 2 / 4 / 16
    "ms_1x1_cin64_C80_rows16": (lambda: mix([(64, 16, 16, F16)], (80, 16, 16, F16), [P(0, 64, 80)], slope=False), ms_batch, 1, {}, "mix_stream", ("rows", 16)),
    "ms_1x1_3in_2rs_C33_rows4": (lambda: mix([(1, 8, 64, F16), (15, 8, 64, F16), (17, 8, 64, F16), (40, 4, 32, F32), (33, 2, 16, F32)],
                                             (33, 8, 64, F16),
                                             [P(0, 1, 10), P(1, 15, 11, cout0=10), P(2, 17, 12, cout0=21),
                                              P(3, 20, 20, c0=7, ksize=0, up=2), P(4, 30, 30, c0=3, ksize=0, up=4)]),
                                 ms_batch, 3, {}, "mix_stream", ("rows", 4)),
    "ms_1x1_up8_fp32dst": (lambda: mix([(17, 8, 64, F16), (17, 1, 8, F32)], (17, 8, 64, F32),
                                       [P(0, 17, 17), P(1, 16, 16, c0=1, ksize=0, up=8)], slope=False), ms_batch, 1, {}, "mix_stream", ("rows", 4)),
    "ms_1x1_rows2_rs": (lambda: mix([(15, 6, 72, F16), (20, 3, 36, F32)], (15, 6, 72, F16),
                                    [P(0, 15, 15), P(1, 15, 15, c0=5, ksize=0, up=2)]), ms_batch, 1, {}, "mix_stream", ("rows", 2)),
    "ms_1x1_rows1_C1": (lambda: mix([(15, 4, 136, F16)], (1, 4, 136, F16), [P(0, 15, 1)]), ms_batch, 1, {}, "mix_stream", ("rows", 1)),
    "ms_3x3_2in_C79_fp32dst": (lambda: mix([(17, 8, 32, F16), (15, 8, 32, F16)], (79, 8, 32, F32),
                                           [P(0, 17, 40, ksize=3, pad=1), P(1, 15, 79, ksize=3, pad=1)]), ms_batch, 5, {}, "mix_stream", ("rows", 2)),
    "ms_proj_C17_2rs": (lambda: mix([(24, 8, 32, F16), (17, 4, 16, F32), (20, 2, 8, F32)], (1, 8, 32, F32),
                                    [P(0, 24, 17), P(1, 17, 17, ksize=0, up=2), P(2, 9, 9, c0=11, ksize=0, up=4)],
                                    kind=ir.OP_MIXPROJ, proj_c=17), ms_batch, 3, {}, "mix_stream", ("rows", 8)),
    "ms_3x3_1in_C17_rs": (lambda: mix([(9, 8, 64, F16), (17, 4, 32, F32)], (17, 8, 64, F16),
                                      [P(0, 9, 17, ksize=3, pad=1), P(1, 17, 17, ksize=0, up=2)], bias=False), ms_batch, 1, {}, "mix_stream", ("rows", 4)),
    "ms_proj_C1": (lambda: mix([(16, 8, 32, F16)], (1, 8, 32, F32), [P(0, 16, 1)], kind=ir.OP_MIXPROJ, proj_c=1), ms_batch, 1, {}, "mix_stream", ("rows", 8)),
    "ms_proj_C17_rs": (lambda: mix([(24, 8, 32, F16), (17, 4, 16, F32)], (1, 8, 32, F32), [P(0, 24, 17), P(1, 17, 17, ksize=0, up=2)],
                                   kind=ir.OP_MIXPROJ, proj_c=17), ms_batch, 1, {}, "mix_stream", ("rows", 8)),
    "ms_proj_C80": (lambda: mix([(64, 8, 32, F16)], (1, 8, 32, F32), [P(0, 64, 80)], kind=ir.OP_MIXPROJ, proj_c=80), ms_batch, 3, {}, "mix_stream", ("rows", 8)),
    # mix_tc: mt 1..5, C > 80, dilation rows, kc, pre_avg / pool / up / c0, fp32 source beside a 16-bit one, bf16, W % 32 != 0
    "tc_mt1_cin9_W40": (lambda: mix([(9, 8, 40, F16)], (16, 8, 40, F16), [P(0, 9, 16, ksize=3, pad=1)]), 2, 1, NO_MS, "mix_tc", ("tc", (1, 1, 16))),
    "tc_mt2_cin17": (lambda: mix([(17, 8, 40, F16)], (32, 8, 40, F16), [P(0, 17, 32)]), 2, 1, NO_MS, "mix_tc", ("tc", (2, 1, 16))),
    "tc_mt3_cin33_bf16": (lambda: mix([(33, 12, 24, BF16)], (48, 12, 24, BF16), [P(0, 33, 48, ksize=3, pad=1)]), 2, 1, NO_MS, "mix_tc", ("tc", (3, 1, 32))),
    "tc_mt4_cin70": (lambda: mix([(70, 8, 48, F16)], (61, 8, 48, F16), [P(0, 70, 61)]), 2, 1, NO_MS, "mix_tc", ("tc", (4, 1, 32))),
    "tc_mt5_C81": (lambda: mix([(17, 8, 40, F16)], (81, 8, 40, F16), [P(0, 17, 81)]), 2, 1, NO_MS, "mix_tc", ("tc", (5, 1, 16))),
    "tc_C176_split": (lambda: mix([(33, 8, 24, F16)], (176, 8, 24, F16), [P(0, 33, 176, ksize=3, pad=1)], slope=False), 2, 1, NO_MS, "mix_tc", ("tc", (5, 1, 32))),
    "tc_dil4_rows4": (lambda: mix([(9, 12, 40, F16)], (16, 12, 40, F16), [P(0, 9, 16, ksize=3, pad=4, dil=4)]), 2, 1, NO_MS, "mix_tc", ("tc", (1, 4, 16))),
    "tc_dil8_rows2": (lambda: mix([(17, 12, 40, F16)], (32, 12, 40, F16), [P(0, 17, 20, ksize=3, pad=8, dil=8),
                                                                           P(0, 17, 12, cout0=20, ksize=3, pad=1)]), 2, 1, NO_MS, "mix_tc", ("tc", (2, 2, 16))),
    # kc 8 by shared memory: at pad 16 a kc-16 tile would take 102912 B, over choose_tc's 100 KB
    "tc_dil16_rows1": (lambda: mix([(33, 8, 40, F16)], (48, 8, 40, F16), [P(0, 33, 48, ksize=3, pad=16, dil=16)]), 2, 1, NO_MS, "mix_tc", ("tc", (3, 1, 8))),
    "tc_kc8_cin5_W40": (lambda: mix([(5, 8, 40, F16)], (24, 8, 40, F16), [P(0, 5, 24, ksize=3, pad=1)]), 2, 1, NO_MS, "mix_tc", ("tc", (2, 1, 8))),
    "tc_pre_avg_pool_up_c0": (lambda: mix([(20, 16, 80, F16), (12, 32, 160, F16), (9, 4, 20, F16), (6, 8, 40, F32)], (24, 8, 40, F16),
                                          [P(0, 9, 24, c0=5, pre_avg=1, ksize=3, pad=1), P(1, 12, 24, pool=4),
                                           P(2, 9, 24, up=2), P(3, 6, 24, ksize=3, pad=1)]), 2, 1, NO_MS, "mix_tc", ("tc", (2, 1, 16))),
    "tc_proj_rs": (lambda: mix([(24, 8, 40, F16), (17, 4, 20, F32)], (1, 8, 40, F32), [P(0, 24, 17), P(1, 17, 17, ksize=0, up=2)],
                               kind=ir.OP_MIXPROJ, proj_c=17), 2, 1, NO_MS, "mix_tc", ("tc", (2, 1, 16))),
    "tc_fp32_dst_rs_bf16": (lambda: mix([(17, 8, 40, BF16), (17, 4, 20, F32)], (17, 8, 40, F32),
                                        [P(0, 17, 17), P(1, 17, 17, ksize=0, up=2)]), 2, 1, NO_MS, "mix_tc", ("tc", (2, 1, 16))),
    # msd: dilations, cout per path, cin, narrow images, H below the dilation
    "msd_dils_cin9_W24": (lambda: mix([(9, 8, 24, F16)], (21, 8, 24, F16),
                                      [P(0, 9, 1, ksize=3, pad=1), P(0, 9, 3, cout0=1, ksize=3, pad=2, dil=2),
                                       P(0, 9, 5, cout0=4, ksize=3, pad=4, dil=4), P(0, 9, 8, cout0=9, ksize=3, pad=8, dil=8),
                                       P(0, 9, 4, cout0=17, ksize=3, pad=16, dil=16)]), 2, 1, {}, "msd"),
    "msd_cin1_W8_dil16": (lambda: mix([(1, 4, 8, F16)], (8, 4, 8, F16), [P(0, 1, 8, ksize=3, pad=16, dil=16)]), 3, 1, {}, "msd"),
    "msd_cin128_W8": (lambda: mix([(128, 12, 8, F16)], (10, 12, 8, F16), [P(0, 128, 2, ksize=3, pad=1),
                                                                         P(0, 128, 8, cout0=2, ksize=3, pad=8, dil=8)]), 2, 1, {}, "msd"),
    # dw_fast / pool2 / upsample / resample and the generic fp32 kernels
    "dw_fast_W12_fp16": (lambda: dw(24, 10, 12, F16), 3, 1, {}, "dw", ("dw", 'fast')),
    "dw_fast_W20_bf16_plain": (lambda: dw(7, 5, 20, BF16, bias=False, slope=False), 2, 1, {}, "dw", ("dw", 'fast')),
    "dw_generic_fp32": (lambda: dw(5, 9, 13, F32), 2, 1, {}, "dw", ("dw", 'generic')),
    "pool2_avg_W12": (lambda: mix([(6, 20, 24, F16)], (6, 10, 12, F16), [P(0, 6, 6, ksize=0, pre_avg=1)], bias=False, slope=False), 2, 1, {}, "pool2", ("kernel", 'pool2')),
    "pool2_max_W12_bf16": (lambda: mix([(6, 20, 24, BF16)], (6, 10, 12, BF16), [P(0, 6, 6, ksize=0, pool=2)], bias=False, slope=False), 2, 1, {}, "pool2", ("kernel", 'pool2')),
    "upsample_x2_W12": (lambda: mix([(5, 3, 6, F16)], (5, 6, 12, F16), [P(0, 5, 5, ksize=0, up=2)], bias=False, slope=False), 2, 1, {}, "pool2", ("kernel", 'upsample')),
    "upsample_x4_c0_bf16": (lambda: mix([(9, 3, 3, BF16)], (4, 12, 12, BF16), [P(0, 4, 4, c0=5, ksize=0, up=4)], bias=False, slope=False), 2, 1, {}, "pool2", ("kernel", 'upsample')),
    "upsample_x8_W8": (lambda: mix([(3, 2, 1, F16)], (3, 16, 8, F16), [P(0, 3, 3, ksize=0, up=8)], bias=False, slope=False), 2, 1, {}, "pool2", ("kernel", 'upsample')),
    "resample_fp32_bias_slope": (lambda: mix([(4, 5, 7, F32)], (4, 20, 28, F32), [P(0, 4, 4, ksize=0, up=4)]), 2, 1, {}, "pool2", ("kernel", 'resample')),
    "resample_avg_c0_fp16": (lambda: mix([(8, 16, 24, F16)], (3, 8, 12, F16), [P(0, 3, 3, c0=4, ksize=0, pre_avg=1)], bias=False, slope=False), 2, 1, {}, "pool2", ("kernel", 'resample')),
    "mix_generic_fp32": (lambda: mix([(9, 16, 20, F32), (5, 8, 10, F32)], (19, 8, 10, F32),
                                     [P(0, 9, 19, pre_avg=1, ksize=3, pad=1), P(1, 5, 19, ksize=3, pad=2, dil=2),
                                      P(0, 9, 9, cout0=3, ksize=0, pool=2)]), 2, 1, {}, "mix_generic"),
    "mix_generic_stride2": (lambda: mix([(6, 16, 20, F16)], (8, 8, 10, F16), [P(0, 6, 8, ksize=3, pad=1, stride=2)]), 2, 1, {}, "mix_generic"),
    # GroupNorm
    "gn_g1_fp32": (lambda: gn(16, 6, 10, F32, 1), 2, 1, {}, "gn"),
    "gn_g4_fp16_no_prelu": (lambda: gn(64, 7, 9, F16, 4, slope=False), 3, 1, {}, "gn"),
    "gn_g32_fp16": (lambda: gn(128, 16, 16, F16, 32), 2, 1, {}, "gn"),
    "gn_g32_fp32_no_prelu": (lambda: gn(64, 5, 5, F32, 32, slope=False), 2, 1, {}, "gn"),
}


@pytest.mark.parametrize("case_id", list(CASES))
def test_one_op_kernel_matches_float64(case_id):
    build, max_batch, n_small, env, kernel, *geometry = CASES[case_id]
    prog = build()
    for name, want in geometry:                     # the choice op_kernel does not report, by the plan's own rule
        assert GEOMETRY[name](prog, prog.ops[0]) == want, (case_id, name)
    run_case(case_id, prog, max_batch(prog) if callable(max_batch) else max_batch, n_small, env, kernel)


def test_cases_reach_every_geometry_branch():
    """Every il_block / mix_stream / mix_tc / dw / resample case names its geometry, and together they reach: every
    (tile, chunked) pair plan_il can choose, mix_stream chunk heights 1 / 2 / 4 / 8 / 16, mix_tc mt 1..5, rows 1 / 2 / 4 and
    kc 8 / 16 / 32, both depthwise kernels and the three resample kernels."""
    seen = collections.defaultdict(set)
    for cid, (_b, _m, _n, _e, kernel, *geometry) in CASES.items():
        if kernel in ("il_block", "mix_stream", "mix_tc", "dw", "pool2"):
            assert geometry, cid
        for name, want in geometry:
            seen[name].add(want)
    reachable = {(th, tw, ch) for th, tw in IL_TILES for ch in (False, True)} - {(16, 64, True)}
    assert seen["tile"] == reachable
    assert seen["rows"] >= {1, 2, 4, 8, 16}
    assert {g[0] for g in seen["tc"]} == {1, 2, 3, 4, 5}
    assert {g[1] for g in seen["tc"]} == {1, 2, 4} and {g[2] for g in seen["tc"]} == {8, 16, 32}
    assert seen["dw"] == {"fast", "generic"} and seen["kernel"] == {"pool2", "upsample", "resample"}


# ---- (b) the shipped programs, op by op ----------------------------------------------------------------------------------
def check_program(prog, max_batch, N, ext_inputs, label, env=None):
    """Run `prog` at batch N; every op's output against the reference of its stored inputs.  Returns the op kernels."""
    plan = plan_with(prog, max_batch, env or {})
    try:
        outs = {}
        ext = [None] * (1 + max(t.external for t in prog.tensors))
        for i, x in ext_inputs.items():
            ext[i] = x.cuda().contiguous()
        for t in prog.tensors:
            if t.external >= 0 and ext[t.external] is None:
                ext[t.external] = torch.full((N, t.C, t.H, t.W), float("nan"), dtype=TORCH_DT[t.dtype], device="cuda")
        plan.run(N, [a.data_ptr() for a in ext], torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()

        def read(t):
            if t not in outs:
                d = prog.tensors[t]
                outs[t] = (ext[d.external].float() if d.external >= 0 else plan.read_tensor(t, N)).cpu().to(torch.float64)
            return outs[t]

        kernels = []
        for k, o in enumerate(prog.ops):
            kern = plan.op_kernel(k)
            kernels.append(kern)
            refs = opref(prog, k, {q.src: read(q.src) for q in o.paths})
            for t, (ref, bound) in refs.items():
                q, msg = check(read(t), ref, bound)
                _note(kern, f"{label}:{o.name}", q)
                assert q <= 1.0, (label, k, o.name, kern, msg)
        return kernels
    finally:
        plan.close()


def _counts(prog, max_batch):
    p = runtime.Plan(prog, max_batch=max_batch)
    try:
        return dict(collections.Counter(p.op_kernel(i) for i in range(len(prog.ops)))), p.launches
    finally:
        p.close()


def _smallest_bench_batch(prog):
    """The smallest max_batch whose kernel choice equals the bs-256 bench plan's (the choice is monotone in max_batch)."""
    want = EXPECTED_KERNELS[("fp16", 256)]
    assert _counts(prog, 256) == want
    lo, hi = 1, 256
    while lo < hi:
        mid = (lo + hi) // 2
        if _counts(prog, mid) == want:
            hi = mid
        else:
            lo = mid + 1
    return lo


def _images(N, h, w, seed):
    return {0: torch.from_numpy(synth.randn_images(N, h, w, seed))}


def test_bench_program_op_by_op_at_the_streaming_kernel_choice():
    cfg, sd = fixtures.checkpoint("csnet-L-x2")
    mb = _smallest_bench_batch(compiler.compile_csnet(cfg, sd, 224, 224, "fp16"))
    prog = compiler.compile_csnet(cfg, sd, 224, 224, "fp16", reuse_arena=False)
    kernels = check_program(prog, mb, 2, _images(2, 224, 224, 41), f"csnet-L-x2/fp16/mb{mb}")
    assert dict(collections.Counter(kernels)) == EXPECTED_KERNELS[("fp16", 256)][0]


def test_bench_program_op_by_op_at_max_batch_2():
    cfg, sd = fixtures.checkpoint("csnet-L-x2")
    prog = compiler.compile_csnet(cfg, sd, 224, 224, "fp16", reuse_arena=False)
    kernels = check_program(prog, 2, 2, _images(2, 224, 224, 42), "csnet-L-x2/fp16/mb2")
    assert dict(collections.Counter(kernels)) == EXPECTED_KERNELS[("fp16", 2)][0]


def test_bf16_program_op_by_op():
    cfg, sd = fixtures.checkpoint("csnet-L-x1")
    prog = compiler.compile_csnet(cfg, sd, 224, 224, "bf16", reuse_arena=False)
    check_program(prog, 2, 2, _images(2, 224, 224, 43), "csnet-L-x1/bf16")


def test_fp32_program_op_by_op():
    cfg, sd = fixtures.checkpoint("csnet-L-x2")
    prog = compiler.compile_csnet(cfg, sd, 224, 224, "fp32", reuse_arena=False)
    kernels = check_program(prog, 2, 2, _images(2, 224, 224, 44), "csnet-L-x2/fp32")
    assert set(kernels) <= {"mix_generic_kernel", "pool2 / upsample / resample kernels", "dw kernels"}


@pytest.mark.parametrize("dtype", ["fp32", "fp16"])
def test_csf_head_op_by_op(dtype):
    import json

    z = np.load(os.path.join(fixtures.GOLDEN, "csf_res2net.npz"))
    meta = json.loads(str(z["__meta__"]))
    sd = synth.synth_state_r({k: tuple(v) for k, v in meta["shapes"].items()}, meta["seed"])
    h = w = 96
    dims = [(256, h // 4, w // 4), (512, h // 8, w // 8), (1024, h // 16, w // 16), (2048, h // 32, w // 32)]
    prog = compiler_r.compile_csf_head(sd, dims, h, w, dtype, reuse_arena=False)
    rng = np.random.default_rng(45)
    dt = ir.DTYPE_NAMES[dtype]
    feats = {i: values(rng, (2,) + d, dt).abs() * 0.5 for i, d in enumerate(dims)}      # post-ReLU backbone features
    kernels = check_program(prog, 2, 2, feats, f"csf_head/{dtype}")
    assert "gn kernels" in kernels
