"""The streaming ILBlock kernel (csrc/il_stream.cuh: TMA operand tiles, wgmma GEMM with register accumulators, register-resident
depthwise tail) against the generic ops, the tiled kernel and the oracle.  CSNET_ILS / CSNET_ILS_MIN_CHUNKS / CSNET_ILS_NS are
read when a plan is created, so a test can pin which kernel runs an ILBLOCK op."""
import collections
import os

import numpy as np
import pytest
import torch

from oracle import csnet_oracle as O
from sod100k_b200 import compiler, runtime, synth
from tests import fixtures

pytestmark = pytest.mark.gpu


def _plan(prog, nb, ils, min_chunks=0, ns=0):
    old = {k: os.environ.get(k) for k in ("CSNET_ILS", "CSNET_ILS_MIN_CHUNKS", "CSNET_ILS_NS")}
    os.environ.update({"CSNET_ILS": "1" if ils else "0", "CSNET_ILS_MIN_CHUNKS": str(min_chunks), "CSNET_ILS_NS": str(ns)})
    try:
        return runtime.Plan(prog, max_batch=nb)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.mark.parametrize("tag,hw,nb,ns", [("csnet-L-x2", (224, 224), 3, 0), ("csnet-L-x2", (224, 224), 2, 2), ("csnet-L-x2", (96, 160), 5, 0),
                                          ("csnet-L-x1", (128, 64), 2, 0), ("csnet-L-x1", (128, 256), 2, 2)])
def test_streaming_kernel_one_block_at_a_time(tag, hw, nb, ns):
    """Fuse exactly one ILBlock (inputs bit-identical to the all-generic program) and run it on the streaming kernel: the
    block outputs must agree with the generic ops to a few fp16 ulps of the tensor's magnitude, exactly like the tiled
    kernel.  Small batches make most CTAs start in the middle of an image (warm-up chunk, look-ahead chunk, bottom flush);
    ns = 2 forces two column strips (halo groups, strip-edge handling)."""
    cfg, sd = fixtures.checkpoint(tag)
    h, w = hw
    x = torch.from_numpy(synth.randn_images(nb, h, w, 31)).cuda()
    base = compiler.compile_csnet(cfg, sd, h, w, "fp16", reuse_arena=False, fuse=False, tensor_core=False)
    p0 = _plan(base, nb, False)
    p0.forward(x)
    full = compiler.compile_csnet(cfg, sd, h, w, "fp16", fuse=True)
    names = [o.name for o in full.ops if o.kind == 3]           # 1x1 blocks and the stem form
    ran = 0
    for name in names:
        prog = compiler.compile_csnet(cfg, sd, h, w, "fp16", reuse_arena=False, fuse={name}, tensor_core=False)
        p1 = _plan(prog, nb, True, 0, ns)
        p1.forward(x)
        for b in (0, 1):
            key = f"{name}/{b}"
            if key not in prog.taps:
                continue
            ref, got = p0.read_tensor(base.taps[key], nb), p1.read_tensor(prog.taps[key], nb)
            assert torch.isfinite(got).all(), key
            err = (got - ref).abs().max().item()
            assert err <= 4e-3 * max(1.0, ref.abs().max().item()), (key, err, ref.abs().max().item())
            ran += 1
        p1.close()
    assert ran >= 6


def test_streaming_and_tiled_kernels_agree_on_the_whole_network():
    """Full fp16 program, batch 16 at 224x224: streaming kernel on (every qualifying block) vs off, and vs the oracle."""
    cfg, sd = fixtures.checkpoint("csnet-L-x2")
    xb, _ = synth.blob_images(16, 224, 224, 1235)
    x = torch.from_numpy(xb).cuda()
    prog = compiler.compile_csnet(cfg, sd, 224, 224, "fp16")
    y1 = torch.sigmoid(_plan(prog, 16, True, 0).forward(x)).cpu()
    y0 = torch.sigmoid(_plan(prog, 16, False).forward(x)).cpu()
    # two fp16-storage executions with different rounding points: measured 2.7e-3 on this blob set (r02)
    assert (y1 - y0).abs().max().item() <= 6e-3
    assert (y1 - y0).abs().mean().item() <= 2e-4
    with torch.no_grad():
        ref = torch.sigmoid(O.csnet_forward(cfg, sd, torch.from_numpy(xb[:4])))
    assert (y1[:4] - ref).abs().max().item() <= 2e-2


def test_streaming_kernel_is_deterministic_and_batch_independent():
    cfg, sd = fixtures.checkpoint("csnet-L-x2")
    x = torch.from_numpy(synth.randn_images(4, 224, 224, 5)).cuda().repeat(8, 1, 1, 1)
    prog = compiler.compile_csnet(cfg, sd, 224, 224, "fp16")
    p = _plan(prog, 32, True, 0)
    y, y2 = p.forward(x), p.forward(x)
    assert torch.equal(y, y2)
    assert torch.equal(y[:4], y[20:24])            # the same images at other batch positions (other CTAs, other chunk ranges)
    assert torch.isfinite(y).all()


@pytest.mark.parametrize("tag,hw,nb", [("csnet-L-x2", (224, 224), 24), ("csnet-L-x1", (224, 224), 24), ("csnet-L-x2", (96, 160), 40)])
def test_streaming_mix_kernel_matches_the_tensor_core_mix_kernel(tag, hw, nb):
    """csrc/mix_stream.cuh (TMA -> wgmma -> epilogue with resample-adds / the cls_layer projection) on and off for the same
    fp16 program: taps of the CSF head and the logits.  Both sides run fp16 operands with fp32 accumulation; the differences are
    accumulation order and the 16-bit rounding of the stored taps."""
    cfg, sd = fixtures.checkpoint(tag)
    h, w = hw
    x = torch.from_numpy(synth.randn_images(nb, h, w, 3)).cuda()
    prog = compiler.compile_csnet(cfg, sd, h, w, "fp16", reuse_arena=False)
    os.environ["CSNET_MS"] = "1"
    p1 = runtime.Plan(prog, max_batch=nb)
    os.environ["CSNET_MS"] = "0"
    p0 = runtime.Plan(prog, max_batch=nb)
    os.environ.pop("CSNET_MS")
    y1, y0 = p1.forward(x), p0.forward(x)
    assert torch.isfinite(y1).all()
    # two fp16-storage executions of the whole net: measured <= 1.2e-2 in logit units at |y| ~ 5.5 (r02); the taps below are tight
    assert (y1 - y0).abs().max().item() <= 5e-3 * max(1.0, y0.abs().max().item())
    n = 0
    for name, tid in prog.taps.items():
        if name.startswith("oct_fuse.fuse"):
            a, b = p1.read_tensor(tid, nb), p0.read_tensor(tid, nb)
            assert (a - b).abs().max().item() <= 2e-3 * max(1.0, b.abs().max().item()), name
            n += 1
    assert n >= 2


@pytest.mark.parametrize("tag,hw", [("csnet-L-x2", (224, 224)), ("csnet-L-x1", (224, 224)), ("csnet-L-x2", (96, 160))])
def test_msblock_direct_kernel_matches_generic_ops(tag, hw):
    """csrc/ms_direct.cuh: only the MSBlock ops leave the generic kernels (inputs bit-identical), taps of the three MS branches."""
    cfg, sd = fixtures.checkpoint(tag)
    h, w = hw
    x = torch.from_numpy(synth.randn_images(3, h, w, 5)).cuda()
    base = compiler.compile_csnet(cfg, sd, h, w, "fp16", reuse_arena=False, fuse=False, tensor_core=False)
    prog = compiler.compile_csnet(cfg, sd, h, w, "fp16", reuse_arena=False, fuse=False, tensor_core={"oct_fuse.ms"})
    p0, p1 = runtime.Plan(base, max_batch=3), runtime.Plan(prog, max_batch=3)
    p0.forward(x)
    p1.forward(x)
    n = 0
    for name in ("oct_fuse.ms/0", "oct_fuse.ms/1", "oct_fuse.ms/2"):
        if name in prog.taps:
            a, b = p1.read_tensor(prog.taps[name], 3), p0.read_tensor(base.taps[name], 3)
            assert torch.isfinite(a).all()
            assert (a - b).abs().max().item() <= 4e-3 * max(1.0, b.abs().max().item()), name
            n += 1
    assert n >= 2


def _kernel_counts(dtype, max_batch):
    """(ops per kernel name, launches per forward) of the csnet-L-x2 plan at 224x224 that bench.py and smoke() run."""
    cfg, sd = fixtures.checkpoint("csnet-L-x2")
    p = runtime.Plan(compiler.compile_csnet(cfg, sd, 224, 224, dtype), max_batch=max_batch)
    try:
        return dict(collections.Counter(p.op_kernel(i) for i in range(len(p.prog.ops)))), p.launches
    finally:
        p.close()


# Recorded on an H100 80GB HBM3 (132 SMs) with none of the CSNET_* switches set.
EXPECTED_KERNELS = {
    ("fp16", 256): ({"il_stream_kernel (TMA + wgmma)": 7, "il_block_kernel (mma.sync, tiled)": 5, "mix_stream_kernel (TMA + wgmma)": 8,
                     "mix_tc_kernel (mma.sync)": 15, "msd_kernel (ms_direct.cuh, FP32 pipe)": 2, "pool2 / upsample / resample kernels": 15,
                     "dw kernels": 22}, 81),
    ("fp16", 2): ({"il_block_kernel (mma.sync, tiled)": 12, "mix_tc_kernel (mma.sync)": 23, "msd_kernel (ms_direct.cuh, FP32 pipe)": 2,
                   "pool2 / upsample / resample kernels": 15, "dw kernels": 22}, 81),
    ("fp32", 256): ({"mix_generic_kernel": 61, "pool2 / upsample / resample kernels": 1, "dw kernels": 66}, 128),
}


@pytest.mark.parametrize("dtype,max_batch", list(EXPECTED_KERNELS))
def test_kernel_selection_of_the_bench_plans(dtype, max_batch):
    """Which kernel runs each op is fixed when the plan is created (max_batch and the SM count pick the streaming or the
    tiled / graph-replayed side): pin it for the bench configuration, its small-batch form and the fp32 program."""
    assert _kernel_counts(dtype, max_batch) == EXPECTED_KERNELS[(dtype, max_batch)]
