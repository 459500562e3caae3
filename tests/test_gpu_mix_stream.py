"""The streaming MIX kernel (csrc/mix_stream.cuh: TMA operand and resample-source tiles, wgmma, epilogue) against the same
fp16 program with CSNET_MS=0 (tensor-core / generic kernels), and its independence of where a CTA's chunk range starts.
CSNET_MS is read when a plan is created.  The sizes cover 3x3 ops with a resample path, 1x1 ops with resample paths at
up 2 and up 4, the MIXPROJ head, chunk heights of 1, 2 and 4 rows, and bottom rows whose bilinear taps are clamped."""
import os

import pytest
import torch

from sod100k_b200 import compiler, runtime, synth
from tests import fixtures

pytestmark = pytest.mark.gpu


def _plan(prog, nb, ms):
    old = os.environ.get("CSNET_MS")
    os.environ["CSNET_MS"] = "1" if ms else "0"
    try:
        return runtime.Plan(prog, max_batch=nb)
    finally:
        if old is None:
            os.environ.pop("CSNET_MS", None)
        else:
            os.environ["CSNET_MS"] = old


# nb: enough 2-row chunks at the smallest streaming op's height for the plan to put every eligible op on mix_stream
CASES = [("csnet-L-x2", (224, 224), 12), ("csnet-L-x1", (224, 224), 12), ("csnet-L-x2", (96, 160), 24)]


@pytest.mark.parametrize("tag,hw,nb", CASES)
def test_mix_stream_matches_the_other_kernels(tag, hw, nb):
    cfg, sd = fixtures.checkpoint(tag)
    h, w = hw
    x = torch.from_numpy(synth.randn_images(nb, h, w, 17)).cuda()
    prog = compiler.compile_csnet(cfg, sd, h, w, "fp16", reuse_arena=False)
    p1, p0 = _plan(prog, nb, True), _plan(prog, nb, False)
    try:
        ops = [i for i in range(len(prog.ops)) if p1.op_kernel(i).startswith("mix_stream")]
        assert any(prog.ops[i].kind == 5 for i in ops)                     # the MIXPROJ head
        assert any(sum(q.ksize == 0 for q in prog.ops[i].paths) == 2 for i in ops)   # resample paths at up 2 and up 4
        y1, y0 = p1.forward(x), p0.forward(x)
        torch.cuda.synchronize()
        assert torch.isfinite(y1).all()
        for i in ops:
            d = prog.ops[i].dst
            a, b = p1.read_tensor(d, nb), p0.read_tensor(d, nb)
            err = (a - b).abs().max().item()
            assert err <= 4e-3 * max(1.0, b.abs().max().item()), (prog.ops[i].name, err, b.abs().max().item())
        assert (y1 - y0).abs().max().item() <= 2e-2 * max(1.0, y0.abs().max().item())
    finally:
        p1.close()
        p0.close()


@pytest.mark.parametrize("tag,hw,nb", CASES)
def test_mix_stream_is_batch_independent(tag, hw, nb):
    """The same four images at batch offsets 0 and k: CTAs start mid-image at different chunks, outputs must not change."""
    cfg, sd = fixtures.checkpoint(tag)
    h, w = hw
    k = nb - 5
    x = torch.from_numpy(synth.randn_images(nb, h, w, 23)).cuda()
    x[k:k + 4] = x[:4]
    prog = compiler.compile_csnet(cfg, sd, h, w, "fp16", reuse_arena=False)
    p = _plan(prog, nb, True)
    try:
        ops = [i for i in range(len(prog.ops)) if p.op_kernel(i).startswith("mix_stream")]
        assert ops
        y = p.forward(x)
        torch.cuda.synchronize()
        assert torch.equal(y[:4], y[k:k + 4])
        for i in ops:
            t = p.read_tensor(prog.ops[i].dst, nb)
            assert torch.equal(t[:4], t[k:k + 4]), prog.ops[i].name
    finally:
        p.close()
