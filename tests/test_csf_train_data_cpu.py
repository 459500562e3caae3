"""CSF+Res2Net training without a GPU: the per-pixel sample functions of csf_train_batch_u8_kernel (compiled for the CPU from
image_io.cuh) against the unmodified reference's ImageDataTrain (tests/golden/csf_train_data.npz), csf_flip against the reference's
recorded flips, and CSFTrainer's accumulation / Adam / decay schedule against a counter-level restatement of solver.train."""
import ctypes as C
import json
import os
import random
import subprocess

import numpy as np
import pytest
import torch

from sod100k_b200 import trainer as TR
from sod100k_b200.data import IMAGENET_MEAN, IMAGENET_STD, csf_flip
from sod100k_b200.runtime import EngineError
from tests import fixtures

EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
MEAN, STD = np.array(IMAGENET_MEAN, np.float64), np.array(IMAGENET_STD, np.float64)
TAGS = ["1x1", "3x5", "37x53", "75x100", "gray"]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu") / "libcsf_train_emu.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-o", out, os.path.join(EMU, "csf_train_emu.cpp")], check=True)
    lib = C.CDLL(out)
    lib.csnet_emu_csf_train_sample.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(fixtures.GOLDEN, "csf_train_data.npz"))
    return z, json.loads(str(z["__meta__"]))


def emu_sample(lib, img, mask, flip):
    """(x fp32 [3, h, w], t fp32 [1, h, w]) as csf_train_batch_u8_kernel computes one sample; mask uint8 [h, w]."""
    img, mask = np.ascontiguousarray(img, np.uint8), np.ascontiguousarray(mask, np.uint8)
    h, w = img.shape[:2]
    x, t = np.empty((3, h, w), np.float32), np.empty((1, h, w), np.float32)
    lib.csnet_emu_csf_train_sample(img.ctypes.data, mask.ctypes.data, h, w, int(flip), MEAN.ctypes.data, STD.ctypes.data, x.ctypes.data,
                                   t.ctypes.data)
    return x, t


def caller_mask(z, tag, kind):
    """What a caller packs: np.array(Image.open(gt)), channel 0 of a 3-D array (load_sal_label)."""
    m = z[f"{tag}/mask_{kind}"]
    return m[:, :, 0] if m.ndim == 3 else m


@pytest.mark.parametrize("flip", [0, 1])
@pytest.mark.parametrize("kind", ["L", "rgb"])
@pytest.mark.parametrize("tag", TAGS)
def test_sample_matches_image_data_train_bit_for_bit(lib, golden, tag, kind, flip):
    z, _ = golden
    key = f"{tag}/{kind}/flip{flip}"
    x, t = emu_sample(lib, z[f"{tag}/image"], caller_mask(z, tag, kind), flip)
    assert z[f"{key}/x"].dtype == np.float32 and z[f"{key}/t"].dtype == np.float32
    assert np.array_equal(x.view(np.uint32), z[f"{key}/x"].view(np.uint32))
    assert np.array_equal(t.view(np.uint32), z[f"{key}/t"].view(np.uint32))
    if kind == "rgb":                                  # the GT's channels differ, so channel 0 is what the label pins
        m = z[f"{tag}/mask_rgb"]
        assert m.ndim == 3 and (m.shape[:2] == (1, 1) or not np.array_equal(m[:, :, 0], m[:, :, 1]))
    if tag == "gray":
        assert np.array_equal(np.repeat(z["gray/gray"][:, :, None], 3, axis=2), z["gray/image"])


def test_flip_reverses_columns_only(lib, golden):
    z, _ = golden
    img, m = z["75x100/image"], caller_mask(z, "75x100", "L")
    x0, t0 = emu_sample(lib, img, m, 0)
    x1, t1 = emu_sample(lib, img, m, 1)
    assert np.array_equal(x1, x0[:, :, ::-1]) and np.array_equal(t1, t0[:, :, ::-1])
    assert not np.array_equal(x1, x0)


def test_csf_flip_replays_the_reference_draws(golden):
    z, meta = golden
    rng = random.Random(meta["draw_seed"])
    assert [csf_flip(rng) for _ in range(meta["draw_items"])] == z["draws"].tolist()
    assert set(z["draws"].tolist()) == {0, 1}
    for tag in TAGS:                                   # each recorded sample's own seed gives its flip
        for kind in ("L", "rgb"):
            for flip in (0, 1):
                assert csf_flip(random.Random(int(z[f"{tag}/{kind}/flip{flip}/seed"]))) == flip


# ---- the schedule ------------------------------------------------------------------------------------------------------------------
def solver_train_restated(epochs, items, iter_size, decay):
    """solver.py:81-127 at counter level: each micro-step's gradient is the set {its index}; net.zero_grad() / optimizer.zero_grad()
    empty the accumulation; a new Adam starts at step 1.  Returns one (summed micro-steps, lr, Adam's own step count) per Adam step."""
    lr, ave_grad, adam_steps, grad, out, k = 5e-5, 0, 0, set(), [], 0
    for epoch in range(epochs):
        grad = set()                                   # self.net.zero_grad()
        for _ in range(items):
            grad = grad | {k}                          # sal_loss.backward()
            k += 1
            ave_grad += 1
            if ave_grad % iter_size == 0:
                adam_steps += 1
                out.append((frozenset(grad), lr, adam_steps))
                grad = set()                           # self.optimizer.zero_grad()
                ave_grad = 0
        if epoch in decay:
            lr = lr * 0.1
            adam_steps = 0                             # a new Adam(...)
    return out


class _OneHotNet(torch.nn.Module):
    """logits = w[k] for micro-step k's one-hot input: micro-step k's gradient lives in w[k] alone."""

    def __init__(self, n):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(n))
        self.frozen = torch.nn.Parameter(torch.zeros(3), requires_grad=False)

    def forward(self, x):
        return (x * self.w).sum().reshape(1, 1, 1, 1)


class _SumBce(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z, t, divisor):
        ctx.save_for_backward(z, t)
        ctx.divisor = divisor
        return torch.nn.functional.binary_cross_entropy_with_logits(z, t, reduction="sum") / divisor

    @staticmethod
    def backward(ctx, g):
        z, t = ctx.saved_tensors
        return (torch.sigmoid(z) - t) / ctx.divisor * g, None, None


class _RecordingAdam:
    """Stands in for FusedAdam: records which micro-steps the bucket holds, lr and its own step count at each step."""
    log = []

    def __init__(self, groups, lr, betas, eps):
        (self.params, self.wd), = groups
        self.lr, self.step_count = lr, 0
        assert betas == (0.9, 0.999) and eps == 1e-8

    def step(self):
        self.step_count += 1
        g = self.params[0].grad
        _RecordingAdam.log.append((frozenset(torch.nonzero(g).reshape(-1).tolist()), self.lr, self.step_count))


@pytest.mark.parametrize("epochs,items,iter_size,decay", [(3, 7, 3, (0,)), (2, 5, 3, (0,)), (2, 10, 10, (15,)), (4, 4, 5, (1, 2)),
                                                           (2, 3, 1, (0,))])
def test_schedule_matches_solver_train(monkeypatch, epochs, items, iter_size, decay):
    monkeypatch.setattr(TR.T, "BceSumFn", _SumBce)
    monkeypatch.setattr(TR.T, "FusedAdam", _RecordingAdam)
    _RecordingAdam.log = []
    n = epochs * items
    net = _OneHotNet(n)
    tr = TR.CSFTrainer(net, iter_size=iter_size, lr_decay_epochs=decay)
    assert tr.divisor == iter_size and tr.flat.params == [net.w]
    k = 0
    for epoch in range(epochs):
        tr.epoch_begin()
        for _ in range(items):
            x = torch.zeros(n)
            x[k] = 1.0
            tr.step(x, torch.ones(1, 1, 1, 1))
            k += 1
        tr.epoch_end(epoch)
    ref = solver_train_restated(epochs, items, iter_size, decay)
    got = _RecordingAdam.log
    assert [(s, st) for s, _, st in got] == [(s, st) for s, _, st in ref]
    assert all(a == pytest.approx(b, rel=1e-15) for (_, a, _), (_, b, _) in zip(got, ref))
    if items % iter_size:                              # an epoch's first step sums fewer than iter_size micro-steps
        assert any(len(s) < iter_size for s, _, _ in ref)


def test_batch_size_divides_the_loss(monkeypatch):
    monkeypatch.setattr(TR.T, "BceSumFn", _SumBce)
    monkeypatch.setattr(TR.T, "FusedAdam", _RecordingAdam)
    tr = TR.CSFTrainer(_OneHotNet(4), iter_size=10, batch_size=4)
    assert tr.divisor == 40
    with pytest.raises(ValueError):
        TR.CSFTrainer(_OneHotNet(4), iter_size=0)


def test_zero_grad_between_steps_raises(monkeypatch):
    monkeypatch.setattr(TR.T, "BceSumFn", _SumBce)
    monkeypatch.setattr(TR.T, "FusedAdam", _RecordingAdam)
    net = _OneHotNet(4)
    tr = TR.CSFTrainer(net, iter_size=3)
    x = torch.tensor([1.0, 0, 0, 0])
    tr.step(x, torch.ones(1, 1, 1, 1))
    assert net.w.grad[0] != 0
    net.zero_grad()
    with pytest.raises(EngineError):
        tr.step(x, torch.ones(1, 1, 1, 1))
