"""CSF+Res2Net training from a set kept on the device: csnet_csf_train_batch_u8 against the reference's ImageDataTrain golden and the
host emulation (bit for bit), csnet_train_bce_sum against float64, and CSFTrainer against solver.train's loop restated on the host
(the module's autograd path, F.binary_cross_entropy_with_logits(sum), torch.optim.Adam, net.zero_grad() at epoch start)."""
import ctypes as C
import json
import math
import os
import random
import subprocess

import numpy as np
import pytest
import torch

from sod100k_b200 import runtime, synth
from sod100k_b200 import train_ops as TO
from sod100k_b200 import trainer as TR
from sod100k_b200.data import SalImages, csf_flip
from sod100k_b200.networks import csf_res2net
from tests import csf_ref, fixtures
from tests.test_csf_train_data_cpu import TAGS, caller_mask, emu_sample

pytestmark = pytest.mark.gpu
DEV = "cuda"
EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")


@pytest.fixture
def deterministic():
    """cuDNN deterministic, no autotuning, TF32 off; restored afterwards."""
    old = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32,
           torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32,
     torch.backends.cuda.matmul.allow_tf32) = old


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu") / "libcsf_train_emu.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-o", out, os.path.join(EMU, "csf_train_emu.cpp")], check=True)
    lib = C.CDLL(out)
    lib.csnet_emu_csf_train_sample.argtypes = [C.c_void_p] * 2 + [C.c_int] * 3 + [C.c_void_p] * 4
    return lib


@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(fixtures.GOLDEN, "csf_train_data.npz"))
    return z, json.loads(str(z["__meta__"]))


def _bits(t):
    return t.detach().cpu().numpy().view(np.uint32)


# ---- (1) the sample kernel ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", TAGS)
def test_sample_kernel_matches_golden_and_emulation(lib, golden, tag):
    z, _ = golden
    for kind in ("L", "rgb"):
        img, mask = z[f"{tag}/image"], caller_mask(z, tag, kind)
        ds = SalImages([z["gray/gray"] if tag == "gray" else img], [mask])
        for flip in (0, 1):
            x, t = ds.csf_train_batch([0], flips=[flip])
            torch.cuda.synchronize()
            key = f"{tag}/{kind}/flip{flip}"
            assert x.shape == (1, 3) + img.shape[:2] and t.shape == (1, 1) + img.shape[:2]
            assert np.array_equal(_bits(x[0]), z[f"{key}/x"].view(np.uint32)), key
            assert np.array_equal(_bits(t[0]), z[f"{key}/t"].view(np.uint32)), key
            ex, et = emu_sample(lib, img, mask, flip)
            assert np.array_equal(_bits(x[0]), ex.view(np.uint32)) and np.array_equal(_bits(t[0]), et.view(np.uint32)), key
        x, t = ds.csf_train_batch([0])                 # neither rng nor flips: no flip
        assert torch.equal(x[0].cpu(), torch.from_numpy(z[f"{tag}/{kind}/flip0/x"]))


def test_sample_kernel_batch_of_one_size(lib):
    g = np.random.default_rng(7)
    sizes = [(37, 53), (20, 30), (37, 53), (37, 53), (75, 100), (37, 53)]
    imgs = [g.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]
    masks = [g.integers(0, 256, (h, w), dtype=np.uint8) for h, w in sizes]
    ds = SalImages(imgs, masks)
    idx = [5, 0, 3, 0, 2]
    x, t = ds.csf_train_batch(idx, random.Random(11))
    r = random.Random(11)
    want = [csf_flip(r) for _ in idx]
    assert set(want) == {0, 1}
    for n, (i, f) in enumerate(zip(idx, want)):
        ex, et = emu_sample(lib, imgs[i], masks[i], f)
        assert np.array_equal(_bits(x[n]), ex.view(np.uint32)) and np.array_equal(_bits(t[n]), et.view(np.uint32)), n
    x2, t2 = ds.csf_train_batch(idx, flips=want)
    assert torch.equal(x2, x) and torch.equal(t2, t)


def test_sample_kernel_rejects_bad_arguments():
    g = np.random.default_rng(8)
    sizes = [(8, 8), (8, 9)]
    ds = SalImages([g.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes],
                   [g.integers(0, 256, (h, w), dtype=np.uint8) for h, w in sizes])
    for kw in (dict(indices=[0, 1]), dict(indices=[0], flips=[2]), dict(indices=[0], flips=[-1]), dict(indices=[0, 0], flips=[1]),
               dict(indices=[0], flips=[0.5]), dict(indices=[2]), dict(indices=[-1]), dict(indices=[]),
               dict(indices=[0], flips=[0], rng=random.Random(0))):
        with pytest.raises(ValueError):
            ds.csf_train_batch(**kw)
    lib = runtime.load_library()
    x = torch.empty((1, 3, 8, 8), device=DEV)
    t = torch.empty((1, 1, 8, 8), device=DEV)
    s = torch.zeros(24, dtype=torch.uint8, device=DEV)
    m, sd = (C.c_double * 3)(0.5, 0.5, 0.5), (C.c_double * 3)(0.2, 0.2, 0.2)
    ok = [ds.x.data_ptr(), ds.m.data_ptr(), ds.geom.data_ptr(), s.data_ptr(), 1, 8, 8, m, sd, x.data_ptr(), t.data_ptr(), None]
    for k, bad in ((0, None), (1, None), (3, None), (4, 0), (4, 65536), (5, 0), (6, 32768), (7, None), (10, None)):
        args = list(ok)
        args[k] = bad
        assert lib.csnet_csf_train_batch_u8(*args) == -1, k
    assert lib.csnet_csf_train_batch_u8(*ok) == 0
    torch.cuda.synchronize()


# ---- (2) the summed BCE ----------------------------------------------------------------------------------------------------------
def bce_sum_ref(z, t, divisor, defect=None):
    """float64 reference and per-element bounds of csnet_train_bce_sum.  loss: the sum of the fp32 terms' float64 values / divisor,
    bound (n + 4) 2^-24 sum(|max(z, 0)| + |z t| + log1p(exp(-|z|))) / divisor (n for the summation chain, 4 for evaluating one term).
    dlogits: (sigmoid(z) - t) * f32(1 / divisor), bound (4 sigmoid + 2 |sigmoid - t|) 2^-24 f32(1 / divisor) + 2^-149.
    defect: 'divisor' divides by 2 divisor, 'drop' loses the gradient of the element where it is largest."""
    z64, t64 = z.double(), t.double()
    d = 2 * divisor if defect == "divisor" else divisor
    inv = float(np.float32(1.0 / d))
    terms = z64.clamp_min(0) - z64 * t64 + torch.log1p(torch.exp(-z64.abs()))
    mag = z64.clamp_min(0) + (z64 * t64).abs() + torch.log1p(torch.exp(-z64.abs()))
    n = z.numel()
    loss = terms.sum().item() / d
    loss_bound = (n + 4) * 2.0 ** -24 * mag.sum().item() / divisor
    sig = torch.sigmoid(z64)
    dl = (sig - t64) * inv
    if defect == "drop":
        dl.view(-1)[int(dl.abs().argmax())] = 0.0
    dl_bound = (4 * sig + 2 * (sig - t64).abs()) * 2.0 ** -24 * float(np.float32(1.0 / divisor)) + 2.0 ** -149
    return loss, loss_bound, dl, dl_bound


def _bce_case(shape, label, seed):
    g = torch.Generator().manual_seed(seed)
    z = (torch.randn(shape, generator=g) * 4).to(DEV)
    t = torch.rand(shape, generator=g) if label == "soft" else (torch.rand(shape, generator=g) > 0.5).float()
    return z, t.to(DEV)


def _bce_sum(z, t, divisor):
    loss = torch.empty(1, device=DEV)
    dl = torch.full_like(z, float("nan"))
    runtime.train_bce_sum(z.data_ptr(), t.data_ptr(), dl.data_ptr(), loss.data_ptr(), z.numel(), divisor,
                          torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return loss, dl


@pytest.mark.parametrize("label", ["soft", "hard"])
@pytest.mark.parametrize("divisor", [1, 10, 20])
@pytest.mark.parametrize("shape", [(1, 1, 1, 1), (1, 1, 75, 100), (1, 1, 520, 520), (4, 1, 64, 64)])
def test_bce_sum_vs_float64(shape, divisor, label):
    z, t = _bce_case(shape, label, sum(shape) + divisor)
    loss, dl = _bce_sum(z, t, divisor)
    loss2, dl2 = _bce_sum(z, t, divisor)
    assert torch.equal(loss, loss2) and torch.equal(dl, dl2), "not bit-identical run to run"
    ref, lb, rdl, dlb = bce_sum_ref(z, t, divisor)
    assert abs(loss.item() - ref) <= lb, (loss.item(), ref, lb)
    assert ((dl.double() - rdl).abs() <= dlb).all()
    torch_loss = torch.nn.functional.binary_cross_entropy_with_logits(z, t, reduction="sum") / divisor
    assert abs(torch_loss.item() - ref) <= lb
    # injected defects exceed the bounds
    ref_d, _, _, _ = bce_sum_ref(z, t, divisor, defect="divisor")
    assert abs(loss.item() - ref_d) > lb
    _, _, rdl_d, _ = bce_sum_ref(z, t, divisor, defect="drop")
    assert not ((dl.double() - rdl_d).abs() <= dlb).all()


def test_new_kernels_are_reached():
    """Every kernel bce_sum.cuh defines, and the sample kernel, runs in this file's checks (the CSNet training suite covers
    train_ops.cu's own kernels)."""
    import re

    from torch.profiler import ProfilerActivity, profile

    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sod100k_b200", "csrc")
    names = set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)", open(os.path.join(root, "bce_sum.cuh")).read()))
    names.add("csf_train_batch_u8_kernel")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        test_bce_sum_vs_float64((1, 1, 75, 100), 10, "soft")
        ds = SalImages([np.zeros((4, 6, 3), np.uint8)], [np.zeros((4, 6), np.uint8)])
        ds.csf_train_batch([0], flips=[1])
        torch.cuda.synchronize()
    seen = " ".join(e.name for e in prof.events())
    assert len(names) == 3 and all(nm in seen for nm in names), sorted(nm for nm in names if nm not in seen)


def test_bce_sum_function_and_bad_arguments():
    z, t = _bce_case((2, 1, 33, 17), "soft", 3)
    zz = z.clone().requires_grad_(True)
    loss = TO.BceSumFn.apply(zz, t, 7)
    loss.backward()
    ref = z.clone().requires_grad_(True)
    (torch.nn.functional.binary_cross_entropy_with_logits(ref, t, reduction="sum") / 7).backward()
    assert abs(loss.item() - (torch.nn.functional.binary_cross_entropy_with_logits(z, t, reduction="sum") / 7).item()) <= 1e-5 * loss.item()
    assert (zz.grad - ref.grad).abs().max().item() <= 1e-6 * ref.grad.abs().max().item()
    lib = runtime.load_library()
    out = torch.empty(1, device=DEV)
    for args in ((None, t.data_ptr(), None, out.data_ptr(), 4, 1), (z.data_ptr(), t.data_ptr(), None, out.data_ptr(), 0, 1),
                 (z.data_ptr(), t.data_ptr(), None, out.data_ptr(), 4, 0), (z.data_ptr(), t.data_ptr(), None, None, 4, 1)):
        assert lib.csnet_train_bce_sum(*args, None) == -1
    with pytest.raises(ValueError):
        TO.BceSumFn.apply(zz, t[:1], 7)


# ---- (3) CSFTrainer against solver.train ----------------------------------------------------------------------------------------
SIZES = [(64, 64), (75, 100), (24, 130), (64, 64), (75, 100)]
ORDERS = [[0, 1, 2, 3, 4], [3, 1, 4, 0, 2]]          # each epoch's loader order
SEEDS = [101, 202]                                   # each epoch's worker seed
ITER, LR, WD = 3, 5e-5, 5e-4


def _net(seed=21):
    m = csf_res2net.build_model()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.synth_state_r(shapes, seed).items()})
    return m.to(DEV).eval()


def _set():
    g = np.random.default_rng(5)
    imgs = [g.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in SIZES]
    masks = []
    for h, w in SIZES:
        m = ((g.random((h, w)) > 0.6) * 255).astype(np.uint8)
        edge = g.random((h, w)) < 0.1                    # antialiased GT edges: soft labels
        m[edge] = g.integers(1, 255, int(edge.sum()))
        masks.append(m)
    return imgs, masks


def host_sample(img, mask, flip):
    """ImageDataTrain.__getitem__ on decoded arrays: load_image, load_sal_label, cv_random_flip, torch.Tensor, .cuda()."""
    x = csf_ref.load_image_test(img)
    t = (np.array(mask, dtype=np.float32) / 255.)[np.newaxis, ...]
    if flip == 1:
        x, t = x[:, :, ::-1].copy(), t[:, :, ::-1].copy()
    return torch.Tensor(x)[None].cuda(), torch.Tensor(t)[None].cuda()


def solver_train(net, imgs, masks, epochs=2, decay=(0,)):
    """solver.py:81-127 restated on host samples; records every micro-step's loss and, at each Adam step, the gradients, the
    parameters before and after, lr, and the bias-corrected second moment."""
    params = [p for p in net.parameters() if p.requires_grad]
    lr = LR
    opt = torch.optim.Adam(params, lr=lr, weight_decay=WD)
    rec = {"loss": [], "steps": []}
    ave_grad = 0
    for epoch in range(epochs):
        net.zero_grad()
        rng = random.Random(SEEDS[epoch])
        for i in ORDERS[epoch]:
            x, t = host_sample(imgs[i], masks[i], csf_flip(rng))
            pred = net(x)
            loss = torch.nn.functional.binary_cross_entropy_with_logits(pred, t, reduction="sum") / (ITER * 1)
            rec["loss"].append(loss.item())
            loss.backward()
            ave_grad += 1
            if ave_grad % ITER == 0:
                assert all(p.grad is not None for p in params)
                st = {"grad": [p.grad.clone() for p in params], "before": [p.detach().clone() for p in params], "lr": lr}
                opt.step()
                st["after"] = [p.detach().clone() for p in params]
                st["vhat"] = [opt.state[p]["exp_avg_sq"] / (1 - 0.999 ** float(opt.state[p]["step"])) for p in params]
                rec["steps"].append(st)
                opt.zero_grad()
                ave_grad = 0
        if epoch in decay:
            lr = lr * 0.1
            opt = torch.optim.Adam(params, lr=lr, weight_decay=WD)
    return rec


def csf_trainer_run(net, ds, ref, trainer_cls=TR.CSFTrainer, epochs=2, decay=(0,)):
    """The same loop on CSFTrainer fed by SalImages.csf_train_batch; FusedAdam.step is wrapped to record what solver_train does.  In
    lockstep with the reference run `ref`: after its k-th Adam step the net continues from the reference's parameters after step k
    (the moments stay FusedAdam's own), so that last-bit differences between the two Adam implementations do not compound through
    the backbone's max-pool and ReLU routing into the next steps' gradients."""
    rec = {"loss": [], "steps": []}
    tr = trainer_cls(net, lr=LR, weight_decay=WD, iter_size=ITER, lr_decay_epochs=decay)
    params = tr.flat.params
    real = TO.FusedAdam.step

    def recording_step(opt, *a, **k):
        st = {"grad": [p.grad.clone() for p in params], "before": [p.detach().clone() for p in params]}
        real(opt, *a, **k)
        st["after"] = [p.detach().clone() for p in params]
        k = len(rec["steps"])
        rec["steps"].append(st)
        if k < len(ref["steps"]):
            with torch.no_grad():
                for p, a in zip(params, ref["steps"][k]["after"]):
                    p.copy_(a)

    TO.FusedAdam.step = recording_step
    try:
        for epoch in range(epochs):
            tr.epoch_begin()
            rng = random.Random(SEEDS[epoch])
            for i in ORDERS[epoch]:
                rec["loss"].append(tr.step(*ds.csf_train_batch([i], rng)).item())
            tr.epoch_end(epoch)
    finally:
        TO.FusedAdam.step = real
    return rec


def compare(ref, got):
    """Failures of `got` against `ref`: losses to 1e-5 relative; each Adam step's gradient bucket to 1e-5 of each tensor's rms; each
    step's parameter change per element within lr (2^-16 + 3 d / (sqrt(vhat) + eps)) + 2^-22 |p|, d = 1e-5 of the tensor's largest
    gradient rms over the steps (the change a gradient error of d can make in Adam's m / sqrt(v), plus fp32 rounding of the update
    and of p)."""
    bad = []
    if len(got["loss"]) != len(ref["loss"]):
        return [f"{len(got['loss'])} micro-steps, reference {len(ref['loss'])}"]
    for k, (a, b) in enumerate(zip(got["loss"], ref["loss"])):
        if abs(a - b) > 1e-5 * abs(b):
            bad.append(f"loss {k}: {a} vs {b}")
    if len(got["steps"]) != len(ref["steps"]):
        return bad + [f"{len(got['steps'])} Adam steps, reference {len(ref['steps'])}"]
    rms = [max(s["grad"][j].double().pow(2).mean().sqrt().item() for s in ref["steps"]) for j in range(len(ref["steps"][0]["grad"]))]
    for k, (g, r) in enumerate(zip(got["steps"], ref["steps"])):
        for j, (ga, gr) in enumerate(zip(g["grad"], r["grad"])):
            rj = gr.double().pow(2).mean().sqrt().item()
            if (ga.double() - gr.double()).abs().max().item() > 1e-5 * rj + 1e-30:
                bad.append(f"step {k} tensor {j}: gradient")
                break
        for j in range(len(r["grad"])):
            d_got = (g["after"][j] - g["before"][j]).double()
            d_ref = (r["after"][j] - r["before"][j]).double()
            bound = r["lr"] * (2.0 ** -16 + 3e-5 * rms[j] / (r["vhat"][j].double().sqrt() + 1e-8)) + 2.0 ** -22 * r["before"][j].double().abs()
            if ((d_got - d_ref).abs() > bound).any():
                q = ((d_got - d_ref).abs() / bound).max().item()
                bad.append(f"step {k} tensor {j}: parameter change, q = {q:.3g}")
                break
    return bad


@pytest.fixture(scope="module")
def reference_run():
    old = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32 = True, False, False
    try:
        imgs, masks = _set()
        net = _net()
        frozen = {k: p.detach().clone() for k, p in net.named_parameters() if not p.requires_grad}
        rec = solver_train(net, imgs, masks)
        yield imgs, masks, rec, frozen
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32 = old


def test_csf_trainer_matches_solver_train(deterministic, reference_run):
    imgs, masks, ref, frozen = reference_run
    # 5 items a epoch, iter_size 3: steps after micro-steps 3, 6 (epoch 1's first, summing only its first item) and 9
    assert len(ref["loss"]) == 10 and len(ref["steps"]) == 3
    net = _net()
    got = csf_trainer_run(net, SalImages(imgs, masks), ref)
    assert compare(ref, got) == []
    for k, p in net.named_parameters():
        if k in frozen:
            assert torch.equal(p.detach(), frozen[k]), k
    assert frozen


class _SkipsAStep(TR.CSFTrainer):
    def _adam(self):
        opt = super()._adam()
        real, calls = opt.step, [0]

        def step(*a, **k):
            calls[0] += 1
            if calls[0] != 2:
                real(*a, **k)
        opt.step = step
        return opt


class _WrongDivisor(TR.CSFTrainer):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.divisor = 1                               # the loss summed, not averaged over the accumulation


class _KeepsPartial(TR.CSFTrainer):
    def epoch_begin(self):
        pass


class _NoResetAtDecay(TR.CSFTrainer):
    def epoch_end(self, epoch):
        if self.schedule.epoch_end(epoch):
            self.opt.lr = self.schedule.lr


@pytest.mark.parametrize("defect", [_SkipsAStep, _WrongDivisor, _KeepsPartial, _NoResetAtDecay])
def test_compare_flags_schedule_defects(deterministic, reference_run, defect):
    imgs, masks, ref, _ = reference_run
    got = csf_trainer_run(_net(), SalImages(imgs, masks), ref, trainer_cls=defect)
    bad = compare(ref, got)
    assert bad, defect.__name__
    if defect in (_SkipsAStep, _NoResetAtDecay):       # the parameter-change bound alone catches these
        assert any("parameter change" in b or "Adam steps" in b for b in bad), bad


# ---- (4) device-fed against host-fed ---------------------------------------------------------------------------------------------
def test_device_fed_equals_host_fed_and_zero_grad_raises(deterministic, golden):
    z, _ = golden
    items = [("37x53", "L", 0), ("37x53", "rgb", 1), ("75x100", "L", 1), ("75x100", "rgb", 0), ("gray", "L", 1), ("gray", "rgb", 0)]
    packed = [(tag, kind) for tag, kind, _ in items]
    ds = SalImages([z[f"{t}/image"] for t, _ in packed], [caller_mask(z, t, k) for t, k in packed])
    nets = [_net(), _net()]
    trs = [TR.CSFTrainer(n, iter_size=2) for n in nets]
    for tag, kind, flip in items:
        a = trs[0].step(*ds.csf_train_batch([packed.index((tag, kind))], flips=[flip]))
        key = f"{tag}/{kind}/flip{flip}"
        x, t = (torch.from_numpy(z[f"{key}/{c}"])[None].cuda() for c in ("x", "t"))
        b = trs[1].step(x, t)
        assert torch.equal(a, b), key
    for (ka, pa), (_, pb) in zip(nets[0].named_parameters(), nets[1].named_parameters()):
        assert torch.equal(pa, pb), ka
    nets[0].zero_grad()
    with pytest.raises(runtime.EngineError):
        trs[0].step(*ds.csf_train_batch([0]))
    assert math.isfinite(b.item())
