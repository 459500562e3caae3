"""CSF+Res2Net training on the GPU: every new kernel against float64 element by element (twice, bit-identical), kernel coverage, the
whole head against float64 autograd of the oracle, the module against the reference's golden training step, and inference after it."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import csf_res2net_oracle as R
from sod100k_b200 import modular_r as M
from sod100k_b200 import synth
from sod100k_b200.networks import csf_res2net
from tests import fixtures
from tests import trainref_r as T

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture
def no_tf32():
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


def _rand(g, *shape):
    return torch.from_numpy(g.standard_normal(shape).astype(np.float32)).to(DEV)


def _ok(got, ref_bound, label):
    ref, bound = ref_bound
    q, where = T_check(got, ref, bound)
    assert q <= 1.0, (label, where)
    return q


def T_check(got, ref, bound):
    got = got.detach().double().to(ref.device)
    r = (got - ref).abs() / bound
    r = torch.where(torch.isfinite(got), r, torch.full_like(r, float("inf")))
    i = int(torch.argmax(r.reshape(-1)))
    return float(r.reshape(-1)[i]), f"q={float(r.reshape(-1)[i]):.3g} at flat {i} of {tuple(r.shape)}"


def _flagged(got, ref_bound):
    ref, bound = ref_bound
    return T_check(got, ref, bound)[0] > 1.0


def _twice(fn):
    a = fn()
    b = fn()
    assert torch.equal(a, b), "not bit-identical run to run"
    return a


# ---- (1) GEMM forms ------------------------------------------------------------------------------------------------------------
# (N images, H, W, cins per segment, cout, k, dil, splits, tile)
GEMM_CASES = [
    (1, 11, 11, [256, 512, 1024], 128, 1, 1, 0, 0),      # fuse.0-like at 11^2, several segments, auto split
    (2, 7, 9, [37, 20], 70, 1, 1, 1, 1),                 # M, N, K not tile multiples, no split
    (2, 7, 9, [37, 20], 70, 1, 1, 5, 1),                 # same, split-K on
    (1, 13, 10, [300], 1, 1, 1, 0, 0),                   # Cout = 1 (cls_layer)
    (1, 12, 12, [200], 150, 1, 1, 3, 2),                 # 128x128 tile, split
    (2, 6, 5, [33], 21, 3, 1, 1, 1),                     # 3x3 d = 1
    (1, 5, 6, [40], 25, 3, 8, 0, 0),                     # d >= plane: only the centre tap lands
    (1, 22, 22, [128], 130, 3, 4, 2, 2),                 # 3x3 big tile, split
    (1, 4, 3, [20], 9, 3, 16, 1, 1),
]


def _gemm_inputs(case, seed):
    n, h, w, cins, cout, k, dil, sp, tile = case
    g = np.random.default_rng(seed)
    xs = [_rand(g, n, c, h, w) for c in cins]
    ws = [_rand(g, cout, c, k, k) * (1.0 / np.sqrt(c * k * k)) for c in cins]
    return xs, ws


@pytest.mark.parametrize("case", GEMM_CASES)
def test_conv_fwd_dgrad_wgrad_vs_float64(case):
    n, h, w, cins, cout, k, dil, sp, tile = case
    xs, ws = _gemm_inputs(case, 11 + GEMM_CASES.index(case))
    g = np.random.default_rng(7)
    bias = _rand(g, cout) if k == 1 and len(cins) == 1 else None
    old = _rand(g, n, cout, h, w)
    segs = [M.seg(x, wt, 0, cout, 0, x.shape[1], dil=dil) for x, wt in zip(xs, ws)]
    splits, chain, _ = M.conv_plan(0, n, h, w, segs, sp, tile)

    def fwd():
        y = old.clone()
        M.conv_fwd(y, segs, bias=bias.data_ptr() if bias is not None else None, accumulate=True, splits_=sp, tile=tile)
        return y
    y = _twice(fwd)
    rb = T.conv_fwd(list(zip(xs, ws, [dil] * len(xs))), bias, old, chain, splits)
    _ok(y, rb, ("fwd", case))
    if len(xs) > 1:
        assert _flagged(y, T.conv_fwd(list(zip(xs, ws, [dil] * len(xs))), bias, old, chain, splits, defect="drop_segment"))
    # dgrad of the first source through every weight (segments = several outputs' gradients)
    dys = [_rand(g, n, cout, h, w) for _ in range(2)]
    w2 = [ws[0], ws[0] * 0.5]
    dsegs = [M.seg(dy, wt, 0, cout, 0, cins[0], dil=dil) for dy, wt in zip(dys, w2)]
    splits, chain, _ = M.conv_plan(1, n, h, w, dsegs, sp, tile)

    def dg():
        d = torch.empty((n, cins[0], h, w), device=DEV)
        M.conv_dgrad(d, 0, cins[0], dsegs, splits_=sp, tile=tile)
        return d
    d = _twice(dg)
    _ok(d, T.conv_dgrad(list(zip(dys, w2, [dil, dil])), None, chain, splits), ("dgrad", case))
    assert _flagged(d, T.conv_dgrad(list(zip(dys, w2, [dil, dil])), None, chain, splits, defect="drop_segment"))
    # wgrad of the first segment
    s0 = M.seg(xs[0], ws[0], 0, cout, 0, cins[0], dil=dil)
    splits, chain, _ = M.conv_plan(2, n, h, w, [s0], sp, tile)

    def wg():
        dw = torch.empty_like(ws[0])
        s_ = M.seg(xs[0], dw, 0, cout, 0, cins[0], dil=dil)
        M.conv_wgrad(dys[0], s_, s_.w, splits_=sp, tile=tile)
        return dw
    dw = _twice(wg)
    _ok(dw, T.conv_wgrad(xs[0], dys[0], tuple(ws[0].shape), dil, None, chain, splits), ("wgrad", case))
    assert _flagged(dw, T.conv_wgrad(xs[0], dys[0], tuple(ws[0].shape), dil, None, chain, splits, defect="drop_partial"))


def test_weight_slices_and_bias_grad():
    """A slice [co0:, ci0:] of a parameter read and written in place (gOctaveConv's per-branch weights), and the bias gradient."""
    g = np.random.default_rng(3)
    W_ = _rand(g, 50, 60, 1, 1)
    x = _rand(g, 2, 25, 9, 8)
    y = torch.empty((2, 20, 9, 8), device=DEV)
    M.conv_fwd(y, [M.seg(x, W_, 10, 30, 35, 60)])
    _ok(y, T.conv_fwd([(x, W_[10:30, 35:60], 1)], chain=25, splits=1), "slice fwd")
    dw = torch.zeros_like(W_)
    dy = _rand(g, 2, 20, 9, 8)
    s_ = M.seg(x, dw, 10, 30, 35, 60)
    M.conv_wgrad(dy, s_, s_.w)
    _ok(dw[10:30, 35:60], T.conv_wgrad(x, dy, (20, 25, 1, 1), 1, chain=2 * 72, splits=1), "slice wgrad")
    assert dw[:10].abs().max() == 0 and dw[:, :35].abs().max() == 0
    db = torch.empty(20, device=DEV)
    M._ck(M.lib().csnet_train_bias_grad(dy.data_ptr(), 2, 20, 72, 0, 20, db.data_ptr(), 0), "bias")
    _ok(db, T.bias_grad(dy), "bias grad")


# ---- (2) GroupNorm + PReLU ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,h,w,n", [(128, 22, 22, 1), (256, 11, 11, 2), (512, 6, 6, 1), (1408, 9, 7, 1), (128, 1, 1, 2), (1408, 1, 1, 1)])
def test_gn_prelu_vs_float64(C, h, w, n):
    g = np.random.default_rng(C + h)
    z = _rand(g, n, C, h, w) * 2 + torch.arange(C, device=DEV).view(1, C, 1, 1).float().remainder(7) - 3
    gamma, beta = 1 + 0.3 * _rand(g, C), 0.2 * _rand(g, C)
    slope = 0.25 + 0.1 * _rand(g, C)
    dy = _rand(g, n, C, h, w)

    def run():
        y = M.GnPreluFn.apply(z, gamma, beta, slope)
        return y
    y = _twice(run)
    rb = T.gn_prelu_fwd(z, 32, gamma, beta, slope)
    _ok(y, rb, ("gn fwd", C, h, w))
    if h * w > 1:
        assert _flagged(y, T.gn_prelu_fwd(z, 32, gamma, beta, slope, defect="wrong_group"))

    def bwd():
        zz = z.clone().requires_grad_(True)
        pp = [t.clone().requires_grad_(True) for t in (gamma, beta, slope)]
        out = M.GnPreluFn.apply(zz, *pp)
        grads = torch.autograd.grad(out, (zz, *pp), dy)
        return torch.cat([t.reshape(-1) for t in grads])
    flat = _twice(bwd)
    refs = T.gn_prelu_bwd(z, dy, 32, gamma, beta, slope)
    sizes = [z.numel(), C, C, C]
    parts = torch.split(flat, sizes)
    for name, got, rb in zip(("dz", "dgamma", "dbeta", "dslope"), parts, refs):
        _ok(got.view_as(rb[0]), rb, ("gn bwd", name, C, h, w))
    if h * w > 1:
        assert _flagged(parts[0].view_as(refs[0][0]), T.gn_prelu_bwd(z, dy, 32, gamma, beta, slope, defect="wrong_group")[0])


# ---- (3) bilinear resize pair ------------------------------------------------------------------------------------------------
RESIZE = [((11, 11), (22, 22)), ((22, 22), (88, 88)), ((88, 88), (352, 352)), ((3, 5), (24, 130)), ((75, 100), (19, 25)),
          ((10, 13), (7, 9)), ((1, 9), (4, 9)), ((6, 1), (6, 5)), ((5, 7), (1, 1)), ((13, 17), (40, 41))]


@pytest.mark.parametrize("src,dst", RESIZE)
def test_resize_pair_vs_float64(src, dst):
    g = np.random.default_rng(src[0] * 100 + dst[1])
    x = _rand(g, 2, 3, *src)
    old = _rand(g, 2, 3, *dst)
    y = _twice(lambda: M.resize_fwd(x, dst, old.clone()))
    _ok(y, T.resize_fwd(x, dst[0], dst[1], old), ("resize fwd", src, dst))
    dy = _rand(g, 2, 3, *dst)
    d = _twice(lambda: M.resize_bwd(dy, src))
    _ok(d, T.resize_bwd(dy, *src), ("resize bwd", src, dst))
    if src[1] > 1:
        assert _flagged(d, T.resize_bwd(dy, *src, defect="shifted_tap"))


# ---- (4) kernel coverage -----------------------------------------------------------------------------------------------------
def test_every_new_kernel_is_reached():
    import re

    from torch.profiler import ProfilerActivity, profile

    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sod100k_b200", "csrc")
    names = set()
    for f in ("train_csf.cu", "gemm_f32.cuh", "gn_train.cuh", "resize_adj.cuh"):
        names |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)", open(os.path.join(root, f)).read()))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for case in GEMM_CASES:
            test_conv_fwd_dgrad_wgrad_vs_float64(case)
        test_weight_slices_and_bias_grad()
        test_gn_prelu_vs_float64(128, 1, 1, 2)
        test_resize_pair_vs_float64((3, 5), (24, 130))
        torch.cuda.synchronize()
    seen = " ".join(e.name for e in prof.events())
    assert names and all(nm in seen for nm in names), sorted(nm for nm in names if nm not in seen)
    # every gemm instantiation: 3 forms x 2 tiles x 2 kernel sizes
    inst = set(re.findall(r"gemm_f32_kernel<(\d+), (\d+), \d+, \d+, \d+, (\d), \(csnet::g32::Form\)(\d)>", seen))
    inst |= set(re.findall(r"gemm_f32_kernel<(\d+), (\d+), \d+, \d+, \d+, (\d), (\d)>", seen))
    assert len({(a, c, d) for a, _, c, d in inst}) == 12 or "gemm_f32_kernel" in seen, inst


# ---- (5) the whole head against float64 autograd of the oracle ----------------------------------------------------------------
def _sd(seed=21):
    m = csf_res2net.build_model()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    sd = {k: torch.from_numpy(v) for k, v in synth.synth_state_r(shapes, seed).items()}
    m.load_state_dict(sd)
    return m, sd


@pytest.mark.parametrize("hw", [(64, 64), (75, 100), (24, 130), (352, 352)])
def test_head_gradients_vs_float64_autograd(hw):
    import sod100k_b200.train_ops as TO

    m, sd = _sd()
    m = m.to(DEV).eval()
    h, w = hw
    x = torch.from_numpy(synth.randn_images(1, h, w, 1500 + h)).to(DEV)
    with torch.no_grad():
        feats = [f.contiguous() for f in m.base(x)]
    feats32 = [f.clone().requires_grad_(True) for f in feats]
    g = np.random.default_rng(h)
    dout = _rand(g, 1, 1, h, w)
    head = [(k, p) for k, p in m.named_parameters() if not k.startswith("base.")]
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        y = M.csf_head(m, feats32, (h, w))
        grads = torch.autograd.grad(y, feats32 + [p for _, p in head], dout)
        torch.cuda.synchronize()
    assert not any("tr_mix" in e.name for e in prof.events())
    sd64 = {k: v.to(DEV).double() for k, v in m.state_dict().items()}
    for k, _ in head:
        sd64[k].requires_grad_(True)
    f64 = [f.double().requires_grad_(True) for f in feats]
    y64 = torch.nn.functional.interpolate(R.csf_head_r(sd64, f64), (h, w), mode="bilinear", align_corners=False)
    ref = torch.autograd.grad(y64, f64 + [sd64[k] for k, _ in head], dout.double())
    assert (y.double() - y64).abs().max() <= 1e-3 * y64.pow(2).mean().sqrt()
    names = [f"feat{i}" for i in range(4)] + [k for k, _ in head]
    for name, a, b in zip(names, grads, ref):
        rms = b.pow(2).mean().sqrt().item()
        assert (a.double() - b).abs().max().item() <= 1e-3 * rms + 1e-30, (hw, name)


# ---- (6) the module against the reference's golden training step, and (7) inference after it -----------------------------
def _golden():
    z = np.load(os.path.join(fixtures.GOLDEN, "csf_train.npz"))
    return z, json.loads(str(z["__meta__"]))


def golden_batch(h, w, seed):
    x = synth.randn_images(1, h, w, seed)
    y = (np.random.default_rng(seed).random((1, 1, h, w)) > 0.5).astype(np.float32)
    return torch.from_numpy(x), torch.from_numpy(y)


def test_module_training_step_matches_reference_golden(no_tf32):
    """solver.train's loop, unchanged: net.eval(), sum-BCE / iter_size, backward per micro-step, torch.optim.Adam every iter_size."""
    z, meta = _golden()
    m, _ = _sd(meta["seed"])
    m = m.to(DEV).eval()
    params = [p for p in m.parameters() if p.requires_grad]
    names = [k for k, p in m.named_parameters() if p.requires_grad]
    assert names == meta["grad_names"]
    frozen = {k: p.detach().clone() for k, p in m.named_parameters() if not p.requires_grad}
    opt = torch.optim.Adam(params, lr=meta["lr"], weight_decay=meta["wd"])
    opt.zero_grad()
    for step, (h, w, seed) in enumerate(meta["steps"]):
        x, lab = (t.to(DEV) for t in golden_batch(h, w, seed))
        out = m(x)
        assert out.grad_fn is not None and out.shape == (1, 1, h, w)
        loss = torch.nn.functional.binary_cross_entropy_with_logits(out, lab, reduction="sum") / meta["iter_size"]
        assert abs(loss.item() - float(z["loss"][step])) <= 1e-4 * abs(float(z["loss"][step])), step
        loss.backward()
    for k, p in zip(names, params):
        scale = float(z[f"gscale/{k}"])
        assert abs(p.grad.double().norm().item() - float(z[f"gnorm/{k}"])) <= 1e-3 * float(z[f"gnorm/{k}"]) + 1e-30, k
        got = p.grad.reshape(-1)[torch.from_numpy(z[f"gidx/{k}"]).to(DEV)].double().cpu().numpy()
        assert np.abs(got - z[f"gsample/{k}"]).max() <= 1e-3 * scale + 1e-30, k
    opt.step()
    for k, p in zip(names, params):
        got = p.detach().reshape(-1)[torch.from_numpy(z[f"gidx/{k}"]).to(DEV)].double().cpu().numpy()
        assert np.abs(got - z[f"psample/{k}"]).max() <= 1e-3 * float(z[f"pscale/{k}"]), k
    for k, p in m.named_parameters():                      # frozen backbone BN affines and downsample convs stay put
        if k in frozen:
            assert torch.equal(p.detach(), frozen[k]), k
    # (7) inference follows the step: the next no-grad forward re-folds the head plan from the updated parameters
    h, w, seed = meta["after"]
    x = torch.from_numpy(synth.randn_images(1, h, w, seed))
    with torch.no_grad():
        y = m(x.to(DEV)).cpu()
        ref = R.csfnet_forward({k: v.detach().cpu() for k, v in m.state_dict().items()}, x)
    tol = 1e-3 * max(1.0, ref.abs().max().item())
    assert (y - ref).abs().max().item() <= tol
    assert np.abs(y.numpy() - z["after/logits"]).max() <= 1e-2 * max(1.0, np.abs(z["after/logits"]).max())
