"""CSF+Res2Net training with bf16 activation storage on the GPU: the tensor-core GEMM, GroupNorm and resize bf16 calls against float64
on their own bf16 operands (twice, bit-identical, each with an injected defect that must exceed its bound), at generic edge shapes and
at every head convolution of real steps; kernel coverage of a bf16 step; the bf16 CSFTrainer against the fp32 one; the interface."""
import copy

import numpy as np
import pytest
import torch

from sod100k_b200 import modular_r as M
from sod100k_b200 import synth
from sod100k_b200.networks import csf_res2net
from sod100k_b200.train_ops import BceSumFn
from sod100k_b200.trainer import CSFTrainer
from tests import trainref_r_bf16 as B

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rand(g, *shape, scale=1.0):
    return torch.from_numpy((scale * g.standard_normal(shape)).astype(np.float32)).to(DEV)


def _bf(t):
    return t.to(torch.bfloat16)


def _q(got, ref_bound):
    ref, bound = ref_bound
    got = got.detach().double().to(ref.device)
    r = (got - ref).abs() / bound
    r = torch.where(torch.isfinite(got), r, torch.full_like(r, float("inf")))
    return float(r.max())


def _ok(got, ref_bound, label):
    q = _q(got, ref_bound)
    assert q <= 1.0, (label, q)


def _flagged(got, ref_bound):
    return _q(got, ref_bound) > 1.0


def _twice(fn):
    a = fn()
    b = fn()
    assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a, b.view(torch.int16) if b.dtype == torch.bfloat16 else b), \
        "not bit-identical run to run"
    return a


# ---- (1) the tensor-core GEMM in every form ------------------------------------------------------------------------------------------
def check_gemm(n, h, w, cins, cout, k, dil, sp, out_dtype=torch.bfloat16, accumulate=True, bias=True, seed=0, defects=True):
    """fwd over len(cins) segments (bias, accumulate), dgrad of the first source over two output gradients, wgrad of the first
    segment: each against float64 on its bf16 operands; returns the split counts the calls used."""
    g = np.random.default_rng(seed)
    xs = [_bf(_rand(g, n, c, h, w)) for c in cins]
    ws = [_rand(g, cout, c, k, k, scale=1.0 / np.sqrt(c * k * k)) for c in cins]
    wb = [M.cast_bf16(t) for t in ws]
    assert all(torch.equal(a.float(), B.round_bf16(t)) for a, t in zip(wb, ws)), "cast_bf16 is not round-to-nearest-even"
    bvec = _rand(g, cout) if bias else None
    old = _rand(g, n, cout, h, w).to(out_dtype)
    segs = [M.seg(x, t, 0, cout, 0, x.shape[1], dil=dil) for x, t in zip(xs, wb)]
    used = []
    s_fwd, _, _ = M.conv_plan_bf16(0, n, h, w, segs, sp)

    def fwd():
        y = old.clone() if accumulate else torch.empty_like(old)
        M.conv_fwd_bf16(y, segs, bias=bvec.data_ptr() if bias else None, accumulate=accumulate, splits_=sp)
        return y
    y = _twice(fwd)
    bf_out = out_dtype == torch.bfloat16
    sg = list(zip(xs, ws, [dil] * len(xs)))
    _ok(y, B.conv_fwd(sg, bvec, old if accumulate else None, s_fwd, bf_out), ("fwd", n, h, w, cins, cout, k, dil, sp))
    if defects:
        if not bf_out:                      # a bf16 store's rounding (2^-8 |r|) is coarser than the truncated weights' error
            assert _flagged(y, B.conv_fwd(sg, bvec, old if accumulate else None, s_fwd, bf_out, defect="truncated_w"))
        if sum(cins) * k * k >= 16:
            assert _flagged(y, B.conv_fwd(sg, bvec, old if accumulate else None, s_fwd, bf_out, defect="drop_k16"))
    used.append(s_fwd)
    dys = [_bf(_rand(g, n, cout, h, w)) for _ in range(2)]
    w2 = [ws[0], ws[0] * 0.5]
    w2b = [M.cast_bf16(t) for t in w2]
    dsegs = [M.seg(dy, t, 0, cout, 0, cins[0], dil=dil) for dy, t in zip(dys, w2b)]
    s_dg, _, _ = M.conv_plan_bf16(1, n, h, w, dsegs, sp)
    dold = _rand(g, n, cins[0], h, w).to(out_dtype)

    def dg():
        d = dold.clone() if accumulate else torch.empty_like(dold)
        M.conv_dgrad_bf16(d, 0, cins[0], dsegs, accumulate=accumulate, splits_=sp)
        return d
    d = _twice(dg)
    dsg = list(zip(dys, w2, [dil, dil]))
    _ok(d, B.conv_dgrad(dsg, dold if accumulate else None, s_dg, bf_out), ("dgrad", n, h, w, cins, cout, k, dil, sp))
    if defects:
        if not bf_out:
            assert _flagged(d, B.conv_dgrad(dsg, dold if accumulate else None, s_dg, bf_out, defect="truncated_w"))
        assert _flagged(d, B.conv_dgrad(dsg, dold if accumulate else None, s_dg, bf_out, defect="drop_k16"))
    used.append(s_dg)
    s0 = M.seg(xs[0], ws[0], 0, cout, 0, cins[0], dil=dil)
    s_wg, _, _ = M.conv_plan_bf16(2, n, h, w, [s0], sp)
    wold = _rand(g, *ws[0].shape)

    def wg():
        dw = wold.clone() if accumulate else torch.empty_like(wold)
        s_ = M.seg(xs[0], dw, 0, cout, 0, cins[0], dil=dil)
        M.conv_wgrad_bf16(dys[0], s_, s_.w, accumulate=accumulate, splits_=sp)
        return dw
    dw = _twice(wg)
    rb = B.conv_wgrad(xs[0], dys[0], tuple(ws[0].shape), dil, wold if accumulate else None, s_wg)
    _ok(dw, rb, ("wgrad", n, h, w, cins, cout, k, dil, sp))
    if defects:
        assert _flagged(dw, B.conv_wgrad(xs[0], dys[0], tuple(ws[0].shape), dil, wold if accumulate else None, s_wg, defect="drop_k16"))
    used.append(s_wg)
    return used


# (N, H, W, cins per segment, cout, k, dil, splits, out dtype, accumulate)
GEMM_CASES = [
    (1, 11, 11, [256, 512, 1024], 128, 1, 1, 0, torch.bfloat16, True),    # fuse.0-like, several segments, auto split
    (2, 7, 9, [37, 20], 70, 1, 1, 1, torch.bfloat16, False),               # ragged M, N, K (odd row widths), no split
    (2, 7, 9, [37, 20], 70, 1, 1, 5, torch.float32, True),                 # same, split-K, fp32 destination
    (1, 13, 10, [300], 1, 1, 1, 0, torch.float32, True),                   # cout = 1 (cls_layer), fp32 map
    (1, 12, 12, [200], 150, 1, 1, 3, torch.bfloat16, True),
    (2, 6, 5, [33], 21, 3, 1, 1, torch.bfloat16, True),                    # 3x3 d = 1
    (1, 10, 13, [25], 25, 3, 2, 0, torch.bfloat16, False),                 # MSBlock widths, 25 channels
    (1, 22, 22, [128], 130, 3, 4, 2, torch.float32, False),
    (1, 19, 25, [64], 27, 3, 8, 0, torch.bfloat16, True),
    (1, 5, 6, [40], 25, 3, 8, 0, torch.bfloat16, True),                    # d >= plane: only the centre tap lands
    (1, 4, 3, [20], 9, 3, 16, 1, torch.bfloat16, True),                    # d = 16, padding 16 > plane
    (1, 3, 4, [24], 20, 3, 12, 2, torch.float32, True),
]


@pytest.mark.parametrize("case", GEMM_CASES)
def test_gemm_bf16_vs_float64(case):
    n, h, w, cins, cout, k, dil, sp, dt, acc = case
    check_gemm(n, h, w, cins, cout, k, dil, sp, dt, acc, bias=k == 1 and len(cins) == 1, seed=GEMM_CASES.index(case))


def test_weight_slices_bf16():
    """A slice [co0:, ci0:] of a parameter read (bf16 copy) and written (fp32 gradient) in place."""
    g = np.random.default_rng(3)
    W_ = _rand(g, 50, 60, 1, 1)
    Wb = M.cast_bf16(W_)
    x = _bf(_rand(g, 2, 25, 9, 8))
    y = torch.empty((2, 20, 9, 8), device=DEV, dtype=torch.bfloat16)
    M.conv_fwd_bf16(y, [M.seg(x, Wb, 10, 30, 35, 60)])
    _ok(y, B.conv_fwd([(x, W_[10:30, 35:60], 1)]), "slice fwd")
    dw = torch.zeros_like(W_)
    dy = _bf(_rand(g, 2, 20, 9, 8))
    s_ = M.seg(x, dw, 10, 30, 35, 60)
    M.conv_wgrad_bf16(dy, s_, s_.w)
    _ok(dw[10:30, 35:60], B.conv_wgrad(x, dy, (20, 25, 1, 1), 1), "slice wgrad")
    assert dw[:10].abs().max() == 0 and dw[:, :35].abs().max() == 0


# ---- (1b) every head convolution of a real bf16 step, at its own shapes -----------------------------------------------------------
def _net(seed=21):
    m = csf_res2net.build_model()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.synth_state_r(shapes, seed).items()})
    return m.to(DEV).eval()


def _record_calls(net, h, w):
    """The (form, N, H, W, [(cin, cout, k, dil)], dst dtype, accumulate) of every GEMM call of one bf16 step at h x w."""
    calls = []

    def wrap(form, fn):
        def f(dst, *a, **kw):
            segs = a[0] if form == 0 else (a[2] if form == 1 else [a[0]])
            acc = kw.get("accumulate", False)
            N, _, H, W = dst.shape
            calls.append((form, N, H, W, tuple((s.cin, s.cout, s.ksize, s.dil) for s in segs), dst.dtype if form < 2 else None, bool(acc)))
            return fn(dst, *a, **kw)
        return f
    orig = (M.conv_fwd_bf16, M.conv_dgrad_bf16, M.conv_wgrad_bf16)
    M.conv_fwd_bf16, M.conv_dgrad_bf16, M.conv_wgrad_bf16 = (wrap(i, f) for i, f in enumerate(orig))
    try:
        net.train_storage = "bf16"
        x = torch.from_numpy(synth.randn_images(1, h, w, 5)).to(DEV)
        t = (torch.rand((1, 1, h, w), device=DEV) > 0.5).float()
        with torch.enable_grad():
            BceSumFn.apply(net(x), t, 1).backward()
        net.zero_grad(set_to_none=True)
    finally:
        M.conv_fwd_bf16, M.conv_dgrad_bf16, M.conv_wgrad_bf16 = orig
    return calls


@pytest.mark.parametrize("hw", [(352, 352), (400, 300), (75, 100)])
def test_gemm_bf16_at_head_shapes(hw):
    """Every distinct GEMM call of a bf16 step at this size, re-run on seeded data of its shapes (segments, k, dilation, split the
    planner picks, destination dtype), against float64; each shape's calls run twice with identical bits."""
    calls = sorted(set(_record_calls(_net(), *hw)), key=str)
    assert len(calls) >= 10
    splits_seen = set()
    for i, (form, N, H, W, segs, dt, acc) in enumerate(calls):
        cout, k, dil = segs[0][1], segs[0][2], segs[0][3]
        used = check_gemm(N, H, W, [s[0] for s in segs] if form == 0 else [segs[0][0]], cout, k, dil, 0, dt or torch.bfloat16, acc,
                          bias=cout == 1, seed=100 + i, defects=False)
        splits_seen.update(used)
    assert max(splits_seen) > 1 and 1 in splits_seen, splits_seen


# ---- (2) GroupNorm + PReLU, bf16 in and out -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,h,w,n", [(128, 88, 88, 1), (256, 11, 11, 2), (512, 25, 19, 1), (1408, 9, 7, 1), (128, 1, 1, 2), (1408, 1, 1, 1)])
def test_gn_prelu_bf16_vs_float64(C, h, w, n):
    g = np.random.default_rng(C + h)
    z = _bf(_rand(g, n, C, h, w) * 2 + torch.arange(C, device=DEV).view(1, C, 1, 1).float().remainder(7) - 3)
    gamma, beta = 1 + 0.3 * _rand(g, C), 0.2 * _rand(g, C)
    slope = 0.25 + 0.1 * _rand(g, C)
    dy = _bf(_rand(g, n, C, h, w))
    y = _twice(lambda: M.GnPreluFn.apply(z, gamma, beta, slope))
    assert y.dtype == torch.bfloat16
    _ok(y, B.gn_prelu_fwd(z, 32, gamma, beta, slope), ("gn fwd", C, h, w))
    if h * w > 1:
        assert _flagged(y, B.gn_prelu_fwd(z, 32, gamma, beta, slope, defect="wrong_group"))

    def bwd():
        zz = z.clone().requires_grad_(True)
        pp = [t.clone().requires_grad_(True) for t in (gamma, beta, slope)]
        grads = torch.autograd.grad(M.GnPreluFn.apply(zz, *pp), (zz, *pp), dy)
        assert grads[0].dtype == torch.bfloat16 and all(t.dtype == torch.float32 for t in grads[1:])
        return torch.cat([grads[0].float().reshape(-1)] + [t.reshape(-1) for t in grads[1:]])
    flat = _twice(bwd)
    refs = B.gn_prelu_bwd(z, dy, 32, gamma, beta, slope)
    parts = torch.split(flat, [z.numel(), C, C, C])
    for name, got, rb in zip(("dz", "dgamma", "dbeta", "dslope"), parts, refs):
        _ok(got.view_as(rb[0]), rb, ("gn bwd", name, C, h, w))
    if h * w > 1:
        assert _flagged(parts[0].view_as(refs[0][0]), B.gn_prelu_bwd(z, dy, 32, gamma, beta, slope, defect="wrong_group")[0])


# ---- (3) bilinear resize pair, bf16 ----------------------------------------------------------------------------------------------------
RESIZE = [((11, 11), (22, 22)), ((22, 22), (88, 88)), ((88, 88), (352, 352)), ((13, 10), (25, 19)), ((75, 100), (19, 25)),
          ((10, 13), (7, 9)), ((1, 9), (4, 9)), ((6, 1), (6, 5)), ((5, 7), (1, 1)), ((13, 17), (40, 41))]


@pytest.mark.parametrize("src,dst", RESIZE)
def test_resize_pair_bf16_vs_float64(src, dst):
    g = np.random.default_rng(src[0] * 100 + dst[1])
    x = _bf(_rand(g, 2, 3, *src))
    old = _bf(_rand(g, 2, 3, *dst))
    y = _twice(lambda: M.resize_fwd(x, dst, old.clone()))
    assert y.dtype == torch.bfloat16
    _ok(y, B.resize_fwd(x, dst[0], dst[1], old), ("resize fwd", src, dst))
    dy = _bf(_rand(g, 2, 3, *dst))
    d = _twice(lambda: M.resize_bwd(dy, src))
    assert d.dtype == torch.bfloat16
    _ok(d, B.resize_bwd(dy, *src), ("resize bwd", src, dst))
    if src[1] > 1:
        assert _flagged(d, B.resize_bwd(dy, *src, defect="shifted_tap"))


# ---- (4) kernel coverage of one bf16 step at 352^2 -----------------------------------------------------------------------------------
def test_bf16_step_kernel_coverage():
    from torch.profiler import ProfilerActivity, profile

    net = _net()
    tr = CSFTrainer(net, iter_size=1, storage="bf16")
    x = torch.from_numpy(synth.randn_images(1, 352, 352, 3)).to(DEV)
    t = (torch.rand((1, 1, 352, 352), device=DEV) > 0.5).float()
    n_calls = [0]
    orig = (M.conv_fwd_bf16, M.conv_dgrad_bf16, M.conv_wgrad_bf16, M.conv_fwd, M.conv_dgrad, M.conv_wgrad)

    def count(fn):
        def f(*a, **kw):
            n_calls[0] += 1
            return fn(*a, **kw)
        return f
    M.conv_fwd_bf16, M.conv_dgrad_bf16, M.conv_wgrad_bf16 = (count(f) for f in orig[:3])
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            tr.step(x, t)
            torch.cuda.synchronize()
    finally:
        M.conv_fwd_bf16, M.conv_dgrad_bf16, M.conv_wgrad_bf16 = orig[:3]
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    gemm = [k for k in names if "gemm_bf16_kernel" in k]
    assert len(gemm) == n_calls[0] > 0, (len(gemm), n_calls[0])          # every head convolution call launched the tensor-core kernel
    assert not any("gemm_f32" in k for k in names)
    assert not any("tr_mix" in k for k in names)
    for k in ("gn_stats_bf16_kernel", "gn_prelu_fwd_bf16_kernel", "gn_bwd_dz_bf16_kernel", "resize_bwd_bf16_kernel", "cast_bf16_kernel"):
        assert any(k in n for n in names), k


# ---- (5) the bf16 step against the fp32 one ------------------------------------------------------------------------------------------
@pytest.fixture
def deterministic():
    old = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = old


def _batch(h, w, i):
    x = torch.from_numpy(synth.randn_images(1, h, w, 300 + i)).to(DEV)
    t = torch.from_numpy(synth.random_masks(1, h, w, 400 + i)).to(DEV).float().view(1, 1, h, w)
    return x, (t > 0.5).float()


def _head_grads(net):
    return {k: p.grad.detach().clone() for k, p in net.named_parameters() if not k.startswith("base.") and p.requires_grad}


@pytest.mark.parametrize("hw", [(352, 352), (300, 400), (75, 100)])
def test_bf16_trainer_against_fp32(deterministic, hw):
    h, w = hw
    net32 = _net()
    tr32 = CSFTrainer(net32, iter_size=10)
    probe = copy.deepcopy(net32)
    probe.train_storage = "bf16"
    netb = copy.deepcopy(net32)
    trb = CSFTrainer(netb, iter_size=10, storage="bf16")
    # one micro-step on identical parameters: each head tensor's gradient within 5e-2 of its rms (rms of the difference)
    x, t = _batch(h, w, 0)
    tr32.step(x, t)
    trb.step(x, t)
    g32, gb = _head_grads(net32), _head_grads(netb)
    for k in g32:
        rms = float(g32[k].double().pow(2).mean().sqrt())
        err = float((gb[k].double() - g32[k].double()).pow(2).mean().sqrt())
        assert err <= 5e-2 * rms, (k, err, rms)
    # 20 micro-steps (two Adam steps): the bf16 loss on the fp32 run's parameters within 1 % of the fp32 loss at each
    tr32 = CSFTrainer(net32, iter_size=10)
    tr32.flat.zero()
    net32.load_state_dict(_net().state_dict())
    for i in range(20):
        x, t = _batch(h, w, i)
        probe.load_state_dict(net32.state_dict())
        with torch.enable_grad():
            lb = float(BceSumFn.apply(probe(x), t, 10).detach())
        l32 = float(tr32.step(x, t))
        assert abs(lb - l32) <= 1e-2 * abs(l32), (i, lb, l32)


def test_bf16_trainer_deterministic_and_refolds(deterministic):
    """Two bf16 runs give bit-identical parameters; inference after bf16 training uses the trained head (the plan is re-folded)."""
    runs = []
    for _ in range(2):
        net = _net()
        tr = CSFTrainer(net, iter_size=2, storage="bf16")
        with torch.no_grad():
            before = net(torch.from_numpy(synth.randn_images(1, 64, 64, 9)).to(DEV))      # a head plan folded from the initial weights
        for i in range(4):
            tr.step(*_batch(64, 96, i))
        runs.append(net)
    for (k, a), b in zip(runs[0].state_dict().items(), runs[1].state_dict().values()):
        assert torch.equal(a, b), k
    net = runs[0]
    x = torch.from_numpy(synth.randn_images(1, 64, 64, 9)).to(DEV)
    with torch.no_grad():
        after = net(x)
        fresh = _net()
        fresh.load_state_dict(net.state_dict())
        want = fresh(x)
    assert not torch.equal(after, before)
    assert torch.equal(after, want)


# ---- (6) interface -----------------------------------------------------------------------------------------------------------------------
def test_storage_interface(deterministic):
    net = _net()
    assert net.train_storage == "fp32"
    x, t = _batch(64, 64, 0)
    ref = copy.deepcopy(net)
    net.set_precision("bf16")                           # inference only: training stays fp32
    with torch.enable_grad():
        a, b = net(x), ref(x)
    assert a.dtype == torch.float32 and torch.equal(a, b)
    net.train_storage = "fp16"
    with torch.enable_grad(), pytest.raises(ValueError):
        net(x)
    with pytest.raises(ValueError):
        CSFTrainer(ref, storage="half")
    net.train_storage = "bf16"
    with torch.enable_grad():
        y = net(x)
    assert y.dtype == torch.float32 and y.grad_fn is not None
