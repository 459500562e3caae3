"""tests/trainref.py, the float64 reference and error bound of every csnet_train_* entry point, checked without a GPU:
  * its values equal torch.autograd in float64 of the F.* restatement of each entry point (to 1e-12 of the scale);
  * its bounds hold for float32 evaluations (torch on the CPU) and for float32 sums taken in a shuffled order;
  * the check has power: each typical kernel mistake (trainref.DEFECTS), applied to the reference, exceeds the bound on
    the inputs the GPU test (tests/test_gpu_train_kernels_vs_float64.py) uses."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import trainref as R
from tests.test_gpu_train_kernels_vs_float64 import BETAS, BY_ID, EPS, LR, make_inputs, reference


def _close(a, b):
    a, b = a.detach().double(), b.detach().double()
    assert float((a - b).abs().max()) <= 1e-12 * max(1.0, float(b.abs().max())), float((a - b).abs().max())


def _within(got, rb):
    q, msg = R.check(got, *rb)
    assert q <= 1.0, msg
    return q


def _w4(w, k):
    """Kernel layout [cin, k*k, cout] -> F.conv2d layout [cout, cin, k, k]."""
    cin, _, cout = w.shape
    return w.reshape(cin, k, k, cout).permute(3, 0, 1, 2)


def _path_autograd(q, ddst, dt):
    """F.* restatement of one path (output slice, value and both gradients) in dtype dt."""
    x = q.src[:, q.c0:q.c0 + q.cin].to(dt).clone().requires_grad_(True)
    dy = ddst[:, q.cout0:q.cout0 + q.cout].to(dt)
    if q.ksize == 0:
        y = F.interpolate(x, scale_factor=q.up, mode="bilinear", align_corners=False)
        y.backward(dy)
        return y.detach(), x.grad, None
    w = _w4(q.w.to(dt), q.ksize).clone().requires_grad_(True)
    y = F.conv2d(x, w, None, q.stride, q.pad, q.dil)
    y.backward(dy)
    cin, k = q.cin, q.ksize
    return y.detach(), x.grad, w.grad.permute(1, 2, 3, 0).reshape(cin, k * k, q.cout)


MIX_IDS = ["c1_w13_slices", "c1_with_resample", "gen_4_resample", "k5", "stride2", "stride2_odd", "k1_dil2_wgrad", "resample_up8",
           "resample_hs1_odd", "k3_ipb_14", "k3_tiny_tiles_w30", "msblock_14", "dil8_7x7"]


def _mix_sum(case, inp, dt):
    p = case.p
    paths = R_paths(case, inp)
    dst = torch.zeros(p["N"], p["C"], p["H"], p["W"], dtype=dt)
    grads = []
    for q in paths:
        y, dx, dw = _path_autograd(q, inp["ddst"], dt)
        dst[:, q.cout0:q.cout0 + q.cout] += y
        grads.append((dx, dw))
    return dst, grads


def R_paths(case, inp):
    from tests.test_gpu_train_kernels_vs_float64 import _paths
    return _paths(case, inp)


@pytest.mark.parametrize("case_id", MIX_IDS)
def test_mix_reference_equals_autograd_and_bounds_fp32(case_id):
    case = BY_ID[case_id]
    inp = make_inputs(case)
    ref = reference(case, inp)
    dst64, g64 = _mix_sum(case, inp, torch.float64)
    _close(ref["dst"][0], dst64)
    dst32, g32 = _mix_sum(case, inp, torch.float32)
    _within(dst32, ref["dst"])
    for i, ((dx, dw), (dx32, dw32)) in enumerate(zip(g64, g32)):
        _close(ref[f"dsrc{i}"][0], dx)
        _within(dx32, ref[f"dsrc{i}"])
        if dw is not None:
            _close(ref[f"dw{i}"][0], dw)
            _within(dw32, ref[f"dw{i}"])


def _shuffled_sum(terms, g):
    """fp32 products summed one by one in a random order (terms: [elements, count] float64)."""
    t = terms.float()
    perm = torch.randperm(t.shape[1], generator=g)
    acc = torch.zeros(t.shape[0], dtype=torch.float32)
    for j in perm.tolist():
        acc = acc + t[:, j]
    return acc


@pytest.mark.parametrize("case_id", ["k3_tiny_tiles_w30", "stride2_odd", "c1_w7", "k1_dil2_wgrad"])
def test_bounds_hold_for_shuffled_fp32_sums(case_id):
    """The conv forward, data gradient and weight gradient as explicit term lists, summed in fp32 in a random order:
    every chain is no longer than the depth the bounds assume on these small shapes."""
    case = BY_ID[case_id]
    inp = make_inputs(case)
    ref = reference(case, inp)
    g = torch.Generator().manual_seed(3)
    q = R_paths(case, inp)[0]
    k = q.ksize
    x = q.src[:, q.c0:q.c0 + q.cin].double()
    dy = inp["ddst"][:, q.cout0:q.cout0 + q.cout].double()
    N, Ho, Wo = dy.shape[0], dy.shape[2], dy.shape[3]
    cols = F.unfold(x, k, dilation=q.dil, padding=q.pad, stride=q.stride)               # [N, cin k k, L]
    wf = q.w.double().reshape(-1, q.cout)                                              # [cin k k, cout]
    # forward: element (n, o, l) = sum_k cols[n, k, l] w[k, o]
    fw = (cols.permute(0, 2, 1)[:, :, :, None] * wf[None, None]).permute(0, 3, 1, 2).reshape(-1, wf.shape[0])
    _within(_shuffled_sum(fw, g).reshape(N, q.cout, Ho, Wo), ref["dst"])
    # weight gradient: element (k, o) = sum over (n, l) of cols[n, k, l] dy[n, o, l]
    dyl = dy.reshape(N, q.cout, -1)
    wt = torch.einsum("nkl,nol->konl", cols, dyl).reshape(wf.shape[0] * q.cout, -1)
    _within(_shuffled_sum(wt, g).reshape(q.cin, k * k, q.cout), ref["dw0"])
    # data gradient: the adjoint terms per source pixel, folded one term at a time in a random order
    Hs, Ws = q.src.shape[2], q.src.shape[3]
    terms = torch.einsum("ko,nol->nkol", wf, dyl)                                       # [N, cin k k, cout, L]
    order = torch.randperm(q.cout * Ho * Wo, generator=g).tolist()
    acc = torch.zeros(N, q.cin, Hs, Ws, dtype=torch.float32)
    for j in order:
        o, l = divmod(j, Ho * Wo)
        one = torch.zeros(N, wf.shape[0], Ho * Wo, dtype=torch.float64)
        one[:, :, l] = terms[:, :, o, l]
        acc = acc + F.fold(one, (Hs, Ws), k, dilation=q.dil, padding=q.pad, stride=q.stride).float()
    _within(acc, ref["dsrc0"])


# ---- depthwise ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case_id", ["dw_h5", "dw_h13_w1", "dw_w3"])
def test_dw_reference_equals_autograd_and_bounds_fp32(case_id):
    case = BY_ID[case_id]
    inp = make_inputs(case)
    ref = reference(case, inp)
    C = case.p["C"]
    for dt in (torch.float64, torch.float32):
        x = inp["x"].to(dt).clone().requires_grad_(True)
        w = inp["w"].to(dt).reshape(C, 1, 3, 3).clone().requires_grad_(True)
        y = F.conv2d(x, w * inp["scale"], None, 1, 1, 1, C)
        y.backward(inp["dy"].to(dt))
        dw = w.grad.reshape(C, 9)
        pairs = ((ref["y"], y), (ref["dxT"], x.grad), (ref["bwd_dx"], x.grad), (ref["dw"], dw), (ref["bwd_dw"], dw))
        for rb, got in pairs:
            (_close(rb[0], got) if dt == torch.float64 else _within(got, rb))


# ---- BatchNorm + PReLU -----------------------------------------------------------------------------------------------------
def _bn_autograd(inp, dt, frozen, mean=None, var=None):
    z = inp["z"].to(dt).clone().requires_grad_(True)
    g, b, a = (inp[k].to(dt).clone().requires_grad_(True) for k in ("gamma", "beta", "slope"))
    if frozen:
        y = F.prelu(F.batch_norm(z, mean.to(dt), var.to(dt), g, b, False, 0.0, inp["eps"]), a)
    else:
        y = F.prelu(F.batch_norm(z, None, None, g, b, True, 0.1, inp["eps"]), a)
    y.backward(inp["dy"].to(dt))
    return y.detach(), z.grad, g.grad, b.grad, a.grad


@pytest.mark.parametrize("case_id", ["bn_s1", "bn_n1", "bn_const_channel", "bn_mean_1e4"])
def test_bn_reference_equals_autograd_and_bounds_fp32(case_id):
    case = BY_ID[case_id]
    inp = make_inputs(case)
    z64 = inp["z"].double()
    mean, var = z64.mean((0, 2, 3)), z64.var((0, 2, 3), unbiased=False)
    st = R.bn_stats(inp["z"])
    _close(st["mean"][0], mean)
    _close(st["var"][0], var)
    # the one-pass shifted form in fp32 (shift = the fp32 mean of 32 samples, fp32 sums of z - K and (z - K)^2 per plane,
    # merged in float64) lies within the bounds
    C = z64.shape[1]
    zc = inp["z"].transpose(0, 1).reshape(C, -1)
    pick = torch.randperm(zc.shape[1], generator=torch.Generator().manual_seed(4))[:32]
    K = zc[:, pick].sum(1) / 32
    d = zc - K[:, None]
    M = zc.shape[1]
    S1 = d.reshape(C, z64.shape[0], -1).sum(2).double().sum(1)
    S2 = (d * d).reshape(C, z64.shape[0], -1).sum(2).double().sum(1)
    m1 = S1 / M
    _within((K.double() + m1).float(), st["mean"])
    _within(torch.clamp((S2 - S1 * m1) / M, min=0).float(), st["var"])
    args = (inp["gamma"], inp["beta"], inp["slope"], inp["eps"])
    for frozen in (0, 1):
        f = R.bn_prelu_fwd(inp["z"], mean, var, *args)
        b = R.bn_prelu_bwd(inp["z"], inp["dy"], mean, var, *args, frozen=frozen)
        y, dz, dg, db, da = _bn_autograd(inp, torch.float64, frozen, mean, var)
        for rb, got in ((f["y"], y), (b["dz"], dz), (b["dgamma"], dg), (b["dbeta"], db), (b["dslope"], da)):
            _close(rb[0], got)
        _close(f["gap"][0], y.mean((2, 3)))
        # fp32 evaluation with the same (fp32-rounded) statistics
        m32, v32 = mean.float(), var.float()
        f = R.bn_prelu_fwd(inp["z"], m32, v32, *args)
        b = R.bn_prelu_bwd(inp["z"], inp["dy"], m32, v32, *args, frozen=frozen)
        evals = [_bn_bwd_fp32(inp, m32, v32, frozen)]
        if frozen:                                  # with constant statistics torch's own fp32 autograd is the same map
            evals.append(_bn_autograd(inp, torch.float32, 1, m32, v32))
        for y, dz, dg, db, da in evals:
            for rb, got in ((f["y"], y), (b["dz"], dz), (b["dgamma"], dg), (b["dbeta"], db), (b["dslope"], da)):
                _within(got, rb)
            _within(y.mean((2, 3)), f["gap"])


def _bn_bwd_fp32(inp, mean, var, frozen):
    """The entry points' formulas evaluated in fp32 with the given statistics: y, then dz (with the batch-statistic terms
    unless frozen), dgamma, dbeta, dslope."""
    z, dy = inp["z"], inp["dy"]
    e = lambda t: t.reshape(1, -1, 1, 1)
    r = torch.rsqrt(e(var) + inp["eps"])
    xh = (z - e(mean)) * r
    u = e(inp["gamma"]) * xh + e(inp["beta"])
    a = e(inp["slope"])
    y = torch.where(u > 0, u, a * u)
    du = torch.where(u > 0, dy, a * dy)
    db, dg = du.sum((0, 2, 3)), (du * xh).sum((0, 2, 3))
    ds = torch.where(u > 0, torch.zeros_like(u), dy * u).sum((0, 2, 3))
    M = z.shape[0] * z.shape[2] * z.shape[3]
    gr = e(inp["gamma"]) * r
    dz = gr * du if frozen else gr * (du - e(db) / M - xh * e(dg) / M)
    return y, dz, dg, db, ds


# ---- pooling ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case_id", ["pool2_vec", "pool4_ragged", "pool8_avg", "pool2_avg_real", "avg_only"])
def test_pool_reference_equals_autograd(case_id):
    case = BY_ID[case_id]
    p = case.p
    inp = make_inputs(case)
    ref = reference(case, inp)
    f = (2 if p["pre_avg"] else 1) * p["pool"]
    Hc, Wc = p["Hs"] // f, p["Ws"] // f
    for dt in (torch.float64, torch.float32):
        x = inp["src"][:, p["c0"]:p["c0"] + p["cin"]].to(dt).clone().requires_grad_(True)
        a = x[:, :, :Hc * f, :Wc * f]
        if p["pre_avg"]:
            a = F.avg_pool2d(a, 2, 2)
        if p["pool"] > 1:
            y, ind = F.max_pool2d(a, p["pool"], p["pool"], return_indices=True)
        else:
            y, ind = a, None
        y.backward(inp["dpool"].to(dt))
        (_close(ref["dst"][0], y) if dt == torch.float64 else _within(y, ref["dst"]))
        if ind is None:
            continue
        # torch's flat index in the pooled-input plane -> row-major position inside the window
        Wa = a.shape[3]
        yy, xx = ind // Wa, ind % Wa
        pos = (yy % p["pool"]) * p["pool"] + xx % p["pool"]
        assert R.check_idx(pos, *ref["idx"]) == 0
        if dt == torch.float64:
            _close(R.pool_bwd(inp["dpool"], pos, p["Hs"], p["Ws"], p["pre_avg"], p["pool"])["dsrc"][0], x.grad)
    if p["pool"] == 1:
        _close(ref["dsrc"][0], _avg_grad(inp, p))


def _avg_grad(inp, p):
    x = inp["src"][:, p["c0"]:p["c0"] + p["cin"]].double().clone().requires_grad_(True)
    Hc, Wc = p["Hs"] // 2, p["Ws"] // 2
    F.avg_pool2d(x[:, :, :Hc * 2, :Wc * 2], 2, 2).backward(inp["dpool"].double())
    return x.grad


# ---- loss, optimiser -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case_id", ["bce_small", "bce_ragged"])
def test_bce_reference_equals_autograd_and_bounds_fp32(case_id):
    case = BY_ID[case_id]
    inp = make_inputs(case)
    ref = reference(case, inp)
    for dt in (torch.float64, torch.float32):
        z = inp["z"].to(dt).clone().requires_grad_(True)
        loss = F.binary_cross_entropy_with_logits(z, inp["t"].to(dt))
        (loss * inp["gs"]).backward()
        if dt == torch.float64:
            _close(ref["loss"][0], loss)
            _close(ref["dl"][0], z.grad)
        else:
            _within(loss, ref["loss"])
            _within(z.grad, ref["dl"])


def _torch_adam(inp, p, dt):
    params = [q.to(dt).clone().requires_grad_(True) for q in inp["params"]]
    groups = [{"params": [q], "weight_decay": wd} for q, wd in zip(params, p["wds"])]
    opt = torch.optim.Adam(groups, lr=LR, betas=BETAS, eps=EPS)
    for s, gs in enumerate(p["gs"]):
        for q, g in zip(params, inp["grads"][s]):
            q.grad = g.to(dt) * gs
        opt.step()
    return [q.detach() for q in params]


def test_adam_reference_equals_torch_optim_and_bounds_fp32():
    case = BY_ID["adam_5_steps"]
    inp = make_inputs(case)
    ref = reference(case, inp)
    for i, q in enumerate(_torch_adam(inp, case.p, torch.float64)):
        _close(ref[f"p{i}"][0], q)
    for i, q in enumerate(_torch_adam(inp, case.p, torch.float32)):
        _within(q, ref[f"p{i}"])


# ---- the check has power ---------------------------------------------------------------------------------------------------
DEFECT_CASES = [
    ("drop_last_channel", "c1_narrow", ["dst", "dsrc0"]),
    ("drop_last_channel", "k3_ipb_14", ["dst", "dsrc0"]),
    ("drop_image", "k3_ipb_14", ["dw0"]),
    ("drop_image", "c1_tiles_over_256", ["dw0"]),
    ("drop_image", "dw_h5", ["dw", "bwd_dw"]),
    ("drop_image", "bn_s1", ["mean", "var", "dgamma0", "dbeta0", "dslope0"]),
    ("drop_border", "k3_band_37", ["dst", "dsrc0"]),
    ("drop_border", "dw_w5", ["y", "dxT", "bwd_dx"]),
    ("drop_border", "pool2_vec", ["dsrc"]),
    ("drop_partial", "k3_tiny_tiles_w30", ["dw0"]),
    ("drop_partial", "dw_h13_w1", ["dw", "bwd_dw"]),
    ("drop_partial", "bn_segments_scalar", ["mean", "gap"]),
    ("drop_partial", "bce_ragged", ["loss"]),
    ("resample_shift", "c1_with_resample", ["dst", "dsrc1"]),
    ("resample_shift", "resample_up8", ["dst", "dsrc0"]),
    ("slice_shift", "c1_w13_slices", ["dst"]),
    ("slice_shift", "resample_hs1_odd", ["dst"]),
    ("pool_last_max", "pool2_vec", ["idx"]),
    ("pool_last_max", "pool4_ragged", ["idx"]),
    ("pool_last_max", "pool8_avg", ["idx"]),
    ("frozen_terms", "bn_s1", ["dz0", "dz1"]),
    ("no_bias_correction", "adam_5_steps", ["p0", "p1", "p2", "p3"]),
]


def test_every_defect_has_a_case():
    assert {d for d, _, _ in DEFECT_CASES} == set(R.DEFECTS)


@pytest.mark.parametrize("defect,case_id,outputs", DEFECT_CASES, ids=[f"{d}-{c}" for d, c, _ in DEFECT_CASES])
def test_each_defect_is_flagged(defect, case_id, outputs):
    case = BY_ID[case_id]
    inp = make_inputs(case)
    good = reference(case, inp)
    bad = reference(case, inp, defect=defect)
    for name in outputs:
        if name == "idx":
            assert R.check_idx(bad["idx"][0], *good["idx"]) > 0
            assert R.check_idx(good["idx"][0], *good["idx"]) == 0
            continue
        ref, bound = good[name]
        # the correct result rounded to fp32 passes; the defective one does not
        assert R.check(ref.float(), ref, bound)[0] <= 1.0, name
        q, _ = R.check(bad[name][0].float(), ref, bound)
        print(f"DEFECT_Q {defect} {case_id}/{name} {q:.3g}")
        assert q > 1.0, (defect, case_id, name, q)
