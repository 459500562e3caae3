"""Test-set evaluation on the device: csnet_salmetric_images_u8, ModelEngine.forward_images_u8(size=None) (CSNet/test.py with
TEST.IMAGE_H = 0), the native programs op by op, SalImages.evaluate against oracle/salmetric.py, and the bounded native-plan cache."""
import collections

import numpy as np
import pytest
import torch

from oracle import csnet_oracle as O
from oracle import salmetric as OS
from sod100k_b200 import compiler, runtime
from sod100k_b200.data import SalImages
from sod100k_b200.salmetric import image_scores
from tests import fixtures
from tests import sk_native as SN
from tests.test_gpu_images_u8 import SHAPES, _assert_near_exact, _images, _model
from tests.test_gpu_kernels_vs_float64 import _images as _net_input, check_program

pytestmark = pytest.mark.gpu


def _native_shapes(n, seed):
    """ECSSD-like sizes, one already at multiples of 16 (test.py's no-resize branch), and n sizes with h, w drawn from [180, 520]."""
    rng = np.random.default_rng(seed)
    return [(400, 300), (300, 400), (300, 400), (320, 224)] + [tuple(int(v) for v in rng.integers(180, 521, size=2)) for _ in range(n)]


def _masks(shapes, seed):
    """A filled ellipse per image with noisy edges, some GT values around the > 128 rule."""
    rng = np.random.default_rng(seed)
    out = []
    for h, w in shapes:
        yy, xx = np.mgrid[:h, :w]
        cy, cx, ry, rx = rng.uniform(0.3, 0.7) * h, rng.uniform(0.3, 0.7) * w, rng.uniform(0.15, 0.4) * h + 1, rng.uniform(0.15, 0.4) * w + 1
        d = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 + rng.normal(0, 0.1, (h, w))
        m = (d < 1).astype(np.uint8) * 255
        m.reshape(-1)[:3] = [128, 129, 127][:m.size]
        out.append(m)
    return out


def _counts(z, geom, m_dev, y=None):
    N, _, H, W = z.shape
    g = torch.from_numpy(geom.view(np.uint8)).cuda()
    ha = torch.full((N, 256), -1, dtype=torch.int32, device="cuda")            # the call zeroes its outputs
    hp = torch.full((N, 256), -1, dtype=torch.int32, device="cuda")
    ad = torch.full((N,), -1, dtype=torch.int64, device="cuda")
    runtime.salmetric_images_u8(z.data_ptr(), N, H, W, g.data_ptr(), m_dev.data_ptr(), y.data_ptr() if y is not None else 0,
                                ha.data_ptr(), hp.data_ptr(), ad.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return ha.cpu().numpy(), hp.cpu().numpy(), ad.cpu().numpy()


@pytest.mark.parametrize("H,W", [(224, 224), (304, 400)])
def test_salmetric_images_counts_the_resized_maps_exactly(H, W):
    shapes = SHAPES + [(400, 300), (300, 400), (16, 16), (H, W)]
    N = len(shapes)
    geom = runtime.image_geometry(shapes)
    total = int(geom["dst_off"][-1] + geom["h"][-1] * geom["w"][-1])
    gts = _masks(shapes, 5)
    gts[2][:] = 0                                                                # an image without foreground
    m_dev = torch.from_numpy(np.concatenate([g.reshape(-1) for g in gts])).cuda()
    z = (torch.randn((N, 1, H, W), generator=torch.Generator().manual_seed(9)) * 4).cuda()
    z[:, :, 0, :3] = torch.tensor([-100.0, 100.0, 0.0], device="cuda")         # saturated ends and the middle bin
    g = torch.from_numpy(geom.view(np.uint8)).cuda()
    y_ref = torch.full((total,), 0xAB, dtype=torch.uint8, device="cuda")
    runtime.resize_logits_to_u8(z.data_ptr(), N, H, W, g.data_ptr(), y_ref.data_ptr(), torch.cuda.current_stream().cuda_stream)
    y_ref = y_ref.cpu().numpy()
    y = torch.full((total,), 0xCD, dtype=torch.uint8, device="cuda")
    ha, hp, ad = _counts(z, geom, m_dev, y)
    assert np.array_equal(y.cpu().numpy(), y_ref)                               # the stored maps are csnet_resize_logits_to_u8's
    ha0, hp0, ad0 = _counts(z, geom, m_dev)                                      # no map stored: the same counts
    assert np.array_equal(ha0, ha) and np.array_equal(hp0, hp) and np.array_equal(ad0, ad)
    maps = []
    for i, (h, w) in enumerate(shapes):
        o = int(geom["dst_off"][i])
        q, gt = y_ref[o:o + h * w].reshape(h, w), gts[i]
        maps.append(q)
        assert np.array_equal(ha[i], np.bincount(q.reshape(-1), minlength=256)), i
        assert np.array_equal(hp[i], np.bincount(q[gt > 128], minlength=256)), i
        assert ad[i] == np.abs(q.astype(np.int64) - gt).sum(), i
        p, r, _ = image_scores(ha[i:i + 1], hp[i:i + 1], ad[i:i + 1], h * w)
        p_ref, r_ref = OS.precision_recall(q, gt)
        assert np.array_equal(p[0], p_ref) and np.array_equal(r[0], r_ref), i
    # an image alone gets the counts it gets inside the batch
    for k in (0, 6, N - 1):
        gk = runtime.image_geometry([shapes[k]])
        gk["dst_off"] = geom["dst_off"][k]
        a1, p1, d1 = _counts(z[k:k + 1].contiguous(), gk, m_dev)
        assert np.array_equal(a1[0], ha[k]) and np.array_equal(p1[0], hp[k]) and d1[0] == ad[k], k


def test_salmetric_images_rejects_bad_arguments():
    z = torch.zeros((2, 1, 32, 32), device="cuda")
    g = torch.from_numpy(runtime.image_geometry([(8, 8), (8, 8)]).view(np.uint8)).cuda()
    m = torch.zeros(128, dtype=torch.uint8, device="cuda")
    ha = torch.zeros((2, 256), dtype=torch.int32, device="cuda")
    hp = torch.zeros((2, 256), dtype=torch.int32, device="cuda")
    ad = torch.zeros(2, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    good = [z.data_ptr(), 2, 32, 32, g.data_ptr(), m.data_ptr(), 0, ha.data_ptr(), hp.data_ptr(), ad.data_ptr(), s]
    runtime.salmetric_images_u8(*good)
    torch.cuda.synchronize()
    for pos, value in ((0, 0), (4, 0), (5, 0), (7, 0), (8, 0), (9, 0), (1, 0), (1, 65536), (2, 0), (3, 0), (2, 32768), (3, -1)):
        bad = list(good)
        bad[pos] = value
        with pytest.raises(runtime.EngineError):
            runtime.salmetric_images_u8(*bad)


@pytest.mark.parametrize("tag", ["csnet-L-x1", "csnet-L-x2"])
def test_native_mode_matches_the_reference_loop(tag):
    m, cfg, sd = _model(tag)
    imgs = _images(_native_shapes(10, 61), 62)
    eng = m.engine()
    got = [g.numpy() for g in eng.forward_images_u8(imgs, size=None, batch=2)]
    assert [g.shape for g in got] == [im.shape[:2] for im in imgs]
    # test.py's IMAGE_H = 0 loop around the same engine forward (fp32 plans), under test_mixed_sizes_match_the_reference_loop's rule
    _assert_near_exact(got, SN.test_py_native_pipeline(lambda x: m(x.cuda()), imgs, scaled=True), 1e-3)
    # ... and around the oracle network: at most one level apart
    ref = SN.test_py_native_pipeline(lambda x: O.csnet_forward(cfg, sd, x), imgs)
    assert max(np.abs(g.astype(np.int32) - r).max() for g, r in zip(got, ref)) <= 1
    # each map is the fixed-size call at the image's padded size
    for im, g in zip(imgs, got):
        assert np.array_equal(eng.forward_images_u8([im], size=SN.padded_size(*im.shape[:2]))[0].numpy(), g)
    # CUDA tensors in, on the device throughout: the same bytes
    dev = eng.forward_images_u8([torch.from_numpy(im).cuda() for im in imgs], size=None, batch=3)
    assert all(d.is_cuda and np.array_equal(d.cpu().numpy(), g) for d, g in zip(dev, got))


@pytest.mark.parametrize("dtype", ["fp16", "fp32"])
@pytest.mark.parametrize("H,W", [(304, 400), (400, 304), (400, 400)])
def test_native_program_op_by_op(H, W, dtype):
    cfg, sd = fixtures.checkpoint("csnet-L-x2")
    prog = compiler.compile_csnet(cfg, sd, H, W, dtype, reuse_arena=False)
    odd = [o.name for o in prog.ops if any(prog.tensors[t].W % 2 for t in o.dsts)]
    assert odd, "W / 16 odd: some ops write odd-width tensors"
    kernels = check_program(prog, 32, 1, _net_input(1, H, W, 71), f"csnet-L-x2/{dtype}/{H}x{W}")
    print("NATIVE_KERNELS", H, W, dtype, dict(collections.Counter(kernels)), "odd-width ops", len(odd))


def _set(n, seed):
    shapes = _native_shapes(n, seed)
    return _images(shapes, seed + 1), _masks(shapes, seed + 2)


def test_evaluate_scores_the_engine_maps_like_eval_py():
    m, cfg, sd = _model("csnet-L-x2")
    imgs, gts = _set(8, 81)
    ds = SalImages(imgs, gts)
    scores, maps = ds.evaluate(m, size=None, batch=4, maps=True)
    maps = [q.cpu().numpy() for q in maps]
    assert all(np.array_equal(q, g.numpy()) for q, g in zip(maps, m.engine().forward_images_u8(imgs, size=None)))
    assert ds.evaluate(m, size=None, batch=3) == scores                         # counts do not depend on the batch
    ref = OS.evaluate(maps, gts)
    assert scores["max_f"] == ref["max_f"] and scores["argmax"] == ref["argmax"] and scores["mean_f"] == ref["mean_f"]
    # MAE from exact integer sums; the oracle adds float32 terms pixel by pixel
    assert scores["mae"] == pytest.approx(ref["mae"], rel=1e-6)
    # test.py + eval.py around the CPU oracle network: SURVEY 8d's 1e-3
    cpu = OS.evaluate(SN.test_py_native_pipeline(lambda x: O.csnet_forward(cfg, sd, x), imgs), gts)
    assert abs(scores["max_f"] - cpu["max_f"]) <= 1e-3 and abs(scores["mae"] - cpu["mae"]) <= 1e-3
    # the fixed-size mode scores forward_images_u8(size=(224, 224))'s maps
    fixed = ds.evaluate(m, size=(224, 224))
    ref224 = OS.evaluate([q.numpy() for q in m.engine().forward_images_u8(imgs)], gts)
    assert fixed["max_f"] == ref224["max_f"] and fixed["mae"] == pytest.approx(ref224["mae"], rel=1e-6)


def test_native_plans_stay_within_the_budget():
    m, _, _ = _model("csnet-L-x1")
    eng = m.engine()
    fixed = eng.plan_for(2, 224, 224, torch.device("cuda", 0))
    fixed_plans = dict(eng._plans)
    shapes = [(40, 40), (60, 60), (70, 90), (100, 100), (130, 120), (41, 39)]       # five padded sizes
    imgs, gts = _images(shapes, 91), _masks(shapes, 92)
    ds = SalImages(imgs, gts)
    eng.native_plan_budget = 1 << 40
    first = ds.evaluate(m, size=None, batch=2)
    arenas = {k: p.arena_bytes for k, p in eng._native_plans.items()}
    assert len(arenas) == 5
    eng.native_plan_budget = max(arenas.values()) + min(arenas.values())        # holds two plans, not five
    eng.trim_native_plans()
    assert sum(p.arena_bytes for p in eng._native_plans.values()) <= eng.native_plan_budget
    eng.native_plan_budget = 0
    eng.trim_native_plans()
    assert not eng._native_plans
    eng.native_plan_budget = max(arenas.values()) + min(arenas.values())
    again = ds.evaluate(m, size=None, batch=2)
    resident = {k: p.arena_bytes for k, p in eng._native_plans.items()}
    assert 1 <= len(resident) < 5 and sum(resident.values()) <= eng.native_plan_budget
    assert max(resident) == max(arenas)                                          # the last size used stays
    assert again == first
    assert eng._plans == fixed_plans and eng._plans[(224, 224, eng.dtype, 0)] is fixed and fixed._h
