"""CSF+Res2Net test-set evaluation on the device: csnet_csf_input_u8 / csnet_csf_maps_u8 / csnet_salmetric_csf_u8 against the reference's
load_image_test and cv2 bytes, torch's sigmoid and oracle/salmetric.py; CSFNet.forward_images_u8 and SalImages.evaluate against
solver.test's loop around the same network and around the CPU oracle network."""
import os

import numpy as np
import pytest
import torch

from oracle import csf_res2net_oracle as R
from oracle import salmetric as OS
from sod100k_b200 import modular_r, runtime, synth
from sod100k_b200.data import SalImages
from sod100k_b200.engine import trim_plans
from sod100k_b200.networks import csf_res2net
from sod100k_b200.salmetric import image_scores
from tests import csf_ref, fixtures

pytestmark = pytest.mark.gpu

SEED = 21
# four sizes, repeated so that runs batch; 75x100, 100x75 and 37x53 are not multiples of 32; one gray image
SHAPES = [(75, 100), (100, 75), (37, 53), (75, 100), (64, 64), (100, 75), (37, 53), (75, 100), (64, 64), (75, 100)]
GRAY = 4


@pytest.fixture(autouse=True, scope="module")
def _deterministic():
    b = torch.backends
    saved = (b.cudnn.deterministic, b.cudnn.benchmark, b.cudnn.allow_tf32, b.cuda.matmul.allow_tf32)
    b.cudnn.deterministic, b.cudnn.benchmark, b.cudnn.allow_tf32, b.cuda.matmul.allow_tf32 = True, False, False, False
    yield
    b.cudnn.deterministic, b.cudnn.benchmark, b.cudnn.allow_tf32, b.cuda.matmul.allow_tf32 = saved


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _geom_dev(geom):
    return torch.from_numpy(geom.view(np.uint8)).cuda()


def _model():
    m = csf_res2net.build_model()
    sd = synth.synth_state_r({k: tuple(v.shape) for k, v in m.state_dict().items()}, SEED)
    sd = {k: torch.from_numpy(v) for k, v in sd.items()}
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval(), sd


def _images(shapes, seed):
    """Smooth seeded images (a gradient plus noise) so the maps spread over many levels; image GRAY is gray [h, w]."""
    rng = np.random.default_rng(seed)
    out = []
    for i, (h, w) in enumerate(shapes):
        yy, xx = np.mgrid[:h, :w]
        base = (yy / max(h - 1, 1) * 180 + xx / max(w - 1, 1) * 60)[:, :, None] + rng.normal(0, 25, (h, w, 3))
        im = np.clip(base, 0, 255).astype(np.uint8)
        out.append(im[:, :, 1].copy() if i == GRAY else im)
    return out


def _masks(shapes, seed):
    rng = np.random.default_rng(seed)
    out = []
    for h, w in shapes:
        yy, xx = np.mgrid[:h, :w]
        d = ((yy - 0.5 * h) / (0.3 * h + 1)) ** 2 + ((xx - 0.5 * w) / (0.3 * w + 1)) ** 2 + rng.normal(0, 0.2, (h, w))
        m = (d < 1).astype(np.uint8) * 255
        m.reshape(-1)[:3] = [128, 129, 127][:m.size]
        out.append(m)
    return out


def _csf_input(imgs, H, W, mean=csf_ref.MEAN, std=csf_ref.STD):
    geom = runtime.image_geometry([(H, W)] * len(imgs))
    x = torch.from_numpy(np.concatenate([np.ascontiguousarray(im).reshape(-1) for im in imgs])).cuda()
    out = torch.full((len(imgs), 3, H, W), float("nan"), device="cuda")
    g = _geom_dev(geom)
    runtime.csf_input_u8(x.data_ptr(), g.data_ptr(), len(imgs), H, W, mean, std, out.data_ptr(), _stream())
    return out.cpu().numpy()


def test_csf_input_matches_load_image_test_bit_for_bit():
    z = np.load(os.path.join(fixtures.GOLDEN, "csf_eval.npz"))
    for tag in ("1x1", "3x5", "37x53", "75x100", "gray"):
        img, ref = z[f"{tag}/image"], z[f"{tag}/x"]
        got = _csf_input([img], *img.shape[:2])[0]
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), tag
    rng = np.random.default_rng(7)
    imgs = [rng.integers(0, 256, size=(300, 400, 3), dtype=np.uint8) for _ in range(3)]
    imgs[1][:16, :16] = np.arange(256, dtype=np.uint8).reshape(16, 16, 1)       # every value in every channel
    got = _csf_input(imgs, 300, 400)
    for i, im in enumerate(imgs):
        assert np.array_equal(got[i].view(np.uint32), csf_ref.load_image_test(im).view(np.uint32)), i


def _logit_sweep():
    """A dense sweep over the range where the map byte changes, the 257 consecutive fp32 values around each logit(k + 0.5) / 255
    (where the ties lie), random logits, and saturated values, as [4, 1, 1024, 1280]."""
    n = 4 * 1024 * 1280
    k = torch.arange(255, dtype=torch.float64) + 0.5
    mid = torch.log(k / (255 - k)).float()
    steps = torch.arange(-128, 129, dtype=torch.int32)
    near = (mid.view(torch.int32)[:, None] + torch.where(mid[:, None] < 0, -steps, steps)).view(torch.float32).reshape(-1)
    rand = torch.randn(1 << 20, generator=torch.Generator().manual_seed(11)) * 4
    ends = torch.tensor([0.0, -0.0, 100.0, -100.0, 1e30, -1e30, float("inf"), float("-inf")])
    sweep = torch.linspace(-12.0, 12.0, n - near.numel() - rand.numel() - ends.numel(), dtype=torch.float32)
    return torch.cat([sweep, near, rand, ends]).view(4, 1, 1024, 1280).cuda()


def test_csf_maps_equal_torch_round_of_sigmoid():
    z = _logit_sweep()
    N, _, H, W = z.shape
    v = 255 * torch.sigmoid(z)
    assert int((v - v.floor() == 0.5).sum()) > 100                               # the sweep holds exact ties
    ref = torch.round(v).clamp(0, 255).to(torch.uint8).reshape(-1)
    geom = runtime.image_geometry([(H, W)] * N)
    y = torch.full((N * H * W,), 0xAB, dtype=torch.uint8, device="cuda")
    runtime.csf_maps_u8(z.data_ptr(), N, H, W, _geom_dev(geom).data_ptr(), y.data_ptr(), _stream())
    bad = (y != ref).nonzero()
    assert bad.numel() == 0, (bad.numel(), z.reshape(-1)[bad[:8, 0]].tolist(), y[bad[:8, 0]].tolist(), ref[bad[:8, 0]].tolist())


def _counts(z, geom, m_dev, y=None, fn=runtime.salmetric_csf_u8):
    N, _, H, W = z.shape
    ha = torch.full((N, 256), -1, dtype=torch.int32, device="cuda")            # the call zeroes its outputs
    hp = torch.full((N, 256), -1, dtype=torch.int32, device="cuda")
    ad = torch.full((N,), -1, dtype=torch.int64, device="cuda")
    g = _geom_dev(geom)
    fn(z.data_ptr(), N, H, W, g.data_ptr(), m_dev.data_ptr(), y.data_ptr() if y is not None else 0, ha.data_ptr(), hp.data_ptr(),
       ad.data_ptr(), _stream())
    return ha.cpu().numpy(), hp.cpu().numpy(), ad.cpu().numpy()


@pytest.mark.parametrize("H,W", [(75, 100), (37, 53), (1, 1)])
def test_salmetric_csf_counts_the_maps_exactly(H, W):
    N = 5
    geom = runtime.image_geometry([(H, W)] * N)
    gts = _masks([(H, W)] * N, H + W)
    gts[1][:] = 0                                                                # an image without foreground
    m_dev = torch.from_numpy(np.concatenate([g.reshape(-1) for g in gts])).cuda()
    z = (torch.randn((N, 1, H, W), generator=torch.Generator().manual_seed(H)) * 4).cuda()
    z.view(-1)[:3] = torch.tensor([-100.0, 100.0, 0.0], device="cuda")[:z.numel()]
    y_ref = torch.full((N * H * W,), 0xAB, dtype=torch.uint8, device="cuda")
    runtime.csf_maps_u8(z.data_ptr(), N, H, W, _geom_dev(geom).data_ptr(), y_ref.data_ptr(), _stream())
    y_ref = y_ref.cpu().numpy()
    y = torch.full((N * H * W,), 0xCD, dtype=torch.uint8, device="cuda")
    ha, hp, ad = _counts(z, geom, m_dev, y)
    assert np.array_equal(y.cpu().numpy(), y_ref)                               # the stored maps are csnet_csf_maps_u8's
    ha0, hp0, ad0 = _counts(z, geom, m_dev)                                      # no map stored: the same counts
    assert np.array_equal(ha0, ha) and np.array_equal(hp0, hp) and np.array_equal(ad0, ad)
    maps = []
    for i in range(N):
        q, gt = y_ref[i * H * W:(i + 1) * H * W].reshape(H, W), gts[i]
        maps.append(q)
        assert np.array_equal(ha[i], np.bincount(q.reshape(-1), minlength=256)), i
        assert np.array_equal(hp[i], np.bincount(q[gt > 128], minlength=256)), i
        assert ad[i] == np.abs(q.astype(np.int64) - gt).sum(), i
        p, r, _ = image_scores(ha[i:i + 1], hp[i:i + 1], ad[i:i + 1], H * W)
        p_ref, r_ref = OS.precision_recall(q, gt)
        assert np.array_equal(p[0], p_ref) and np.array_equal(r[0], r_ref), i
    # other batch splits give every image the same counts
    for a, b in ((0, 1), (1, 3), (3, 5), (4, 5)):
        gk = geom[a:b].copy()
        a1, p1, d1 = _counts(z[a:b].contiguous(), gk, m_dev)
        assert np.array_equal(a1, ha[a:b]) and np.array_equal(p1, hp[a:b]) and np.array_equal(d1, ad[a:b]), (a, b)


def test_csf_calls_reject_bad_arguments():
    z = torch.zeros((2, 1, 8, 8), device="cuda")
    g = _geom_dev(runtime.image_geometry([(8, 8), (8, 8)]))
    m = torch.zeros(128, dtype=torch.uint8, device="cuda")
    x = torch.zeros(384, dtype=torch.uint8, device="cuda")
    xin = torch.zeros((2, 3, 8, 8), device="cuda")
    ha = torch.zeros((2, 256), dtype=torch.int32, device="cuda")
    hp = torch.zeros((2, 256), dtype=torch.int32, device="cuda")
    ad = torch.zeros(2, dtype=torch.int64, device="cuda")
    s = _stream()
    good = [z.data_ptr(), 2, 8, 8, g.data_ptr(), m.data_ptr(), 0, ha.data_ptr(), hp.data_ptr(), ad.data_ptr(), s]
    runtime.salmetric_csf_u8(*good)
    torch.cuda.synchronize()
    for pos, value in ((0, 0), (4, 0), (5, 0), (7, 0), (8, 0), (9, 0), (1, 0), (1, 65536), (2, 0), (3, 0), (2, 32768), (3, -1)):
        bad = list(good)
        bad[pos] = value
        with pytest.raises(runtime.EngineError):
            runtime.salmetric_csf_u8(*bad)
    good = [z.data_ptr(), 2, 8, 8, g.data_ptr(), m.data_ptr(), s]
    runtime.csf_maps_u8(*good)
    for pos, value in ((0, 0), (4, 0), (5, 0), (1, 0), (1, 65536), (2, 0), (3, -1), (3, 32768)):
        bad = list(good)
        bad[pos] = value
        with pytest.raises(runtime.EngineError):
            runtime.csf_maps_u8(*bad)
    good = [x.data_ptr(), g.data_ptr(), 2, 8, 8, csf_ref.MEAN, csf_ref.STD, xin.data_ptr(), s]
    runtime.csf_input_u8(*good)
    torch.cuda.synchronize()
    for pos, value in ((0, 0), (1, 0), (7, 0), (2, 0), (2, 65536), (3, 0), (4, -1), (4, 32768)):
        bad = list(good)
        bad[pos] = value
        with pytest.raises(runtime.EngineError):
            runtime.csf_input_u8(*bad)
    lib = runtime.load_library()
    assert lib.csnet_csf_input_u8(x.data_ptr(), g.data_ptr(), 2, 8, 8, None, None, xin.data_ptr(), s) == -1


@pytest.fixture(scope="module")
def net():
    return _model()


@pytest.fixture(scope="module")
def data():
    return _images(SHAPES, 3), _masks(SHAPES, 4)


def test_evaluate_equals_the_solver_test_loop(net, data):
    m, sd = net
    imgs, gts = data
    m.set_precision("fp32")
    m.plan_budget = csf_res2net.PLAN_BUDGET
    ds = SalImages(imgs, gts)
    scores, maps = ds.evaluate(m, batch=1, maps=True)
    maps = [q.cpu().numpy() for q in maps]
    assert [q.shape for q in maps] == [tuple(s) for s in SHAPES]
    loop = csf_ref.solver_test(m, imgs)
    for i, (q, r) in enumerate(zip(maps, loop)):
        assert np.array_equal(q, r), (i, int((q != r).sum()))
    ref = OS.evaluate(maps, gts)
    assert scores["max_f"] == ref["max_f"] and scores["mean_f"] == ref["mean_f"] and scores["argmax"] == ref["argmax"]
    assert scores["mae"] == pytest.approx(ref["mae"], rel=1e-6)
    assert max(len(np.unique(q)) for q in maps) > 16                            # the maps are not flat
    # batched runs: within one level of batch 1 (cuDNN and the head may pick other kernels at other batches)
    s4, maps4 = ds.evaluate(m, batch=4, maps=True)
    assert max(np.abs(q.cpu().numpy().astype(np.int32) - r).max() for q, r in zip(maps4, maps)) <= 1
    assert ds.evaluate(m, batch=4) == s4                                        # the counts are exact
    # solver.test around the CPU oracle network (torch's CPU sigmoid)
    cpu = OS.evaluate(csf_ref.solver_test(lambda x: R.csfnet_forward(sd, x.cpu()), imgs), gts)
    assert abs(scores["max_f"] - cpu["max_f"]) <= 1e-3 and abs(scores["mae"] - cpu["mae"]) <= 1e-3, (scores, cpu)
    with pytest.raises(ValueError):
        ds.evaluate(m, size=(224, 224))


def test_forward_images_u8_host_and_cuda_inputs_agree(net, data):
    m, _ = net
    imgs, gts = data
    m.set_precision("fp32")
    host = m.forward_images_u8(imgs, batch=3)
    assert all(not q.is_cuda and q.is_pinned() and tuple(q.shape) == tuple(s) for q, s in zip(host, SHAPES))
    dev = m.forward_images_u8([torch.from_numpy(im).cuda() for im in imgs], batch=3)
    assert all(d.is_cuda and np.array_equal(d.cpu().numpy(), h.numpy()) for d, h in zip(dev, host))
    tensors = m.forward_images_u8([torch.from_numpy(im) for im in imgs], batch=3)
    assert all(np.array_equal(t.numpy(), h.numpy()) for t, h in zip(tensors, host))
    _, maps3 = SalImages(imgs, gts).evaluate(m, batch=3, maps=True)
    assert all(np.array_equal(q.cpu().numpy(), h.numpy()) for q, h in zip(maps3, host))
    # the gray image is cv2.IMREAD_COLOR's three equal channels
    gray3 = np.repeat(imgs[GRAY][:, :, None], 3, axis=2)
    assert np.array_equal(m.forward_images_u8([gray3])[0].numpy(), m.forward_images_u8([imgs[GRAY]])[0].numpy())
    assert m.forward_images_u8([]) == []
    with pytest.raises(ValueError):
        m.forward_images_u8([np.zeros((4, 4, 4), np.uint8)])
    with pytest.raises(ValueError):
        m.forward_images_u8([np.zeros((4, 4, 3), np.float32)])


def test_fp16_equals_the_fp16_loop(net, data):
    m, _ = net
    imgs, gts = data
    m.set_precision("fp16")
    try:
        _, maps = SalImages(imgs, gts).evaluate(m, batch=1, maps=True)
        loop = csf_ref.solver_test(m, imgs)
        for i, (q, r) in enumerate(zip(maps, loop)):
            assert np.array_equal(q.cpu().numpy(), r), (i, int((q.cpu().numpy() != r).sum()))
    finally:
        m.set_precision("fp32")


def test_plans_stay_within_a_small_budget(net, data):
    m, _ = net
    imgs, gts = data
    ds = SalImages(imgs, gts)
    trim_plans(m._plans, 0, m._plan_version)                                      # every plan below is made at max_batch 2
    m.plan_budget = 1 << 40
    first = ds.evaluate(m, batch=2)
    arenas = {k: p.arena_bytes for k, p in m._plans.items() if k[2] == "fp32"}
    assert len(arenas) >= 4
    m.plan_budget = max(arenas.values()) + min(arenas.values())
    try:
        assert ds.evaluate(m, batch=2) == first
        resident = {k: p.arena_bytes for k, p in m._plans.items()}
        assert 1 <= len(resident) < 4 and sum(resident.values()) <= m.plan_budget
        assert set(m._plan_version) == set(m._plans)
        m.plan_budget = 0                                                         # only the plan in use stays
        assert ds.evaluate(m, batch=2) == first
        assert len(m._plans) == 1
    finally:
        m.plan_budget = csf_res2net.PLAN_BUDGET


def test_grad_enabled_never_takes_the_training_path(net, data, monkeypatch):
    m, _ = net
    imgs, gts = data
    ds = SalImages(imgs[:3], gts[:3])
    ref = ds.evaluate(m, batch=2)

    def stub(*a, **k):
        raise AssertionError("the training head ran")

    monkeypatch.setattr(modular_r, "csf_head", stub)
    assert any(q.requires_grad for q in m.parameters())
    with torch.enable_grad():
        assert ds.evaluate(m, batch=2) == ref
        m.forward_images_u8(imgs[:3])
        with pytest.raises(AssertionError):                                       # the stub is what forward reaches with grad
            m(torch.zeros((1, 3, 32, 32), device="cuda"))


def test_train_mode_raises(net, data):
    m, _ = net
    imgs, gts = data
    ds = SalImages(imgs[:2], gts[:2])
    m.train()
    try:
        with torch.no_grad():
            with pytest.raises(NotImplementedError):
                ds.evaluate(m)
            with pytest.raises(NotImplementedError):
                m.forward_images_u8(imgs[:2])
    finally:
        m.eval()
