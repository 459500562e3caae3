"""Images of any size through the engine (csnet_resize_u8_to_input, csnet_resize_logits_to_u8, csnet_plan_run_host_images_u8,
ModelEngine.forward_images_u8) against the reference's host loop CSNet/test.py:71-98 restated with scipy (tests/sk_resize.py)."""
import numpy as np
import pytest
import torch

from oracle import csnet_oracle as O
from sod100k_b200 import runtime
from sod100k_b200.model import csnet
from tests import fixtures
from tests import sk_resize as SK
from tests.emu import image_io as E

pytestmark = pytest.mark.gpu

MEAN, STD = SK.IMAGENET_MEAN, SK.IMAGENET_STD
SIZE = (224, 224)
# the CPU test's shapes (tests/test_resize_oracle.py): down, up, identity, one-pixel / one-sample axes, extreme ratios, odd sizes
SHAPES = [(500, 375), (100, 80), (224, 224), (1, 1), (1, 37), (53, 1), (17, 1000), (181, 517), (1, 333), (333, 1), (81, 7)]


def _model(tag):
    cfg, sd = fixtures.checkpoint(tag)
    m = csnet.CSNet(cfg)
    m.load_state_dict(sd)
    return m.cuda().eval(), cfg, sd


def _images(shapes, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in shapes]


def _mixed(n, seed):
    """n seeded sizes with h, w in [180, 520], plus the extreme shapes."""
    rng = np.random.default_rng(seed)
    return [tuple(int(v) for v in rng.integers(180, 521, size=2)) for _ in range(n)] + SHAPES


def _assert_near_exact(got, scaled, window):
    """uint8 maps equal the truncated float maps except within `window` of an integer, where they may differ by 1."""
    for g, v in zip(got, scaled):
        v = v.astype(np.float64)
        d = np.abs(g.astype(np.int32) - np.floor(v).astype(np.int32))
        near = np.abs(v - np.round(v)) < window
        assert d[~near].max(initial=0) == 0 and d.max(initial=0) <= 1


def test_device_primitives_match_zoom():
    imgs = _images(SHAPES, 11)
    geom = runtime.image_geometry([im.shape[:2] for im in imgs])
    N, (H, W) = len(imgs), SIZE
    g = torch.from_numpy(geom.view(np.uint8)).cuda()
    x = torch.from_numpy(np.concatenate([im.reshape(-1) for im in imgs])).cuda()
    x_in = torch.empty((N, 3, H, W), dtype=torch.float32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    runtime.resize_u8_to_input(x.data_ptr(), g.data_ptr(), N, H, W, MEAN, STD, x_in.data_ptr(), stream)
    m, s = np.asarray(MEAN, np.float32).astype(np.float64), np.asarray(STD, np.float32).astype(np.float64)
    got = x_in.cpu().numpy()
    for i, im in enumerate(imgs):
        want = np.transpose((SK.resize(im.astype(np.float64) / 255.0, SIZE) - m) / s, (2, 0, 1)).astype(np.float32)
        assert (np.abs(got[i].astype(np.float64) - want) <= np.spacing(np.maximum(np.abs(got[i]), np.abs(want)))).all(), i
    z = (torch.randn((N, 1, H, W), generator=torch.Generator().manual_seed(3)) * 4).cuda()
    y = torch.full((int(geom["dst_off"][-1] + geom["h"][-1] * geom["w"][-1]),), 0xAB, dtype=torch.uint8, device="cuda")
    runtime.resize_logits_to_u8(z.data_ptr(), N, H, W, g.data_ptr(), y.data_ptr(), stream)
    y = y.cpu().numpy()
    zs = z.cpu().numpy()
    got, scaled = [], []
    for i, im in enumerate(imgs):
        o, (h, w) = int(geom["dst_off"][i]), im.shape[:2]
        got.append(y[o:o + h * w].reshape(h, w))
        scaled.append(SK.resize(E.sigmoid(zs[i, 0]), (h, w)) * np.float32(255))
    # the CPU test's 1e-5 window, widened for the device expf (within 2 ulp of the host's: <= 3e-5 of a level after * 255)
    _assert_near_exact(got, scaled, 1e-4)


@pytest.mark.parametrize("dtype", ["fp32", "fp16"])
def test_network_size_images_give_the_uint8_path_bytes(dtype):
    m, _, _ = _model("csnet-L-x2")
    m.set_precision(dtype)
    img = np.random.default_rng(7).integers(0, 256, size=(12, 224, 224, 3), dtype=np.uint8)
    want = m.engine().forward_host_u8(torch.from_numpy(img))
    got = m.engine().forward_images_u8(list(img))
    assert all(torch.equal(g, w) for g, w in zip(got, want))


@pytest.mark.parametrize("tag", ["csnet-L-x1", "csnet-L-x2"])
def test_mixed_sizes_match_the_reference_loop(tag):
    m, cfg, sd = _model(tag)
    imgs = _images(_mixed(64, 21), 22)                        # 75 images: the host pipeline runs its chunks
    eng = m.engine()
    got = [g.numpy() for g in eng.forward_images_u8(imgs)]
    assert [g.shape for g in got] == [im.shape[:2] for im in imgs]
    # the reference loop around the same engine forward (fp32 plan): exact but where fp32 rounding can cross an integer
    _assert_near_exact(got, SK.test_py_pipeline(lambda x: m(x.cuda()), imgs, SIZE, scaled=True), 1e-3)
    # ... and around the oracle network: the 1e-3 sigmoid gate is 0.255 of a level, so at most one level apart
    ref = SK.test_py_pipeline(lambda x: O.csnet_forward(cfg, sd, x), imgs, SIZE)
    assert max(np.abs(g.astype(np.int32) - r).max() for g, r in zip(got, ref)) <= 1
    # CUDA tensors in, on the device throughout: the same bytes
    dev = eng.forward_images_u8([torch.from_numpy(im).cuda() for im in imgs])
    assert all(d.is_cuda and np.array_equal(d.cpu().numpy(), g) for d, g in zip(dev, got))
    # an image alone gives the bytes it gets inside the batch
    for k in (0, 5, len(imgs) - 1):
        assert np.array_equal(eng.forward_images_u8([imgs[k]])[0].numpy(), got[k])


def test_fp16_is_within_three_levels_of_fp32():
    m, _, _ = _model("csnet-L-x2")
    imgs = _images(_mixed(16, 31), 32)
    y32 = m.engine().forward_images_u8(imgs)
    m.set_precision("fp16")
    y16 = m.engine().forward_images_u8(imgs)
    assert max((a.int() - b.int()).abs().max().item() for a, b in zip(y16, y32)) <= 3


def test_bad_images_and_geometry_are_rejected():
    m, _, _ = _model("csnet-L-x1")
    eng = m.engine()
    ok = np.zeros((20, 30, 3), np.uint8)
    for bad in (np.zeros((20, 30), np.uint8), np.zeros((20, 30, 4), np.uint8), np.zeros((20, 30, 1), np.uint8),
                np.zeros((0, 30, 3), np.uint8), np.zeros((20, 0, 3), np.uint8), np.zeros((20, 30, 3), np.float32),
                torch.zeros((20, 30, 3), dtype=torch.int16), [[1, 2, 3]]):
        with pytest.raises(ValueError):
            eng.forward_images_u8([ok, bad])
    with pytest.raises(ValueError):
        eng.forward_images_u8([ok, torch.from_numpy(ok).cuda()])
    # the C call checks every entry before any copy or launch: the output buffer stays untouched
    plan = eng.plan_for(2, 64, 64, torch.device("cuda", 0))
    x = torch.zeros(2 * 20 * 30 * 3, dtype=torch.uint8).pin_memory()
    y = torch.full((2 * 20 * 30,), 0xAB, dtype=torch.uint8).pin_memory()
    good = runtime.image_geometry([(20, 30), (20, 30)])
    plan.run_host_images_u8(2, x.data_ptr(), x.numel(), good, y.data_ptr(), y.numel(), MEAN, STD)
    assert (y != 0xAB).any()
    src1, dst1 = int(good["src_off"][1]), int(good["dst_off"][1])
    # an empty side, a side over 32767, the second image past the input's end, a negative offset, a map not starting where the
    # previous one ends
    for field, value in (("h", 0), ("w", 32768), ("h", 21), ("src_off", src1 + 1), ("src_off", -1), ("dst_off", dst1 - 1)):
        g = good.copy()
        g[field][1] = value
        y.fill_(0xAB)
        with pytest.raises(runtime.EngineError):
            plan.run_host_images_u8(2, x.data_ptr(), x.numel(), g, y.data_ptr(), y.numel(), MEAN, STD)
        assert (y == 0xAB).all()
    with pytest.raises(runtime.EngineError):                   # the input buffer one byte short
        plan.run_host_images_u8(2, x.data_ptr(), x.numel() - 1, good, y.data_ptr(), y.numel(), MEAN, STD)
    with pytest.raises(runtime.EngineError):                   # the output buffer one byte short
        plan.run_host_images_u8(2, x.data_ptr(), x.numel(), good, y.data_ptr(), y.numel() - 1, MEAN, STD)
