"""Training data on the device (sod100k_b200.data.SalImages: csnet_train_batch_u8, csnet_val_mae_u8) against the host emulation of
the same kernels (tests/emu/train_data.py) and train.py's validation loop in torch (tests/sal_data.py)."""
import random

import numpy as np
import pytest
import torch

from sod100k_b200 import data, runtime
from sod100k_b200.model import csnet
from sod100k_b200.trainer import Trainer
from tests import fixtures
from tests import sal_data as SD
from tests.emu import train_data as E

pytestmark = pytest.mark.gpu

MEAN, STD = data.IMAGENET_MEAN, data.IMAGENET_STD
SIZE = (224, 224)
# edge shapes: 1-pixel images and axes, extreme ratios, identity size, the smallest sides every crop fits (30)
EDGE = [(1, 1), (1, 37), (53, 1), (17, 1000), (224, 224), (30, 30), (31, 517), (81, 7)]


def _set(n, seed, gray_every=5):
    """n seeded images with h, w in [180, 520] plus the edge shapes; every `gray_every`-th image gray."""
    rng = np.random.default_rng(seed)
    shapes = [tuple(int(v) for v in rng.integers(180, 521, size=2)) for _ in range(n)] + EDGE
    imgs, masks = [], []
    for i, (h, w) in enumerate(shapes):
        imgs.append(rng.integers(0, 256, size=(h, w) if i % gray_every == 2 else (h, w, 3), dtype=np.uint8))
        masks.append(rng.integers(0, 256, size=(h, w), dtype=np.uint8))
    return imgs, masks


def _params(sizes, seed):
    """augment_params where the image allows a crop; elsewhere a random window inside the image with a random flip."""
    rng, r = random.Random(seed), np.random.default_rng(seed)
    out = []
    for h, w in sizes:
        try:
            out.append(data.augment_params(rng, h, w))
        except ValueError:
            ch, cw = int(r.integers(1, h + 1)), int(r.integers(1, w + 1))
            out.append((int(r.integers(0, h - ch + 1)), int(r.integers(0, w - cw + 1)), ch, cw, int(r.integers(0, 3))))
    return out


def _emulated(imgs, masks, idx, params, size):
    xs, ts = zip(*[E.train_sample(imgs[i], masks[i], p, size, MEAN, STD) for i, p in zip(idx, params)])
    return np.stack(xs), np.stack(ts)


def test_builder_is_bit_identical_to_the_emulation():
    imgs, masks = _set(56, 1)
    ds = data.SalImages(imgs, masks)
    idx = list(range(len(imgs)))[::-1]                         # not in packing order
    params = _params([imgs[i].shape[:2] for i in idx], 2)
    x, t = ds.train_batch(idx, samples=params)
    ex, et = _emulated(imgs, masks, idx, params, SIZE)
    assert np.array_equal(x.cpu().numpy(), ex) and np.array_equal(t.cpu().numpy(), et)
    # an odd network size too (several column slices, a partial row tile)
    x, t = ds.train_batch(idx[:9], samples=params[:9], size=(130, 300))
    ex, et = _emulated(imgs, masks, idx[:9], params[:9], (130, 300))
    assert np.array_equal(x.cpu().numpy(), ex) and np.array_equal(t.cpu().numpy(), et)


def test_uncropped_network_size_image_is_the_resize_path():
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, size=(224, 224, 3), dtype=np.uint8)
    mask = rng.integers(0, 256, size=(224, 224), dtype=np.uint8)
    ds = data.SalImages([img, img[:100]], [mask, mask[:100]])
    x, t = ds.train_batch([0])
    assert torch.equal(x, ds.val_batch([0]))
    xr = torch.empty_like(x)
    g = torch.from_numpy(runtime.image_geometry([(224, 224)]).view(np.uint8)).cuda()
    runtime.resize_u8_to_input(torch.from_numpy(img).cuda().data_ptr(), g.data_ptr(), 1, 224, 224, MEAN, STD, xr.data_ptr(),
                               torch.cuda.current_stream().cuda_stream)
    assert torch.equal(x, xr)
    assert np.array_equal(t.cpu().numpy()[0, 0], (mask / 255.0).astype(np.float32))


def test_a_sample_alone_equals_it_inside_a_batch():
    imgs, masks = _set(20, 4)
    ds = data.SalImages(imgs, masks)
    idx = list(range(len(imgs)))
    params = _params([im.shape[:2] for im in imgs], 5)
    x, t = ds.train_batch(idx, samples=params)
    for k in (0, 7, len(idx) - 1):
        xk, tk = ds.train_batch([idx[k]], samples=[params[k]])
        assert torch.equal(xk[0], x[k]) and torch.equal(tk[0], t[k])


def test_trainer_steps_fed_from_sal_images_equal_steps_fed_the_emulation():
    """Three Trainer.steps on SalImages.train_batch against three on the emulated batches uploaded as tensors: the same inputs, so the
    same losses and bit-identical parameters (every gradient kernel merges its partial sums in a fixed order)."""
    rng = np.random.default_rng(6)
    shapes = [tuple(int(v) for v in rng.integers(40, 200, size=2)) for _ in range(12)]
    imgs = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in shapes]
    masks = [(rng.random((h, w)) < 0.4).astype(np.uint8) * 255 for h, w in shapes]
    size = (64, 96)
    outs = []
    for fed in ("sal_images", "emulated"):
        cfg, sd = fixtures.checkpoint("csnet-L-x2")
        m = csnet.CSNet(cfg)
        m.load_state_dict(sd)
        m.cuda().train()
        tr = Trainer(m, lr=1e-3, weight_decay=5e-3)
        ds = data.SalImages(imgs, masks) if fed == "sal_images" else None
        aug = random.Random(7)
        order = torch.randperm(len(imgs), generator=torch.Generator().manual_seed(8))
        losses = []
        for idx in order.split(4):
            if ds is not None:
                losses.append(tr.step(*ds.train_batch(idx, aug, size=size)))
            else:
                params = [data.augment_params(aug, *shapes[i]) for i in idx.tolist()]
                x, t = _emulated(imgs, masks, idx.tolist(), params, size)
                losses.append(tr.step(torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda()))
        torch.cuda.synchronize()
        outs.append(([float(l) for l in losses], {k: v.detach().clone() for k, v in m.state_dict().items()}))
    assert all(abs(a - b) <= 1e-6 * abs(a) for a, b in zip(outs[0][0], outs[1][0]))
    for k, v in outs[0][1].items():
        assert torch.equal(v, outs[1][1][k]), k


def test_val_mae_matches_the_torch_loop_and_is_deterministic():
    cfg, sd = fixtures.checkpoint("csnet-L-x2")
    m = csnet.CSNet(cfg)
    m.load_state_dict(sd)
    m.cuda().eval()
    imgs, masks = _set(24, 9)
    # masks shaped like saliency GT: a blob of 255 on 0, plus some grey edge values
    for k, mk in enumerate(masks):
        h, w = mk.shape
        yy, xx = np.mgrid[:h, :w]
        r = ((yy - h / 2) / max(h, 1)) ** 2 + ((xx - w / 2) / max(w, 1)) ** 2
        masks[k] = np.where(r < 0.08, 255, np.where(r < 0.1, mk, 0)).astype(np.uint8)
    ds = data.SalImages(imgs, masks)
    idx = list(range(len(imgs)))
    with torch.no_grad():
        z = m(ds.val_batch(idx))
    got = ds.val_mae(z, idx)
    assert got.dtype == torch.float64 and got.is_cuda and got.shape == (len(idx),)
    want = SD.val_mae_loop(z, masks)
    slack = SD.val_mae_slack(z, masks)
    for g, w_, s in zip(got.tolist(), want, slack):
        assert abs(g - w_) <= 1e-6 * abs(w_) + s, (g, w_, s)
    assert torch.equal(ds.val_mae(z, idx), got)                  # a second run
    perm = torch.randperm(len(idx), generator=torch.Generator().manual_seed(10))
    again = ds.val_mae(z[perm], perm)                           # another batch order
    assert torch.equal(again, got[perm])
    part = ds.val_mae(z[3:9].clone(), idx[3:9])                 # another batch composition
    assert torch.equal(part, got[3:9])


def test_rejections_raise_before_any_device_work(monkeypatch):
    ok_img, ok_mask = np.zeros((40, 50, 3), np.uint8), np.zeros((40, 50), np.uint8)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    bad_sets = [
        ([], []),                                               # an empty set
        ([ok_img], []),                                         # counts differ
        ([ok_img.astype(np.float32)], [ok_mask]),               # wrong dtype
        ([np.zeros((40, 50, 4), np.uint8)], [ok_mask]),         # wrong channels
        ([np.zeros((2, 40, 50, 3), np.uint8)], [ok_mask]),      # wrong rank
        ([ok_img], [np.zeros((40, 50, 1), np.uint8)]),          # mask rank
        ([ok_img], [np.zeros((40, 51), np.uint8)]),             # mask of another size
        ([ok_img], [ok_mask.astype(np.int16)]),                 # mask dtype
        ([np.zeros((0, 50, 3), np.uint8)], [np.zeros((0, 50), np.uint8)]),            # a side of 0
        ([np.zeros((1, 32768), np.uint8)], [np.zeros((1, 32768), np.uint8)]),         # a side over 32767
        ([[[1, 2, 3]]], [ok_mask]),                             # not an array
    ]
    for imgs, masks in bad_sets:
        with pytest.raises(ValueError):
            data.SalImages(imgs, masks)
    assert torch.cuda.memory_allocated() == before
    ds = data.SalImages([ok_img, np.zeros((20, 20, 3), np.uint8)], [ok_mask, np.zeros((20, 20), np.uint8)])

    def launched(*a, **k):
        raise AssertionError("a rejected call launched a kernel")

    for name in ("train_batch_u8", "val_mae_u8", "resize_u8_to_input"):
        monkeypatch.setattr(runtime, name, launched)
    bad_calls = [
        lambda: ds.train_batch([0, 2]),                                         # an index past the set
        lambda: ds.train_batch([-1]),
        lambda: ds.train_batch([]),
        lambda: ds.train_batch([1], random.Random(0)),                          # seed 0's first crop does not fit 20 x 20
        lambda: ds.train_batch([0], random.Random(0), samples=[(0, 0, 40, 50, 0)]),   # both
        lambda: ds.train_batch([0], samples=[(0, 0, 41, 50, 0)]),               # a window past the image
        lambda: ds.train_batch([0], samples=[(1, 0, 40, 50, 0)]),
        lambda: ds.train_batch([0], samples=[(0, -1, 4, 5, 0)]),
        lambda: ds.train_batch([0], samples=[(0, 0, 0, 5, 0)]),                 # an empty window
        lambda: ds.train_batch([0], samples=[(0, 0, 4, 5, 3)]),                 # an unknown flip
        lambda: ds.train_batch([0, 1], samples=[(0, 0, 4, 5, 0)]),              # one window for two samples
        lambda: ds.val_batch([2]),
        lambda: ds.val_mae(torch.zeros((1, 1, 8, 8), device="cuda"), [0, 1]),   # logits for another batch size
        lambda: ds.val_mae(torch.zeros((2, 1, 8, 8)), [0, 1]),                  # host logits
        lambda: ds.val_mae(torch.zeros((2, 1, 8, 8), dtype=torch.float16, device="cuda"), [0, 1]),
        lambda: ds.val_mae(torch.zeros((2, 2, 8, 8), device="cuda"), [0, 1]),
    ]
    for call in bad_calls:
        with pytest.raises(ValueError):
            call()


def test_non_default_stream():
    imgs, masks = _set(6, 11)
    ds = data.SalImages(imgs, masks)
    idx = list(range(len(imgs)))
    params = _params([im.shape[:2] for im in imgs], 12)
    x0, t0 = ds.train_batch(idx, samples=params)
    z = torch.randn((len(idx), 1, 224, 224), generator=torch.Generator().manual_seed(13)).mul_(4).cuda()
    mae0 = ds.val_mae(z, idx)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)                           # keep the side stream busy so an unordered read would see garbage
        x1, t1 = ds.train_batch(idx, samples=params)
        mae1 = ds.val_mae(z, idx)
        ev = torch.cuda.Event()
        ev.record(s)
    ev.synchronize()
    assert torch.equal(x0, x1) and torch.equal(t0, t1) and torch.equal(mae0, mae1)
