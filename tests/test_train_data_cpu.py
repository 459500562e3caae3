"""Training data without a GPU: sod100k_b200.data.augment_params against the reference's recorded draws (tests/golden/augment.json),
and the per-pixel arithmetic of train_batch_u8_kernel / val_mae_u8_kernel (sod100k_b200/csrc/image_io.cuh, compiled for the host by
tests/emu) against SalData.__getitem__ restated with scipy and train.py's val loop in torch (tests/sal_data.py)."""
import json
import os
import random

import numpy as np
import pytest
import torch

from sod100k_b200 import data
from tests import sal_data as SD
from tests.emu import train_data as E

HERE = os.path.dirname(os.path.abspath(__file__))
MEAN, STD = data.IMAGENET_MEAN, data.IMAGENET_STD
FLIPS = {None: 0, "lr": 1, "ud": 2}


def test_augment_params_draw_the_reference_params():
    with open(os.path.join(HERE, "golden", "augment.json")) as f:
        cases = json.load(f)["cases"]
    errors = 0
    for c in cases:
        rng = random.Random(c["seed"])
        h, w = c["h"], c["w"]
        for d in c["draws"]:
            if isinstance(d, str):
                with pytest.raises(ValueError, match="too small"):
                    data.augment_params(rng, h, w)
                errors += 1
                continue
            row1, row2, col1, col2, flip = d
            assert data.augment_params(rng, h, w) == (row1, col1, h + row2 - row1, w + col2 - col1, FLIPS[flip])
    assert errors > 0


def _sample(h, w, seed, gray=False):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, size=(h, w) if gray else (h, w, 3), dtype=np.uint8)
    mask = rng.integers(0, 256, size=(h, w), dtype=np.uint8)
    return img, mask


def _within_one_ulp(got, want):
    want = want.astype(np.float32)
    ulp = np.spacing(np.maximum(np.abs(got), np.abs(want)))
    return (np.abs(got.astype(np.float64) - want.astype(np.float64)) <= ulp).all()


# (image h, w), (y0, x0, ch, cw, flip), network size: every flip, no crop, the largest crops (14 + 15 off a side), 1-pixel-wide
# crop results, down- and up-sampling, a crop that is a single pixel, gray images
TRAIN_CASES = [
    ((300, 400), (13, 12, 280, 373, 1), (224, 224), False),
    ((300, 400), (8, 6, 284, 379, 2), (224, 224), False),
    ((300, 400), (0, 0, 300, 400, 0), (224, 224), False),
    ((224, 224), (0, 0, 224, 224, 0), (224, 224), False),
    ((180, 520), (14, 14, 151, 491, 1), (224, 224), False),
    ((520, 180), (14, 14, 491, 151, 2), (224, 224), False),
    ((100, 80), (3, 7, 90, 60, 1), (224, 224), False),
    ((40, 300), (10, 5, 1, 280, 0), (224, 224), False),
    ((300, 40), (5, 10, 280, 1, 1), (224, 224), False),
    ((35, 35), (14, 14, 1, 1, 2), (64, 96), False),
    ((333, 211), (2, 9, 320, 190, 2), (96, 160), True),
    ((250, 250), (1, 1, 240, 240, 1), (224, 224), True),
]


@pytest.mark.parametrize("src,params,size,gray", TRAIN_CASES)
def test_train_sample_matches_sal_data_within_one_ulp(src, params, size, gray):
    img, mask = _sample(*src, seed=src[0] * 5 + src[1] + params[4], gray=gray)
    x, t = E.train_sample(img, mask, params, size, MEAN, STD)
    # the kernel takes mean / std as float32 and widens them to float64
    m, s = np.asarray(MEAN, np.float32).astype(np.float64), np.asarray(STD, np.float32).astype(np.float64)
    want_x, want_t = SD.sal_item(img, mask, size, params, mean=m, std=s)
    assert x.shape == (3, *size) and t.shape == (1, *size)
    assert _within_one_ulp(x, want_x)
    assert _within_one_ulp(t, want_t)


def test_uncropped_network_size_sample_is_exact():
    img, mask = _sample(224, 224, 5)
    x, t = E.train_sample(img, mask, (0, 0, 224, 224, 0), (224, 224), MEAN, STD)
    m, s = np.asarray(MEAN, np.float32).astype(np.float64), np.asarray(STD, np.float32).astype(np.float64)
    assert np.array_equal(x, np.transpose((img / 255.0 - m) / s, (2, 0, 1)).astype(np.float32))
    assert np.array_equal(t[0], (mask / 255.0).astype(np.float32))


def test_flip_of_a_flipped_image_is_the_plain_crop():
    img, mask = _sample(120, 90, 9)
    y0, x0, ch, cw = 4, 7, 100, 70
    for flip, flipped in ((1, lambda a: a[:, ::-1]), (2, lambda a: a[::-1])):
        pre = np.zeros_like(img)
        pre[y0:y0 + ch, x0:x0 + cw] = flipped(img[y0:y0 + ch, x0:x0 + cw])
        prem = np.zeros_like(mask)
        prem[y0:y0 + ch, x0:x0 + cw] = flipped(mask[y0:y0 + ch, x0:x0 + cw])
        a = E.train_sample(pre, prem, (y0, x0, ch, cw, flip), (224, 224), MEAN, STD)
        b = E.train_sample(img, mask, (y0, x0, ch, cw, 0), (224, 224), MEAN, STD)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


# GT sizes (h, w) against a 224 x 224 map: down, up, identity, one-pixel / one-sample axes, odd ratios
MAE_SHAPES = [(300, 400), (224, 224), (100, 80), (1, 1), (1, 333), (333, 1), (17, 1000), (520, 181)]


@pytest.mark.parametrize("shape", MAE_SHAPES)
def test_val_mae_matches_the_torch_loop(shape):
    rng = np.random.default_rng(shape[0] * 31 + shape[1])
    z = (rng.standard_normal((1, 1, 224, 224)) * 4).astype(np.float32)
    gt = rng.integers(0, 256, size=shape, dtype=np.uint8)
    got = E.val_mae(z[0, 0], gt)
    zt = torch.from_numpy(z)
    want = SD.val_mae_loop(zt, [gt])[0]
    slack = SD.val_mae_slack(zt, [gt])[0]
    assert abs(got - want) <= 1e-6 * abs(want) + slack, (got, want, slack)


def test_val_mae_is_zero_where_every_pixel_truncates_to_its_gt():
    # at identity size, sigmoids half-way between a GT level and the next one truncate to that level
    gt = np.random.default_rng(3).integers(0, 255, size=(224, 224), dtype=np.uint8)   # s < 1
    s = (gt.astype(np.float64) + 0.5) / 255.0
    z = np.log(s / (1 - s)).astype(np.float32)
    assert E.val_mae(z, gt) == 0.0
