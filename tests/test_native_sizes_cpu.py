"""Native-size evaluation without a GPU: the padded-size rule of CSNet/test.py (TEST.IMAGE_H = 0), how images are cut into network
runs, and the counting of csnet_salmetric_images_u8 (host emulation) reduced by SalMetric against oracle/salmetric.py."""
import math

import numpy as np
import pytest

from oracle import salmetric as O
from sod100k_b200 import engine
from sod100k_b200.salmetric import SalMetric, image_scores
from tests.emu import salmetric as E

SHAPES = [(16, 16), (224, 224), (400, 304), (17, 16), (16, 17), (15, 16), (31, 33), (1, 1), (1, 37), (53, 1), (17, 1000),
          (300, 400), (400, 300), (181, 517), (48, 47), (49, 64)]


def _test_py_input_size(h, w):
    """CSNet/test.py:75-84 with TEST.IMAGE_H = TEST.IMAGE_W = 0, on the shape of the image array."""
    if h % 16 != 0 or w % 16 != 0:
        return (math.ceil(h / 16) * 16, math.ceil(w / 16) * 16)
    return (h, w)


@pytest.mark.parametrize("h,w", SHAPES)
def test_padded_size_is_test_py_rule(h, w):
    assert engine.native_size(h, w) == _test_py_input_size(h, w)


def test_runs_group_by_padded_size_in_ascending_order():
    sizes = [(300, 400), (17, 1000), (400, 300), (299, 400), (16, 16), (289, 400), (1, 1), (300, 400)]
    order, runs = engine.image_runs(sizes, None, 2)
    assert sorted(order) == list(range(len(sizes)))
    keys = [(H, W) for _, _, H, W in runs]
    assert keys == sorted(keys)
    assert len({k for k in keys}) == len(set(engine.native_size(*s) for s in sizes))
    for a, b, H, W in runs:
        assert 1 <= b - a <= 2
        assert all(engine.native_size(*sizes[i]) == (H, W) for i in order[a:b])
    # the first run of a size is its largest: one plan per size, created once
    for (H, W) in set(keys):
        n = [b - a for a, b, h, w in runs if (h, w) == (H, W)]
        assert n[0] == max(n)
    # a fixed size keeps the input order and, without a batch limit, one run
    assert engine.image_runs(sizes, (224, 224), None) == (list(range(len(sizes))), [(0, len(sizes), 224, 224)])
    with pytest.raises(ValueError):
        engine.image_runs(sizes, None, 0)


def _case(seed, H, W, h, w):
    rng = np.random.default_rng(seed)
    z = (rng.standard_normal((H, W)) * 3).astype(np.float32)
    z.reshape(-1)[:3] = [-100.0, 100.0, 0.0]                 # saturated ends of the sigmoid and the middle bin
    gt = ((rng.random((h, w)) > 0.6) * 255).astype(np.uint8)
    gt.reshape(-1)[:3] = [128, 129, 127][:gt.size]            # around the > 128 rule
    return z, gt


def test_emulated_counting_reproduces_the_oracle_metric():
    shapes = [((304, 400), (300, 397)), ((224, 224), (224, 224)), ((16, 16), (1, 1)), ((16, 48), (7, 33)), ((64, 16), (53, 1)),
              ((400, 304), (400, 304))]
    counts, maps, gts = [], [], []
    for k, ((H, W), (h, w)) in enumerate(shapes):
        z, gt = _case(100 + k, H, W, h, w)
        if k == 1:
            gt[:] = 0                                          # an image without foreground
        ha, hp, ad, q = E.salmetric_image(z, gt)
        assert ha.sum() == h * w and hp.sum() == int((gt > 128).sum())
        assert np.array_equal(ha, np.bincount(q.reshape(-1), minlength=256))
        assert ad == int(np.abs(q.astype(np.int64) - gt).sum())
        p_ref, r_ref = O.precision_recall(q, gt)
        p, r, _ = image_scores(ha[None], hp[None], np.array([ad]), h * w)
        assert np.array_equal(p[0], p_ref) and np.array_equal(r[0], r_ref)
        counts.append((ha, hp, ad, h * w))
        maps.append(q)
        gts.append(gt)
    m = SalMetric()
    m.add_images(*(np.array(c) for c in zip(*counts)))
    got, ref = m.compute(), O.evaluate(maps, gts)
    for key in ("max_f", "mean_f", "precision", "recall", "mean_precision", "mean_recall", "argmax"):
        assert got[key] == ref[key], key
    # the counts give each image's MAE from an exact integer sum; the oracle adds float32 terms pixel by pixel
    assert got["mae"] == pytest.approx(ref["mae"], rel=1e-6)


def test_add_images_sums_in_image_order_like_the_oracle():
    """Many images: add_images' float64 running sums give oracle.evaluate's scores bit for bit."""
    rng = np.random.default_rng(7)
    maps, gts = [], []
    for _ in range(300):
        h, w = (int(v) for v in rng.integers(1, 40, size=2))
        maps.append(np.minimum(rng.exponential(rng.uniform(5, 120), (h, w)), 255).astype(np.uint8))
        gts.append(((rng.random((h, w)) > rng.uniform(0.2, 1.0)) * 255).astype(np.uint8))
    ha = np.array([np.bincount(q.reshape(-1), minlength=256) for q in maps])
    hp = np.array([np.bincount(q[g > 128], minlength=256) for q, g in zip(maps, gts)])
    ad = np.array([np.abs(q.astype(np.int64) - g).sum() for q, g in zip(maps, gts)])
    m = SalMetric()
    m.add_images(ha, hp, ad, np.array([q.size for q in maps]))
    got, ref = m.compute(), O.evaluate(maps, gts)
    for key in ("max_f", "mean_f", "precision", "recall", "mean_precision", "mean_recall", "argmax"):
        assert got[key] == ref[key], key
    assert got["mae"] == pytest.approx(ref["mae"], rel=1e-6)
