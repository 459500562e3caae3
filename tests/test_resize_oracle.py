"""The per-pixel resize arithmetic of sod100k_b200/csrc/image_io.cuh, compiled for the host (tests/emu), against
scipy.ndimage.zoom as skimage >= 0.19 calls it (tests/sk_resize.py).  No GPU needed."""
import numpy as np
import pytest

from tests import sk_resize as SK
from tests.emu import image_io as E

MEAN, STD = SK.IMAGENET_MEAN, SK.IMAGENET_STD
# image (h, w) -> network (H, W): down, up, identity, one-pixel and one-sample axes, extreme aspect ratios, odd sizes
IN_CASES = [((500, 375), (224, 224)), ((100, 80), (224, 224)), ((224, 224), (224, 224)), ((64, 96), (64, 96)), ((1, 1), (224, 224)),
            ((1, 37), (224, 224)), ((53, 1), (224, 224)), ((17, 1000), (224, 224)), ((181, 517), (224, 224)), ((333, 211), (96, 160))]
# network (H, W) -> map (h, w)
OUT_CASES = [((224, 224), (500, 375)), ((224, 224), (100, 80)), ((224, 224), (224, 224)), ((224, 224), (1, 1)), ((224, 224), (1, 333)),
             ((224, 224), (333, 1)), ((224, 224), (17, 1000)), ((224, 224), (81, 7)), ((96, 160), (181, 517)), ((96, 160), (96, 160))]


def _image(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, size=(h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("src,size", IN_CASES)
def test_resize_in_matches_zoom_within_one_ulp(src, size):
    img = _image(*src, seed=src[0] * 7 + src[1])
    got = E.resize_in(img, size, MEAN, STD)
    # the kernel takes mean / std as float32 and widens them to float64
    m, s = np.asarray(MEAN, np.float32).astype(np.float64), np.asarray(STD, np.float32).astype(np.float64)
    want = np.transpose((SK.resize(img.astype(np.float64) / 255.0, size) - m) / s, (2, 0, 1)).astype(np.float32)
    assert got.shape == want.shape == (3, *size)
    ulp = np.spacing(np.maximum(np.abs(got), np.abs(want)))
    assert (np.abs(got.astype(np.float64) - want) <= ulp).all()
    if src == size:                                          # identity: exactly csnet_plan_run_host_u8's pre_u8_kernel
        exact = np.transpose((img.astype(np.float64) / 255.0 - m) / s, (2, 0, 1)).astype(np.float32)
        assert np.array_equal(got, exact)


@pytest.mark.parametrize("size,dst", OUT_CASES)
def test_resize_out_matches_zoom(size, dst):
    z = (np.random.default_rng(size[0] + dst[0] * 13 + dst[1]).standard_normal(size) * 4).astype(np.float32)
    got = E.resize_out(z, dst)
    s = E.sigmoid(z)
    v = SK.resize(s, dst)                                    # zoom of a float32 map: float32
    assert v.dtype == np.float32
    want = (v * 255).astype(np.uint8)
    assert got.shape == want.shape == dst
    d = np.abs(got.astype(np.int32) - want.astype(np.int32))
    scaled = v.astype(np.float64) * 255.0
    near = np.abs(scaled - np.round(scaled)) < 1e-5           # fp32 rounding of the interpolated value may cross an integer there
    assert d[~near].max(initial=0) == 0 and d.max() <= 1
    if size == dst:                                          # identity: exactly post_u8_kernel's (uint8)(sigmoid * 255.f)
        assert np.array_equal(got, (s * np.float32(255)).astype(np.uint8))
