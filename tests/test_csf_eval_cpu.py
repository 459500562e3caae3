"""CSF+Res2Net test-set evaluation without a GPU: the per-pixel input and map functions of the device path (compiled for the CPU from
image_io.cuh) and the numpy restatement the GPU tests use, both against the unmodified reference's load_image_test and cv2.imwrite
bytes (tests/golden/csf_eval.npz); and the exact-size grouping of engine.image_runs."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from sod100k_b200 import engine
from tests import csf_ref, fixtures

EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
MEAN, STD = np.array(csf_ref.MEAN, np.float64), np.array(csf_ref.STD, np.float64)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu") / "libcsf_io_emu.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-o", out, os.path.join(EMU, "csf_io_emu.cpp")], check=True)
    lib = C.CDLL(out)
    lib.csnet_emu_csf_input.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.csnet_emu_csf_out_byte.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(fixtures.GOLDEN, "csf_eval.npz"))
    return z, json.loads(str(z["__meta__"]))


def _emu_input(lib, img):
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    out = np.empty((3, h, w), np.float32)
    lib.csnet_emu_csf_input(img.ctypes.data, h, w, MEAN.ctypes.data, STD.ctypes.data, out.ctypes.data)
    return out


def _emu_bytes(lib, pred):
    s = np.ascontiguousarray(pred, np.float32)
    q = np.empty(s.shape, np.uint8)
    lib.csnet_emu_csf_out_byte(s.ctypes.data, s.size, q.ctypes.data)
    return q


TAGS = ["1x1", "3x5", "37x53", "75x100", "gray"]


@pytest.mark.parametrize("tag", TAGS)
def test_input_matches_load_image_test_bit_for_bit(lib, golden, tag):
    z, _ = golden
    img, ref = z[f"{tag}/image"], z[f"{tag}/x"]
    assert ref.dtype == np.float32
    assert np.array_equal(_emu_input(lib, img).view(np.uint32), ref.view(np.uint32))
    assert np.array_equal(csf_ref.load_image_test(img).view(np.uint32), ref.view(np.uint32))
    if tag == "gray":                                  # cv2.IMREAD_COLOR replicates a gray PNG to three equal channels
        assert np.array_equal(np.repeat(z["gray/gray"][:, :, None], 3, axis=2), img)


def test_input_single_rounding_differs():
    """The three-rounding rule is not CSNet's single rounding: the two differ at many (value, channel) pairs, so matching the golden
    above pins the rule."""
    u = np.arange(256, dtype=np.uint8)
    three = np.stack([csf_ref.load_image_test(np.repeat(u[None, :, None], 3, axis=2))[c, 0] for c in range(3)])
    one = np.stack([((u.astype(np.float64) / 255 - MEAN[c]) / STD[c]).astype(np.float32) for c in range(3)])
    assert (three != one).sum() > 300


@pytest.mark.parametrize("name", ["ties", "edges", "random"])
def test_map_bytes_match_cv2_imwrite(lib, golden, name):
    z, meta = golden
    pred, png = z[f"maps/{name}/pred"], z[f"maps/{name}/png"]
    assert pred.dtype == np.float32 and png.dtype == np.uint8 and png.shape == pred.shape
    assert np.array_equal(_emu_bytes(lib, pred), png)
    assert np.array_equal(csf_ref.map_bytes(pred), png)
    if name == "ties":                                 # every k + 0.5 for k in [0, 255): half to even, not truncation or half up
        assert meta["ties"] == 255 and pred.size == 255
        assert np.array_equal(np.float32(255) * pred[0], np.arange(255, dtype=np.float32) + np.float32(0.5))
        assert np.array_equal(png[0], 2 * ((np.arange(255) + 1) // 2))


def test_map_bytes_saturate(lib):
    s = np.array([-1.0, -0.0, 1.0, 1.5, np.inf, -np.inf, np.nan], np.float32)
    assert _emu_bytes(lib, s).tolist() == [0, 0, 255, 255, 255, 0, 0]


def test_exact_size_runs_keep_input_order_and_cap_the_batch():
    sizes = [(300, 400), (75, 100), (300, 400), (100, 75), (75, 100), (300, 400), (75, 100), (300, 400), (37, 53)]
    order, runs = engine.image_runs(sizes, None, 2, key=engine.exact_size)
    assert sorted(order) == list(range(len(sizes)))
    keys = [(H, W) for _, _, H, W in runs]
    assert keys == sorted(keys)
    for a, b, H, W in runs:
        assert 1 <= b - a <= 2
        assert all(sizes[i] == (H, W) for i in order[a:b])
    for s in set(sizes):                               # input order within a size
        idx = [i for i in order if sizes[i] == s]
        assert idx == sorted(idx)
    assert engine.image_runs(sizes, None, None, key=engine.exact_size)[1] == [(0, 1, 37, 53), (1, 4, 75, 100), (4, 5, 100, 75),
                                                                             (5, 9, 300, 400)]
    # 75 x 100 and 100 x 75 pad to different sizes, 37 x 53 and 48 x 64 to the same: exact grouping keeps them apart
    two = [(37, 53), (48, 64)]
    assert len(engine.image_runs(two, None, None)[1]) == 1
    assert len(engine.image_runs(two, None, None, key=engine.exact_size)[1]) == 2


def test_default_key_gives_todays_runs():
    sizes = [(300, 400), (17, 1000), (400, 300), (299, 400), (16, 16), (289, 400), (1, 1), (300, 400)]
    for size, batch in ((None, 2), (None, None), ((224, 224), 3), ((224, 224), None)):
        assert engine.image_runs(sizes, size, batch) == engine.image_runs(sizes, size, batch, key=engine.native_size)
    assert engine.image_runs(sizes, None, 2) == ([4, 6, 1, 0, 3, 5, 7, 2], [(0, 2, 16, 16), (2, 3, 32, 1008), (3, 5, 304, 400),
                                                                         (5, 7, 304, 400), (7, 8, 400, 304)])
