"""Generate tests/golden/csf_eval.npz: CSF+Res2Net's test-path input and map bytes from the UNMODIFIED reference code and OpenCV.

    python tests/golden/make_csf_eval_golden.py

Needs the reference checkout and cv2 (absent on the GPU box — the fixture is what travels).  Only dataset/dataset.py is imported from
the reference (solver.py imports scipy.misc, which recent scipy no longer has).

  input  seeded RGB images written as PNG (cv2 stores BGR, so the RGB array is flipped on the way out) at 1x1, 3x5, 37x53 and
         75x100, plus a gray image written as a 1-channel PNG, which cv2.imread(IMREAD_COLOR) reads back as 3 equal channels.
         dataset.load_image_test runs on each file.  Stored: `{tag}/image`, the decoded RGB uint8 [h, w, 3] the reference normalises,
         and `{tag}/x`, its fp32 [3, h, w]; for the gray case also `gray/gray`, the 1-channel uint8 [h, w] written to disk.
  maps   solver.py:73-75 restated on seeded fp32 maps pred: multi_fuse = 255 * pred, cv2.imwrite to PNG, read back unchanged.
         `ties` holds values for which 255 * pred is exactly a half-integer in fp32, found by search around (k + 0.5) / 255 for every
         k, `edges` values near 0 and 1, `random` uniform values.  Stored: `maps/{name}/pred` and `maps/{name}/png`.
"""
from __future__ import annotations

import importlib.util
import json
import os
import sys
import tempfile

import cv2
import numpy as np

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("CSF_REFERENCE", os.path.join(os.path.dirname(ROOT), "reference", "CSF+Res2Net"))

SEED = 31
SIZES = {"1x1": (1, 1), "3x5": (3, 5), "37x53": (37, 53), "75x100": (75, 100)}
GRAY = (20, 30)


def reference_dataset():
    spec = importlib.util.spec_from_file_location("csf_reference_dataset", os.path.join(REF, "dataset", "dataset.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def tie_values() -> np.ndarray:
    """fp32 values s with np.float32(255) * s exactly k + 0.5, for every k in [0, 255) where one exists near (k + 0.5) / 255."""
    out = []
    for k in range(255):
        s0 = np.float32((k + 0.5) / 255.0)
        for d in range(-8, 9):
            s = np.float32(s0 + d * np.spacing(s0))
            if np.float32(255) * s == np.float32(k + 0.5):
                out.append(s)
                break
    return np.array(out, np.float32)


def write_map(path: str, pred: np.ndarray) -> np.ndarray:
    multi_fuse = 255 * pred                      # solver.py:74, an fp32 array
    assert multi_fuse.dtype == np.float32
    assert cv2.imwrite(path, multi_fuse)         # solver.py:75
    return cv2.imread(path, cv2.IMREAD_UNCHANGED)


def main():
    ds = reference_dataset()
    rng = np.random.default_rng(SEED)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for tag, (h, w) in SIZES.items():
            rgb = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
            path = os.path.join(tmp, f"{tag}.png")
            assert cv2.imwrite(path, rgb[:, :, ::-1])
            x, size = ds.load_image_test(path)
            assert size == (h, w) and x.dtype == np.float32
            out[f"{tag}/image"], out[f"{tag}/x"] = rgb, x
        gray = rng.integers(0, 256, size=GRAY, dtype=np.uint8)
        path = os.path.join(tmp, "gray.png")
        assert cv2.imwrite(path, gray)
        x, _ = ds.load_image_test(path)
        out["gray/gray"], out["gray/image"], out["gray/x"] = gray, np.repeat(gray[:, :, None], 3, axis=2), x

        ties = tie_values()
        eps = np.float32(2.0 ** -24)
        edges = np.array([0.0, eps, 1e-30, 1e-3, 1.0 / 510, np.nextafter(np.float32(1.0 / 510), 0), 0.5, 1 - 1.0 / 510,
                          1 - eps, np.nextafter(np.float32(1), 0), 1.0], np.float32)
        maps = {"ties": ties.reshape(1, -1), "edges": edges.reshape(1, -1),
                "random": rng.random((37, 53), dtype=np.float32)}
        for name, pred in maps.items():
            out[f"maps/{name}/pred"] = pred
            out[f"maps/{name}/png"] = write_map(os.path.join(tmp, f"map_{name}.png"), pred)
    meta = dict(seed=SEED, sizes=SIZES, gray=GRAY, ties=int(ties.size), numpy=np.__version__, cv2=cv2.__version__)
    np.savez_compressed(os.path.join(HERE, "csf_eval.npz"), __meta__=np.array(json.dumps(meta)), **out)
    print("wrote csf_eval.npz", meta)


if __name__ == "__main__":
    main()
