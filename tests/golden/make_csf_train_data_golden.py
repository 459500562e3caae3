"""Generate tests/golden/csf_train_data.npz: CSF+Res2Net's training samples from the UNMODIFIED reference ImageDataTrain.

    python tests/golden/make_csf_train_data_golden.py

Needs the reference checkout, cv2, PIL and torchvision (absent on the GPU box — the fixture is what travels).  Only dataset/dataset.py
is imported from the reference.

  files    seeded RGB images written as PNG (cv2 stores BGR, so the RGB array is flipped on the way out) at 1x1, 3x5, 37x53 and
           75x100, plus a gray image written as a 1-channel PNG, which cv2.imread reads back as 3 equal channels.  Each image has two
           GTs of its size: an 'L' PNG and an 'RGB' PNG whose three channels differ (load_sal_label takes channel 0).
  samples  ImageDataTrain(root, list).__getitem__(item) under random.seed(s), for seeds that give both flips of every (image, GT).
           The `random` module the reference calls is wrapped so that every randint draw is recorded.  Stored per tag, GT kind
           (`L`, `rgb`) and flip f: `{tag}/{kind}/flip{f}/x` (sal_image, fp32 [3, h, w]), `.../t` (sal_label, fp32 [1, h, w]) and
           `.../seed`.  Per tag: `{tag}/image`, the decoded RGB uint8 [h, w, 3]; `{tag}/mask_L`, np.array(Image.open(gt)) of the 'L'
           GT, uint8 [h, w]; `{tag}/mask_rgb`, that of the 'RGB' GT, uint8 [h, w, 3]; for the gray case also `gray/gray`.
  draws    random.seed(DRAW_SEED), then __getitem__ over DRAW_ITEMS items in turn: `draws`, the flips drawn, in order.
"""
from __future__ import annotations

import importlib.util
import json
import os
import random
import sys
import tempfile
import types

import cv2
import numpy as np
from PIL import Image

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("CSF_REFERENCE", os.path.join(os.path.dirname(ROOT), "reference", "CSF+Res2Net"))

SEED = 47
SIZES = {"1x1": (1, 1), "3x5": (3, 5), "37x53": (37, 53), "75x100": (75, 100)}
GRAY = (20, 30)
DRAW_SEED, DRAW_ITEMS = 2024, 40


def reference_dataset():
    spec = importlib.util.spec_from_file_location("csf_reference_dataset", os.path.join(REF, "dataset", "dataset.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    ds_mod = reference_dataset()
    drawn = []

    def randint(a, b):
        v = random.randint(a, b)
        drawn.append(v)
        return v

    ds_mod.random = types.SimpleNamespace(randint=randint)          # cv_random_flip's only use of `random`
    rng = np.random.default_rng(SEED)
    out, lines, tags = {}, [], []
    with tempfile.TemporaryDirectory() as tmp:
        images = {tag: rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for tag, (h, w) in SIZES.items()}
        gray = rng.integers(0, 256, size=GRAY, dtype=np.uint8)
        for tag, rgb in images.items():
            assert cv2.imwrite(os.path.join(tmp, f"{tag}.png"), rgb[:, :, ::-1])
            out[f"{tag}/image"] = rgb
        assert cv2.imwrite(os.path.join(tmp, "gray.png"), gray)
        out["gray/gray"], out["gray/image"] = gray, np.repeat(gray[:, :, None], 3, axis=2)
        for tag in list(SIZES) + ["gray"]:
            h, w = out[f"{tag}/image"].shape[:2]
            m_l = rng.integers(0, 256, size=(h, w), dtype=np.uint8)
            m_rgb = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
            Image.fromarray(m_l, "L").save(os.path.join(tmp, f"{tag}_L.png"))
            Image.fromarray(m_rgb, "RGB").save(os.path.join(tmp, f"{tag}_rgb.png"))
            out[f"{tag}/mask_L"] = np.array(Image.open(os.path.join(tmp, f"{tag}_L.png")))
            out[f"{tag}/mask_rgb"] = np.array(Image.open(os.path.join(tmp, f"{tag}_rgb.png")))
            assert np.array_equal(out[f"{tag}/mask_L"], m_l) and np.array_equal(out[f"{tag}/mask_rgb"], m_rgb)
            for kind in ("L", "rgb"):
                lines.append(f"{tag}.png {tag}_{kind}.png")
                tags.append((tag, kind))
        with open(os.path.join(tmp, "train.lst"), "w") as f:
            f.write("\n".join(lines) + "\n")
        ds = ds_mod.ImageDataTrain(tmp, os.path.join(tmp, "train.lst"))
        for item, (tag, kind) in enumerate(tags):
            for flip in (0, 1):
                for s in range(1000):
                    drawn.clear()
                    random.seed(s)
                    sample = ds[item]
                    if drawn == [flip]:
                        break
                else:
                    raise RuntimeError("no seed gives flip", flip)
                x, t = sample["sal_image"].numpy(), sample["sal_label"].numpy()
                h, w = out[f"{tag}/image"].shape[:2]
                assert x.dtype == np.float32 and x.shape == (3, h, w) and t.dtype == np.float32 and t.shape == (1, h, w)
                key = f"{tag}/{kind}/flip{flip}"
                out[f"{key}/x"], out[f"{key}/t"], out[f"{key}/seed"] = x, t, np.int64(s)
        drawn.clear()
        random.seed(DRAW_SEED)
        for i in range(DRAW_ITEMS):
            ds[i % len(ds)]
        out["draws"] = np.array(drawn, np.int64)
        assert len(drawn) == DRAW_ITEMS
    meta = dict(seed=SEED, sizes=SIZES, gray=GRAY, draw_seed=DRAW_SEED, draw_items=DRAW_ITEMS, numpy=np.__version__,
                cv2=cv2.__version__, pillow=Image.__version__ if hasattr(Image, "__version__") else None)
    np.savez_compressed(os.path.join(HERE, "csf_train_data.npz"), __meta__=np.array(json.dumps(meta)), **out)
    print("wrote csf_train_data.npz", meta)


if __name__ == "__main__":
    main()
