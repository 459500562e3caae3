"""Record the reference's augmentation draws: Augment(15, 15, p_flip=0.5).get_params of the UNMODIFIED
CSNet_training/utils/prepare_data.py for several seeds and image sizes, too-small images included.

    python tests/golden/make_augment_golden.py    # writes tests/golden/augment.json

Needs /root/reference (absent on the GPU box — the fixture is what travels).  skimage and torchvision are not dependencies of this
project and get_params calls neither, so the module is imported with empty stand-ins for them (a harness-side shim, like the
`collections.Iterable` one of make_golden.py).  Each case seeds the module-level `random` the reference draws from and records
successive draws, a draw that raises ValueError included, so the state carried past an error is checked too."""
from __future__ import annotations

import importlib.util
import json
import os
import random
import sys
import types

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
SRC = "/root/reference/CSNet_training/utils/prepare_data.py"

# (seed, h, w, draws): ordinary sizes, the smallest sides that always fit (30), sides that sometimes do not, 1-pixel images
CASES = [(0, 300, 400, 40), (1, 224, 224, 40), (2, 520, 180, 40), (3, 30, 30, 40), (4, 29, 400, 40), (5, 400, 20, 40),
         (6, 16, 16, 40), (7, 1, 1, 10), (8, 2, 300, 20), (2024, 375, 500, 40)]


def load_reference():
    for name in ("skimage", "skimage.io", "skimage.transform", "torchvision", "torchvision.transforms"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["skimage"].io = sys.modules["skimage.io"]
    sys.modules["skimage.transform"].resize = None
    sys.modules["torchvision"].transforms = sys.modules["torchvision.transforms"]
    spec = importlib.util.spec_from_file_location("prepare_data", SRC)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    ref = load_reference()
    aug = ref.Augment(size_h=15, size_w=15, p_flip=0.5)
    out = []
    for seed, h, w, n in CASES:
        random.seed(seed)
        draws = []
        for _ in range(n):
            try:
                row1, row2, col1, col2, flip, padding = aug.get_params(_Shape(h, w))
                assert padding is None
                draws.append([row1, row2, col1, col2, flip])
            except ValueError as e:
                draws.append(str(e))
        out.append({"seed": seed, "h": h, "w": w, "draws": draws})
    with open(os.path.join(HERE, "augment.json"), "w") as f:
        json.dump({"source": "CSNet_training/utils/prepare_data.py:38-57 Augment(15, 15, p_flip=0.5).get_params", "cases": out}, f)
        f.write("\n")


class _Shape:
    """get_params reads only img.shape[:2]."""

    def __init__(self, h, w):
        self.shape = (h, w, 3)


if __name__ == "__main__":
    main()
