"""Test infrastructure: CSNet/test.py's per-image loop with TEST.IMAGE_H = 0 (every image at its own size), restated on the host
with the skimage resizes of tests/sk_resize.py."""
from __future__ import annotations

import math

import numpy as np
import torch

from tests.sk_resize import IMAGENET_MEAN, IMAGENET_STD, resize


def padded_size(h: int, w: int):
    """test.py:80-84: an image whose h or w is not a multiple of 16 goes in at (ceil(h / 16) * 16, ceil(w / 16) * 16)."""
    if h % 16 != 0 or w % 16 != 0:
        return (math.ceil(h / 16) * 16, math.ceil(w / 16) * 16)
    return (h, w)


def test_py_native_pipeline(forward, imgs, mean=IMAGENET_MEAN, std=IMAGENET_STD, scaled=False):
    """CSNet/test.py:71-98 with TEST.IMAGE_H = 0 for a list of uint8 [h, w, 3] images: img_as_float, resized to padded_size only when
    h or w is not a multiple of 16, normalised, the network (`forward`: float32 [N,3,H,W] CPU tensor -> logits [N,1,H,W]; images of
    one padded size go in one call, images are independent), sigmoid, resized to (h, w), * 255, astype(uint8).  Returns the uint8 maps
    in input order; scaled=True returns the float32 maps * 255 before the cast instead."""
    groups = {}
    for i, im in enumerate(imgs):
        groups.setdefault(padded_size(*im.shape[:2]), []).append(i)
    maps = [None] * len(imgs)
    for size, idx in groups.items():
        xs = []
        for i in idx:
            x = imgs[i].astype(np.float64) / 255.0
            if x.shape[:2] != size:
                x = resize(x, size)
            xs.append(np.transpose((x - np.asarray(mean)) / np.asarray(std), (2, 0, 1)))
        with torch.no_grad():
            pred = torch.sigmoid(forward(torch.FloatTensor(np.stack(xs))))[:, 0].cpu().numpy()
        for i, p in zip(idx, pred):
            maps[i] = resize(p, imgs[i].shape[:2]) * 255
    return maps if scaled else [v.astype(np.uint8) for v in maps]


test_py_native_pipeline.__test__ = False
