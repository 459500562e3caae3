"""Test infrastructure: the reference's skimage resizes and its per-image test loop, restated on the host.

CSNet/test.py:71-98 calls skimage.transform.resize(img, shape, mode='reflect', anti_aliasing=False).  For skimage >= 0.19 and
float input (order 1) that is exactly scipy.ndimage.zoom(img, out / in per axis, order=1, mode='mirror', grid_mode=True), the
channel axis at factor 1 (skimage itself is not a dependency of this project; scipy is)."""
from __future__ import annotations

import numpy as np
import torch
from scipy import ndimage

IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)          # CSNet/test.py:68-69


def resize(img: np.ndarray, shape) -> np.ndarray:
    """skimage resize(img, shape, mode='reflect', anti_aliasing=False) of a float image [h, w] or [h, w, C]; float32 stays float32."""
    img = np.asarray(img)
    zoom = [o / i for o, i in zip(shape, img.shape[:2])] + [1.0] * (img.ndim - 2)
    return ndimage.zoom(img, zoom, order=1, mode="mirror", grid_mode=True)


def test_py_pipeline(forward, imgs, size, mean=IMAGENET_MEAN, std=IMAGENET_STD, scaled=False):
    """CSNet/test.py:71-98 on the host for a list of uint8 [h, w, 3] images: img_as_float, resize to `size`, normalise, the network
    (`forward`: float32 [N,3,H,W] CPU tensor -> logits [N,1,H,W], one batched call; images are independent), sigmoid, resize back
    to each image's (h, w), * 255, astype(uint8).  Returns the uint8 maps in input order; scaled=True returns the float32 maps
    * 255 before the cast instead."""
    x = np.stack([np.transpose((resize(im.astype(np.float64) / 255.0, size) - np.asarray(mean)) / np.asarray(std), (2, 0, 1))
                  for im in imgs])
    with torch.no_grad():
        pred = torch.sigmoid(forward(torch.FloatTensor(x)))[:, 0].cpu().numpy()
    maps = [resize(p, im.shape[:2]) * 255 for p, im in zip(pred, imgs)]
    return maps if scaled else [v.astype(np.uint8) for v in maps]


test_py_pipeline.__test__ = False
