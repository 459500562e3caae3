"""Test infrastructure: the reference's training data and validation MAE, restated on the host.

`sal_item` is SalData.__getitem__ (CSNet_training/utils/prepare_data.py:109-139) for decoded uint8 arrays: img_as_float, the
Augment crop and flip, skimage's resize (tests/sk_resize.py) of the image and, in train mode, of the GT, normalisation.  `val_mae_loop`
is the per-image loop of train.py:262-279 in torch."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from tests.sk_resize import IMAGENET_MEAN, IMAGENET_STD, resize


def sal_item(img: np.ndarray, gt: np.ndarray, size, params=None, mode="train", mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """uint8 img [h, w, 3] or [h, w], uint8 gt [h, w]; params (y0, x0, ch, cw, flip) or None for no augmentation.  Returns the float64
    (img [3, H, W], gt [1, H, W]) of the reference, before train.py's .float(); in val mode gt stays at (h, w).  img_as_float multiplies
    by 1 / 255 where this divides by 255: the two differ by at most a float64 ulp, far below the fp32 rounding that follows."""
    img = img.astype(np.float64) / 255.0
    gt = gt.astype(np.float64) / 255.0
    if img.ndim == 2:
        img = np.repeat(img[:, :, np.newaxis], 3, 2)
    if params is not None and mode == "train":
        y0, x0, ch, cw, flip = params
        img, gt = img[y0:y0 + ch, x0:x0 + cw], gt[y0:y0 + ch, x0:x0 + cw]
        if flip == 1:
            img, gt = np.fliplr(img), np.fliplr(gt)
        elif flip == 2:
            img, gt = np.flipud(img), np.flipud(gt)
    img = resize(img, size)
    if mode == "train":
        gt = resize(gt, size)
    img = (img - np.asarray(mean, np.float64)) / np.asarray(std, np.float64)
    return np.transpose(img, (2, 0, 1)), gt[np.newaxis]


def val_mae_loop(logits: torch.Tensor, gts) -> list:
    """train.py:262-279 for one batch: logits [N,1,H,W] (on the device the loop runs on), gts uint8 [h, w] each.  Returns each image's
    MAE as the float the reference's `mae.item()` gives."""
    out = []
    s = torch.sigmoid(logits)
    for i, g in enumerate(gts):
        h, w = g.shape
        r = (F.interpolate(s[i].unsqueeze(dim=0), size=(h, w), mode="bilinear") * 255.0).int().float() / 255.0
        t = torch.from_numpy(g.astype(np.float64) / 255.0)[None].float().to(logits.device).unsqueeze(dim=0)
        out.append(F.l1_loss(r, t, reduction="mean").item())
    return out


def val_mae_slack(logits: torch.Tensor, gts, window=1e-4) -> list:
    """Per image, 1 / (255 h w) for each pixel whose resized value * 255 in val_mae_loop lies within `window` of an integer: there
    another fp32 evaluation of the same expression may truncate to the neighbouring level."""
    out = []
    s = torch.sigmoid(logits)
    for i, g in enumerate(gts):
        h, w = g.shape
        v = (F.interpolate(s[i].unsqueeze(dim=0), size=(h, w), mode="bilinear") * 255.0).double()
        near = int(((v - v.round()).abs() < window).sum().item())
        out.append(near / (255.0 * h * w))
    return out
