"""TEST INFRASTRUCTURE — numpy restatement of CSF+Res2Net's test loop (CSF+Res2Net/solver.py:62-78 with dataset.py:83-96).

load_image_test and map_bytes follow the reference line by line on an already decoded RGB image and an fp32 sigmoid map; the
golden tests pin them to the unmodified reference and cv2 (tests/golden/csf_eval.npz), and the GPU tests use solver_test as the
reference loop around any network call."""
from __future__ import annotations

import numpy as np
import torch

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def load_image_test(rgb: np.ndarray) -> np.ndarray:
    """dataset.py:87-96 after cv2.imread + cvtColor: uint8 RGB [h, w, 3] -> fp32 [3, h, w]."""
    in_ = np.array(rgb, dtype=np.float32)
    in_ = in_ / 255
    in_ -= np.array(MEAN)
    in_ /= np.array(STD)
    return in_.transpose((2, 0, 1))


def map_bytes(pred: np.ndarray) -> np.ndarray:
    """solver.py:74-75: multi_fuse = 255 * pred (fp32), which cv2.imwrite converts to uint8 by rounding half to even and saturating."""
    multi_fuse = 255 * np.asarray(pred, np.float32)
    return np.clip(np.rint(multi_fuse), 0, 255).astype(np.uint8)


def solver_test(net, images):
    """solver.test's loop around `net` (a callable on a CUDA fp32 [1, 3, h, w] tensor): one image at a time, sigmoid on the device,
    the map to the host, 255 *, and the bytes cv2.imwrite would write."""
    maps = []
    for im in images:
        rgb = np.repeat(im[:, :, None], 3, axis=2) if im.ndim == 2 else im
        x = torch.from_numpy(np.ascontiguousarray(load_image_test(rgb))[None]).cuda()
        with torch.no_grad():
            preds = net(x)
        pred = np.squeeze(torch.sigmoid(preds).cpu().data.numpy())
        maps.append(map_bytes(pred).reshape(rgb.shape[:2]))
    return maps
