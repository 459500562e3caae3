"""Training data on the device: the reference's SalData (CSNet_training/utils/prepare_data.py:91-139) and the MAE of its validation
loop (CSNet_training/train.py:250-293) for a dataset kept in GPU memory as uint8.

A `SalImages` set packs its images and masks once into two device buffers and a device geometry table.  Each step's batch is then
built by one kernel (csnet_train_batch_u8): only the crop windows and flips, drawn on the host exactly as `Augment.get_params`
draws them, cross PCIe.  The training loop of train.py becomes

    ds = SalImages(images, masks)
    rng = random.Random(seed)
    for idx in torch.randperm(len(ds)).split(batch_size):
        if len(idx) == batch_size:                                  # drop_last
            loss = trainer.step(*ds.train_batch(idx, rng))

and a test set is scored like CSNet/test.py followed by eval.py with `SalImages(images, gts).evaluate(model)`.

CSF+Res2Net trains on the same packed set: `csf_train_batch` builds ImageDataTrain's samples (no crop, no resize, a flip per item)
and trainer.CSFTrainer runs solver.train's step, gradient accumulation and Adam schedule on them.  The reference skips an image whose
label differs in size ('IMAGE ERROR'); a SalImages set refuses such a pair when it is packed.
"""
from __future__ import annotations

import random
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import runtime

IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)          # prepare_data.py:101-102
CROP = 15                   # Augment(size_h=15, size_w=15), prepare_data.py:122
P_FLIP = 0.5


def augment_params(rng: random.Random, h: int, w: int) -> Tuple[int, int, int, int, int]:
    """One draw of Augment(15, 15, p_flip=0.5).get_params (prepare_data.py:38-57) for an image of (h, w): the same rng.randrange /
    rng.random calls in the same order, so an equally seeded random.Random gives the reference's crops and flips.  Returns the crop
    window (y0, x0, ch, cw) = img[row1:row2, col1:col2] and the flip (0 none, 1 'lr', 2 'ud').  Raises the reference's ValueError
    when the image is too small for the crop (after the same four draws)."""
    row1 = rng.randrange(CROP)
    row2 = -rng.randrange(CROP) - 1
    col1 = rng.randrange(CROP)
    col2 = -rng.randrange(CROP) - 1
    if row1 - row2 >= h or col1 - col2 >= w:
        raise ValueError("Image size too small, please choose smaller crop size")
    flip = 0
    if rng.random() < P_FLIP:
        flip = 1 if rng.random() < 0.5 else 2
    return row1, col1, h + row2 - row1, w + col2 - col1, flip


def csf_flip(rng: random.Random) -> int:
    """One draw of CSF+Res2Net's cv_random_flip (dataset.py:109-114): random.randint(0, 1), 1 flipping image and label along W.  With
    num_thread = 1 the reference's DataLoader seeds its worker's `random` module with random.seed(base_seed) at every epoch, base_seed
    drawn from torch's generator; a random.Random(base_seed) per epoch drawing once per item, in loader order, replays its flips."""
    return rng.randint(0, 1)


def _u8(a, what: str) -> torch.Tensor:
    if isinstance(a, np.ndarray):
        a = torch.from_numpy(np.ascontiguousarray(a))
    if not isinstance(a, torch.Tensor) or a.dtype != torch.uint8:
        raise ValueError(f"{what}: expected a uint8 numpy array or tensor, got {getattr(a, 'dtype', type(a).__name__)}")
    return a


def _indices(indices, n: int) -> np.ndarray:
    idx = indices.cpu().numpy() if isinstance(indices, torch.Tensor) else np.asarray(indices)
    if idx.ndim != 1 or idx.size == 0 or not np.issubdtype(idx.dtype, np.integer):
        raise ValueError(f"indices: expected a non-empty 1-D integer sequence, got {idx.dtype} {idx.shape}")
    if idx.min() < 0 or idx.max() >= n:
        raise ValueError(f"indices: outside [0, {n})")
    if idx.size > 65535:
        raise ValueError("indices: at most 65535 samples a batch")
    return idx.astype(np.int64)


class SalImages:
    """A saliency training / validation set resident on one GPU as uint8.

    images: uint8 [h, w, 3] (or gray [h, w], repeated to 3 channels as prepare_data.py:118-120 does); masks: uint8 [h, w] of the same
    size, single-channel as io.imread(as_gray=True) returns a PNG GT.  Numpy arrays, CPU tensors or CUDA tensors.  Anything else
    raises ValueError before any device work."""

    def __init__(self, images: Sequence, masks: Sequence, device: int = 0):
        images, masks = list(images), list(masks)
        if not images:
            raise ValueError("an empty set")
        if len(images) != len(masks):
            raise ValueError(f"{len(images)} images but {len(masks)} masks")
        imgs, msks = [], []
        for i, (im, mk) in enumerate(zip(images, masks)):
            im, mk = _u8(im, f"image {i}"), _u8(mk, f"mask {i}")
            if not (im.dim() == 2 or (im.dim() == 3 and im.shape[2] == 3)):
                raise ValueError(f"image {i}: expected [h, w, 3] or [h, w], got {tuple(im.shape)}")
            if mk.dim() != 2:
                raise ValueError(f"mask {i}: expected [h, w], got {tuple(mk.shape)}")
            if tuple(mk.shape) != tuple(im.shape[:2]):
                raise ValueError(f"mask {i}: size {tuple(mk.shape)} differs from its image's {tuple(im.shape[:2])}")
            if not (1 <= im.shape[0] <= 32767 and 1 <= im.shape[1] <= 32767):
                raise ValueError(f"image {i}: h and w must lie in [1, 32767], got {tuple(im.shape[:2])}")
            imgs.append(im)
            msks.append(mk)
        self.device = torch.device("cuda", device)
        self.sizes = np.array([tuple(im.shape[:2]) for im in imgs], np.int64)
        self.geom_host = runtime.image_geometry(self.sizes)
        hw = (self.sizes[:, 0] * self.sizes[:, 1]).tolist()
        self.x = torch.empty(3 * sum(hw), dtype=torch.uint8, device=self.device)
        self.m = torch.empty(sum(hw), dtype=torch.uint8, device=self.device)
        for im, mk, o, n in zip(imgs, msks, self.geom_host["dst_off"].tolist(), hw):
            dst = self.x[3 * o:3 * (o + n)].view(im.shape[0], im.shape[1], 3)
            dst.copy_(im.unsqueeze(2).expand(-1, -1, 3) if im.dim() == 2 else im)
            self.m[o:o + n].copy_(mk.reshape(-1))
        self.geom = self._upload(self.geom_host)

    def __len__(self) -> int:
        return len(self.sizes)

    def _upload(self, arr: np.ndarray) -> torch.Tensor:
        """A small host table to the device on the current stream without a host sync (the pinned staging block stays reserved until
        the copy has run)."""
        return torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8)).pin_memory().to(self.device, non_blocking=True)

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def train_batch(self, indices, rng: Optional[random.Random] = None, samples=None, size=(224, 224), mean=IMAGENET_MEAN,
                    std=IMAGENET_STD) -> Tuple[torch.Tensor, torch.Tensor]:
        """SalData.__getitem__ in train mode for each index, then train.py's .float(): (x fp32 [N,3,H,W], target fp32 [N,1,H,W]) on the
        current stream.  `rng` draws each sample's crop and flip with augment_params, in index order; `samples` gives them instead as
        N tuples (y0, x0, ch, cw, flip); neither means no augmentation."""
        idx = _indices(indices, len(self))
        if rng is not None and samples is not None:
            raise ValueError("pass rng or samples, not both")
        s = np.zeros(len(idx), runtime.SAMPLE_DTYPE)
        s["image"] = idx
        if samples is not None:
            p = np.asarray(samples)
            if p.shape != (len(idx), 5) or not np.issubdtype(p.dtype, np.integer):
                raise ValueError(f"samples: expected {len(idx)} integer tuples (y0, x0, ch, cw, flip), got {p.dtype} {p.shape}")
            y0, x0, ch, cw, fl = (p[:, k].astype(np.int64) for k in range(5))
            h, w = self.sizes[idx, 0], self.sizes[idx, 1]
            if ((y0 < 0) | (x0 < 0) | (ch < 1) | (cw < 1) | (y0 + ch > h) | (x0 + cw > w)).any():
                raise ValueError("samples: a crop window lies outside its image")
            if not np.isin(fl, (0, 1, 2)).all():
                raise ValueError("samples: flip must be 0, 1 or 2")
        elif rng is not None:
            y0, x0, ch, cw, fl = np.array([augment_params(rng, *self.sizes[i]) for i in idx], np.int64).T
        else:
            y0 = x0 = fl = 0
            ch, cw = self.sizes[idx, 0], self.sizes[idx, 1]
        s["y0"], s["x0"], s["h"], s["w"], s["flip"] = y0, x0, ch, cw, fl
        N, (H, W) = len(idx), (int(size[0]), int(size[1]))
        x = torch.empty((N, 3, H, W), dtype=torch.float32, device=self.device)
        t = torch.empty((N, 1, H, W), dtype=torch.float32, device=self.device)
        sd = self._upload(s)
        runtime.train_batch_u8(self.x.data_ptr(), self.m.data_ptr(), self.geom.data_ptr(), sd.data_ptr(), N, H, W, mean, std,
                               x.data_ptr(), t.data_ptr(), self._stream())
        return x, t

    def csf_train_batch(self, indices, rng: Optional[random.Random] = None, flips=None, mean=IMAGENET_MEAN,
                        std=IMAGENET_STD) -> Tuple[torch.Tensor, torch.Tensor]:
        """CSF+Res2Net's ImageDataTrain.__getitem__ (dataset.py:23-33) for each index: (x fp32 [N,3,H,W], t fp32 [N,1,H,W]) on the current
        stream, without a host sync (csnet_csf_train_batch_u8).  The images are never cropped or resized, so every index must name an
        image of one exact size H x W.  x is load_image's normalisation (img_csf_in_value, mean / std as doubles), t the mask / 255 in
        fp32 (load_sal_label; a 3-channel GT's channel 0 is the mask the caller packs).  `rng` draws one flip per index with csf_flip,
        in index order; `flips` gives them instead (0 or 1 each, 1 = 'lr'); neither means no flip.  Mixed sizes, bad flips and bad
        indices raise ValueError before any device work."""
        idx = _indices(indices, len(self))
        if rng is not None and flips is not None:
            raise ValueError("pass rng or flips, not both")
        sizes = {(int(self.sizes[i, 0]), int(self.sizes[i, 1])) for i in idx}
        if len(sizes) != 1:
            raise ValueError(f"csf_train_batch takes images of one size, got {sorted(sizes)}")
        if flips is not None:
            fl = np.asarray(flips)
            if fl.shape != (len(idx),) or not np.issubdtype(fl.dtype, np.integer) or not np.isin(fl, (0, 1)).all():
                raise ValueError(f"flips: expected {len(idx)} integers, each 0 or 1, got {fl.dtype} {fl.shape}")
        elif rng is not None:
            fl = np.array([csf_flip(rng) for _ in idx], np.int64)
        else:
            fl = 0
        N, (H, W) = len(idx), sizes.pop()
        s = np.zeros(N, runtime.SAMPLE_DTYPE)
        s["image"], s["h"], s["w"], s["flip"] = idx, H, W, fl
        x = torch.empty((N, 3, H, W), dtype=torch.float32, device=self.device)
        t = torch.empty((N, 1, H, W), dtype=torch.float32, device=self.device)
        sd = self._upload(s)
        runtime.csf_train_batch_u8(self.x.data_ptr(), self.m.data_ptr(), self.geom.data_ptr(), sd.data_ptr(), N, H, W, mean, std,
                                   x.data_ptr(), t.data_ptr(), self._stream())
        return x, t

    def val_batch(self, indices, size=(224, 224), mean=IMAGENET_MEAN, std=IMAGENET_STD) -> torch.Tensor:
        """SalData in val mode: each image resized to `size` and normalised (no augmentation; exactly test.py's image path,
        csnet_resize_u8_to_input) -> fp32 [N,3,H,W] on the current stream."""
        idx = _indices(indices, len(self))
        N, (H, W) = len(idx), (int(size[0]), int(size[1]))
        x = torch.empty((N, 3, H, W), dtype=torch.float32, device=self.device)
        g = self._upload(self.geom_host[idx])
        runtime.resize_u8_to_input(self.x.data_ptr(), g.data_ptr(), N, H, W, mean, std, x.data_ptr(), self._stream())
        return x

    def val_mae(self, logits: torch.Tensor, indices) -> torch.Tensor:
        """train.py:262-279 for a batch: each image's MAE between its sigmoid map, resized to its GT's size by
        F.interpolate(bilinear) and quantised to 1/255, and its GT.  logits: CUDA fp32 [N,1,H,W] of the images `indices`.  Returns
        float64 [N] on the device (no host sync); the reference's epoch MAE is their mean."""
        idx = _indices(indices, len(self))
        if not isinstance(logits, torch.Tensor) or logits.device != self.device or logits.dtype != torch.float32 or logits.dim() != 4 \
                or logits.shape[0] != len(idx) or logits.shape[1] != 1:
            raise ValueError(f"logits: expected fp32 [{len(idx)},1,H,W] on {self.device}, got "
                             f"{getattr(logits, 'dtype', type(logits).__name__)} {tuple(getattr(logits, 'shape', ()))}")
        z = logits.contiguous()
        N, H, W = len(idx), z.shape[2], z.shape[3]
        mae = torch.empty(N, dtype=torch.float64, device=self.device)
        g = self._upload(self.geom_host[idx])
        runtime.val_mae_u8(z.data_ptr(), N, H, W, self.m.data_ptr(), g.data_ptr(), mae.data_ptr(), self._stream())
        return mae

    def evaluate(self, model, size=None, batch: int = 32, maps: bool = False, mean=IMAGENET_MEAN, std=IMAGENET_STD):
        """CSNet/test.py followed by eval.py (sal_metric.cpp) on this set, on the device from packed images to scores: each image goes
        through `model`'s engine as ModelEngine.forward_images_u8(images, size, batch=batch) runs it (size=None: TEST.IMAGE_H = 0,
        every image at its own size padded to multiples of 16), and its uint8 map at the image's original size is scored against its
        mask by csnet_salmetric_images_u8.  Only the counts, 2 x 256 + 1 numbers per image, come to the host, where SalMetric.add_images
        turns them into scores, adding the images in input order as sal_metric.cpp does.  Returns SalMetric.compute()'s dict (max_f,
        mean_f, precision, recall, mean_precision, mean_recall, mae, argmax); with maps=True, (scores, maps) where maps are each
        image's uint8 [h, w] map on the device, in input order.

        A CSFNet `model` is CSF+Res2Net/solver.py:test followed by the same SalMetric: every image at its own size (size must be None;
        the reference never resizes), grouped by exact size, and scored on CSFNet.forward_images_u8's maps (csnet_salmetric_csf_u8).
        mean / std go to its input kernel as doubles."""
        from .engine import exact_size, image_runs, native_size
        from .networks.csf_res2net import CSFNet
        from .salmetric import SalMetric

        csf = isinstance(model, CSFNet)
        if csf and size is not None:
            raise ValueError("CSF+Res2Net evaluates every image at its own size: size must be None")
        order, runs = image_runs(self.sizes, size, batch, key=exact_size if csf else native_size)
        g = self._upload(self.geom_host[order])
        N = len(self)
        hist_all = torch.empty((N, 256), dtype=torch.int32, device=self.device)
        hist_pos = torch.empty((N, 256), dtype=torch.int32, device=self.device)
        abs_sum = torch.empty(N, dtype=torch.int64, device=self.device)
        y = torch.empty(self.m.numel(), dtype=torch.uint8, device=self.device) if maps else None
        stream = self._stream()
        count = runtime.salmetric_csf_u8 if csf else runtime.salmetric_images_u8

        def score(logits, a, b, H, W, g_run):
            count(logits.data_ptr(), b - a, H, W, g_run, self.m.data_ptr(), y.data_ptr() if maps else 0,
                  hist_all[a].data_ptr(), hist_pos[a].data_ptr(), abs_sum[a].data_ptr(), stream)

        if csf:
            model.run_packed_images(self.x, g, runs, mean, std, score)
        else:
            model.engine().run_packed_images(self.x, g, runs, size is None, mean, std, score)
        inv = np.argsort(np.asarray(order, np.int64))
        ha, hp, ad = (t.cpu().numpy()[inv] for t in (hist_all, hist_pos, abs_sum))
        hw = self.sizes[:, 0] * self.sizes[:, 1]
        metric = SalMetric()
        metric.add_images(ha, hp, ad, hw)
        scores = metric.compute()
        if not maps:
            return scores
        offs = self.geom_host["dst_off"].tolist()
        return scores, [y[o:o + int(n)].view(int(h), int(w)) for o, n, (h, w) in zip(offs, hw, self.sizes)]
