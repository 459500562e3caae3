"""Training data on the device (sod100k_b200.data.SalImages) against what the reference's loaders cost, csnet-L-x2 at 224 x 224.

Workload: seeded synthetic uint8 images and masks, h and w drawn from [180, 520] (DUTS-like sizes), resident on the GPU.  Reports
  builder_ms        csnet_train_batch_u8 for one batch of `--batch` augmented samples (CUDA events)
  step_*_img_s      Trainer.step fed from SalImages.train_batch (crop / flip drawn on the host, one kernel builds the batch) against
                    the same step on one fixed device batch, alternated in one run
  host_img_s_core   SalData.__getitem__ (CSNet_training/utils/prepare_data.py:109-139) restated with scipy (tests/sal_data.py), one
                    core, on a sample: what one DataLoader worker delivers
  val_mae_ms        SalImages.val_mae for `--val` images in one call, against train.py:262-279's torch loop (one F.interpolate, l1_loss
                    and .item() per image) on the same GPU and logits
Prints one JSON line with the GPU's name and power limit (read-only nvidia-smi query)."""
import argparse
import json
import os
import random
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

from scripts.images_e2e import event_ms, gpu_info
from sod100k_b200 import checkpoints, data
from sod100k_b200.trainer import Trainer
from tests import sal_data as SD


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--images", type=int, default=1024, help="images in the device-resident set")
    ap.add_argument("--steps", type=int, default=4, help="training steps per arm and round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--val", type=int, default=1000)
    ap.add_argument("--sample", type=int, default=24, help="images in the host restatement's timing")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_images_e2e.py measures on the GPU; no CUDA device visible")
    name, power = gpu_info()
    rng = np.random.default_rng(2024)
    n_img = max(a.images, a.val, a.batch)
    sizes = [tuple(int(v) for v in rng.integers(180, 521, size=2)) for _ in range(n_img)]
    imgs = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in sizes]
    masks = []
    for h, w in sizes:                                       # a salient blob and a grey rim, like a GT map
        yy, xx = np.mgrid[:h, :w]
        r = ((yy - h * rng.uniform(0.3, 0.7)) / h) ** 2 + ((xx - w * rng.uniform(0.3, 0.7)) / w) ** 2
        masks.append(np.where(r < 0.05, 255, np.where(r < 0.06, 128, 0)).astype(np.uint8))
    ds = data.SalImages(imgs, masks)
    H = W = 224
    B = a.batch
    m, _, _ = checkpoints.build_from_npz("csnet-L-x2")
    m.cuda()

    # the builder kernel alone
    aug = random.Random(0)
    idx = list(range(B))
    samples = [data.augment_params(aug, *sizes[i]) for i in idx]
    (builder_ms,) = event_ms([lambda: ds.train_batch(idx, samples=samples)], 20, 3)

    # Trainer.step fed from SalImages against the same step on one fixed device batch, alternated
    tr = Trainer(m, lr=1e-4, weight_decay=5e-3)
    x_fix, t_fix = ds.train_batch(idx, aug)
    perm = torch.Generator().manual_seed(1)
    batches = iter(())

    def fed():
        nonlocal batches
        b = next(batches, None)
        if b is None or len(b) < B:                          # drop_last
            batches = iter(torch.randperm(len(ds), generator=perm).split(B))
            b = next(batches)
        return tr.step(*ds.train_batch(b, aug))

    arms = {"sal_images": fed, "fixed_batch": lambda: tr.step(x_fix, t_fix)}
    for f in arms.values():
        f()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, f in arms.items():
            t0 = time.perf_counter()
            for _ in range(a.steps):
                f()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) / a.steps)
    step_img_s = {k: B / float(np.median(v)) for k, v in times.items()}

    # SalData.__getitem__ on the host, one core
    S = min(a.sample, n_img)
    aug = random.Random(3)
    t0 = time.perf_counter()
    for i in range(S):
        SD.sal_item(imgs[i], masks[i], (H, W), data.augment_params(aug, *sizes[i]))
    host_s = (time.perf_counter() - t0) / S

    # validation MAE: one call against train.py's per-image loop
    m.eval()
    V = a.val
    vidx = list(range(V))
    with torch.no_grad():
        z = torch.cat([m(ds.val_batch(vidx[k:k + B])) for k in range(0, V, B)])
    (mae_ms,) = event_ms([lambda: ds.val_mae(z, vidx)], 10, 2)
    t0 = time.perf_counter()
    loop = SD.val_mae_loop(z, masks[:V])
    torch.cuda.synchronize()
    loop_ms = (time.perf_counter() - t0) * 1e3
    got = ds.val_mae(z, vidx).cpu().numpy()
    max_diff = float(np.abs(got - np.asarray(loop)).max())

    res = {
        "metric": "train_images_e2e", "gpu": name, "power_limit": power, "model": "csnet-L-x2", "network_hw": [H, W],
        "batch": B, "images": len(ds), "hw_range": [180, 520], "steps": a.steps, "rounds": a.rounds,
        "device_set_MB": (ds.x.numel() + ds.m.numel()) / 1e6,
        "builder_ms": builder_ms, "builder_img_s": B / builder_ms * 1e3,
        "step_sal_images_img_s": step_img_s["sal_images"], "step_fixed_batch_img_s": step_img_s["fixed_batch"],
        "step_ms_rounds": {k: [t * 1e3 for t in v] for k, v in times.items()},
        "host_sal_data_ms_per_img": host_s * 1e3, "host_img_s_core": 1.0 / host_s, "host_sample": S,
        "host_cores_for_fixed_step": step_img_s["fixed_batch"] * host_s,
        "val_images": V, "val_mae_ms": mae_ms, "torch_loop_ms": loop_ms, "val_speedup": loop_ms / mae_ms,
        "val_mae_max_abs_diff": max_diff,
    }
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
