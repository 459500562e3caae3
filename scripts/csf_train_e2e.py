"""One epoch of CSF+Res2Net training (CSF+Res2Net/solver.py:train, iter_size 10, batch 1) two ways on the same seeded set and weights.

Workload: native_eval.seeded_set (64 images, most at ECSSD's 300 x 400 and 400 x 300, the rest with h or w drawn from [180, 520]) with
its masks, seeded synthetic weights (synth.synth_state_r, seed 21), one fixed image order and a random.Random(seed) of flips per epoch.
  host    solver.train restated on decoded arrays: numpy load_image / load_sal_label / flip per image, torch.Tensor, .cuda(), the module,
          F.binary_cross_entropy_with_logits(sum) / iter_size, backward, torch.optim.Adam every iter_size micro-steps
  device  CSFTrainer fed by SalImages.csf_train_batch: the set packed on the device once, one sample kernel, BceSumFn, one FusedAdam
The two loops alternate, each starting from the same weights, `--rounds` times.  Per loop: img/s (wall time of the epoch ending in a
device synchronise), host CPU seconds per micro-step (time.process_time), and the epoch's mean loss.  CUDA events time the two new
kernels (csnet_csf_train_batch_u8, csnet_train_bce_sum) on one 300 x 400 sample.  Prints one JSON line with the GPU's name and power
limit (read-only nvidia-smi query)."""
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
from scripts.native_eval import seeded_set
from sod100k_b200 import runtime, synth
from sod100k_b200.data import SalImages, csf_flip
from sod100k_b200.networks import csf_res2net
from sod100k_b200.trainer import CSFTrainer
from tests import csf_ref

ITER_SIZE, LR, WD = 10, 5e-5, 5e-4


def host_epoch(net, imgs, masks, order, seed):
    """solver.train's epoch, with aveGrad starting at 0."""
    opt = torch.optim.Adam([p for p in net.parameters() if p.requires_grad], lr=LR, weight_decay=WD)
    net.zero_grad()
    rng = random.Random(seed)
    ave_grad, r_loss = 0, 0
    for i in order:
        x = csf_ref.load_image_test(imgs[i])                         # load_image
        t = (np.array(masks[i], dtype=np.float32) / 255.)[np.newaxis, ...]
        if csf_flip(rng) == 1:                                        # cv_random_flip
            x, t = x[:, :, ::-1].copy(), t[:, :, ::-1].copy()
        x, t = torch.Tensor(x)[None].cuda(), torch.Tensor(t)[None].cuda()
        pred = net(x)
        loss = torch.nn.functional.binary_cross_entropy_with_logits(pred, t, reduction="sum") / ITER_SIZE
        r_loss += loss.data
        loss.backward()
        ave_grad += 1
        if ave_grad % ITER_SIZE == 0:
            opt.step()
            opt.zero_grad()
            ave_grad = 0
    return r_loss


def device_epoch(net, ds, order, seed):
    tr = CSFTrainer(net, lr=LR, weight_decay=WD, iter_size=ITER_SIZE)
    tr.epoch_begin()
    rng = random.Random(seed)
    r_loss = 0
    for i in order:
        r_loss += tr.step(*ds.csf_train_batch([i], rng))
    tr.epoch_end(0)
    return r_loss


def timed(fn, n):
    torch.cuda.synchronize()
    w0, c0 = time.perf_counter(), time.process_time()
    r = fn()
    torch.cuda.synchronize()
    w1, c1 = time.perf_counter(), time.process_time()
    return {"img_s": n / (w1 - w0), "epoch_s": w1 - w0, "host_cpu_ms_per_step": (c1 - c0) / n * 1e3, "mean_loss": float(r) / n}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("csf_train_e2e.py measures on the GPU; no CUDA device visible")
    name, power = gpu_info()
    sizes, imgs, masks = seeded_set(a.images, 2025)
    n = len(imgs)
    order = np.random.default_rng(3).permutation(n).tolist()
    net = csf_res2net.build_model()
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    sd = {k: torch.from_numpy(v) for k, v in synth.synth_state_r(shapes, 21).items()}
    net = net.cuda().eval()
    ds = SalImages(imgs, masks)
    res = {"metric": "csf_train_e2e", "gpu": name, "power_limit": power, "images": n, "distinct_sizes": len(set(sizes)),
           "iter_size": ITER_SIZE, "batch": 1, "rounds": []}
    # warm-up: cuDNN algorithm choice and first-use costs for every size, in both loops
    net.load_state_dict(sd)
    host_epoch(net, imgs, masks, order, 0)
    net.load_state_dict(sd)
    device_epoch(net, ds, order, 0)
    for r in range(a.rounds):
        row = {}
        net.load_state_dict(sd)
        row["host"] = timed(lambda: host_epoch(net, imgs, masks, order, 100 + r), n)
        net.load_state_dict(sd)
        row["device"] = timed(lambda: device_epoch(net, ds, order, 100 + r), n)
        res["rounds"].append(row)
    for k in ("host", "device"):
        res[f"{k}_img_s"] = float(np.median([row[k]["img_s"] for row in res["rounds"]]))
        res[f"{k}_cpu_ms_per_step"] = float(np.median([row[k]["host_cpu_ms_per_step"] for row in res["rounds"]]))

    stream = torch.cuda.current_stream().cuda_stream
    big = [i for i, s in enumerate(sizes) if s == (300, 400)][0]
    x = torch.empty((1, 3, 300, 400), device="cuda")
    t = torch.empty((1, 1, 300, 400), device="cuda")
    s = np.zeros(1, runtime.SAMPLE_DTYPE)
    s["image"], s["h"], s["w"], s["flip"] = big, 300, 400, 1
    sd_dev = torch.from_numpy(s.view(np.uint8).copy()).cuda()
    z = torch.randn((1, 1, 300, 400), device="cuda")
    dl, loss = torch.empty_like(z), torch.empty(1, device="cuda")
    k_in, k_bce = event_ms([
        lambda: runtime.csf_train_batch_u8(ds.x.data_ptr(), ds.m.data_ptr(), ds.geom.data_ptr(), sd_dev.data_ptr(), 1, 300, 400,
                                           csf_res2net.CSFNet.IMAGENET_MEAN, csf_res2net.CSFNet.IMAGENET_STD, x.data_ptr(),
                                           t.data_ptr(), stream),
        lambda: runtime.train_bce_sum(z.data_ptr(), t.data_ptr(), dl.data_ptr(), loss.data_ptr(), z.numel(), ITER_SIZE, stream)], 50, 5)
    res["kernels_us_300x400"] = {"csf_train_batch_u8": k_in * 1e3, "train_bce_sum": k_bce * 1e3}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
