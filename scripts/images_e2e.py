"""Images of any size through csnet-L-x2 (fp16 storage, 224x224 network input): CSNet/test.py:71-98 with both resizes.

Workload: 256 seeded synthetic uint8 images, h and w drawn from [180, 520] (saliency test sets differ in size per image).  Times
  host_ms     ModelEngine.forward_images_u8 on numpy images, host to host (packing into pinned memory included)
  c_call_ms   csnet_plan_run_host_images_u8 alone on the already packed pinned buffer (host_pack_ms: the packing alone)
  cuda_ms     forward_images_u8 on CUDA tensors (packing on the device, both resizes around the network, current stream)
  restated    the reference's host loop on a bounded sample: scipy zoom per image, the engine's fp32-input host call, zoom back
and, with CUDA events on the device-resident batch, the two resize kernels against the network forward between them.
Prints one JSON line with the GPU's name and power limit (read-only nvidia-smi query)."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

from sod100k_b200 import checkpoints, runtime
from tests import sk_resize as SK


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:                                   # the timings stand without it
        return f"unknown ({e})", "unknown"


def wall_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t)), t


def event_ms(fns, steps, warmup):
    """Median device time of each function in `fns`, run back to back on the current stream."""
    for _ in range(warmup):
        for f in fns:
            f()
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(len(fns) + 1)] for _ in range(steps)]
    for e in ev:
        e[0].record()
        for i, f in enumerate(fns):
            f()
            e[i + 1].record()
    torch.cuda.synchronize()
    return [float(np.median([e[i].elapsed_time(e[i + 1]) for e in ev])) for i in range(len(fns))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=32, help="images in the host restatement's timing")
    ap.add_argument("--dtype", default="fp16")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("images_e2e.py measures on the GPU; no CUDA device visible")
    name, power = gpu_info()
    rng = np.random.default_rng(2024)
    sizes = [tuple(int(v) for v in rng.integers(180, 521, size=2)) for _ in range(a.batch)]
    imgs = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in sizes]
    H = W = 224
    N = len(imgs)
    m, _, _ = checkpoints.build_from_npz("csnet-L-x2")
    m.cuda().eval().set_precision(a.dtype)
    eng = m.engine()
    eng.freeze(True)
    in_bytes = sum(3 * h * w for h, w in sizes)
    out_bytes = sum(h * w for h, w in sizes)

    with torch.no_grad():
        host_ms, _ = wall_ms(lambda: eng.forward_images_u8(imgs), a.steps, a.warmup)
        plan = eng.plan_for(N, H, W, torch.device("cuda", 0))
        geom = runtime.image_geometry(sizes)
        x = eng._pinned_images[:in_bytes]
        y = torch.empty(out_bytes, dtype=torch.uint8, pin_memory=True)
        c_ms, _ = wall_ms(lambda: plan.run_host_images_u8(N, x.data_ptr(), in_bytes, geom, y.data_ptr(), out_bytes, SK.IMAGENET_MEAN,
                                                          SK.IMAGENET_STD), a.steps, a.warmup)
        timgs = [torch.from_numpy(im) for im in imgs]
        pack_ms, _ = wall_ms(lambda: torch.cat([t.reshape(-1) for t in timgs], out=x), a.steps, a.warmup)
        alloc_ms, _ = wall_ms(lambda: torch.empty(out_bytes, dtype=torch.uint8, pin_memory=True), a.steps, a.warmup)
        dimgs = [torch.from_numpy(im).cuda() for im in imgs]
        cuda_ms, _ = wall_ms(lambda: eng.forward_images_u8(dimgs), a.steps, a.warmup)

        # the two kernels against the network between them, device-resident batch
        stream = torch.cuda.current_stream().cuda_stream
        xd = torch.cat([t.reshape(-1) for t in dimgs])
        gd = torch.from_numpy(geom.view(np.uint8)).cuda()
        x_in = torch.empty((N, 3, H, W), dtype=torch.float32, device="cuda")
        logits = plan.forward(x_in)
        yd = torch.empty(out_bytes, dtype=torch.uint8, device="cuda")
        k_in, k_fwd, k_out = event_ms([
            lambda: runtime.resize_u8_to_input(xd.data_ptr(), gd.data_ptr(), N, H, W, SK.IMAGENET_MEAN, SK.IMAGENET_STD, x_in.data_ptr(), stream),
            lambda: plan.run(N, [x_in.data_ptr(), logits.data_ptr()], stream),
            lambda: runtime.resize_logits_to_u8(logits.data_ptr(), N, H, W, gd.data_ptr(), yd.data_ptr(), stream)], a.steps, a.warmup)

        # the reference's host loop on a sample: zoom + normalise per image, the engine's host call, sigmoid + zoom back per image
        S = min(a.sample, N)
        sub = imgs[:S]
        x_host = torch.empty((S, 3, H, W), dtype=torch.float32).pin_memory()
        eng.forward_host(x_host)                                 # warm the plan's host staging
        t0 = time.perf_counter()
        for i, im in enumerate(sub):
            v = (SK.resize(im.astype(np.float64) / 255.0, (H, W)) - np.asarray(SK.IMAGENET_MEAN)) / np.asarray(SK.IMAGENET_STD)
            x_host[i] = torch.from_numpy(np.transpose(v, (2, 0, 1)).astype(np.float32))
        t1 = time.perf_counter()
        z = eng.forward_host(x_host)
        t2 = time.perf_counter()
        s = torch.sigmoid(z)[:, 0].numpy()
        for i, im in enumerate(sub):
            (SK.resize(s[i], im.shape[:2]) * 255).astype(np.uint8)
        t3 = time.perf_counter()

    res = {
        "metric": "images_e2e", "gpu": name, "power_limit": power, "model": "csnet-L-x2", "dtype": a.dtype, "network_hw": [H, W],
        "batch": N, "hw_range": [180, 520], "steps": a.steps, "warmup": a.warmup, "packed_in_MB": in_bytes / 1e6, "maps_MB": out_bytes / 1e6,
        "host_ms": host_ms, "host_img_s": N / host_ms * 1e3,
        "c_call_ms": c_ms, "c_call_img_s": N / c_ms * 1e3, "host_pack_ms": pack_ms, "host_alloc_maps_ms": alloc_ms,
        "cuda_ms": cuda_ms, "cuda_img_s": N / cuda_ms * 1e3,
        "kernels_ms": {"resize_in": k_in, "network": k_fwd, "resize_out": k_out},
        "resize_share_of_chunk": (k_in + k_out) / (k_in + k_fwd + k_out),
        "resize_in_GB_s": (in_bytes + N * 3 * H * W * 4) / k_in / 1e6,
        "resize_out_GB_s": (N * H * W * 4 + out_bytes) / k_out / 1e6,
        "restated_sample": S,
        "restated_ms_per_img": {"resize_in": (t1 - t0) / S * 1e3, "network_host_call": (t2 - t1) / S * 1e3,
                                "sigmoid_resize_out": (t3 - t2) / S * 1e3},
        "restated_img_s": S / (t3 - t0),
    }
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
