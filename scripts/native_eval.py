"""Test-set evaluation with every image at its own size (CSNet/test.py with TEST.IMAGE_H = 0, then eval.py's SalMetric) on the device.

Workload: a seeded set of uint8 images and masks, csnet-L-x2, most of them at ECSSD's sizes (400 x 300 and 300 x 400, with some
400 x h and w x 400, h, w in [180, 400]) and the rest with h and w drawn from [180, 520].  Times
  evaluate            SalImages.evaluate(size=None): packed set on the device -> scores, wall time ending in the host reduction,
                      with every native plan already resident; the host reduction (SalMetric.add_images) alone
  forward_cuda        ModelEngine.forward_images_u8(size=None) on CUDA tensors, and forward_host on numpy images
  first_pass          the first evaluate of a fresh engine: the same work plus one plan per padded size; the plan cost per size is
                      split on a sample of sizes into compile (compiler.compile_csnet), create (runtime.Plan) and first run (graph capture
                      for small batches, module load) against the same run warm
  fixed_224           the same set through evaluate / forward_images_u8 at size=(224, 224), and with CUDA events on one batch of
                      the whole set's 224 x 224 logits: csnet_salmetric_images_u8 (no map stored) against csnet_resize_logits_to_u8
  reference_sample    the reference's host loop on a bounded sample: scipy zoom to the padded size, the engine's host call at that
                      size per image, zoom back, astype(uint8), then the numpy SalMetric (oracle/salmetric.py) on the sample
Prints one JSON line with the GPU's name and power limit (read-only nvidia-smi query)."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

from oracle import salmetric as OS
from scripts.images_e2e import event_ms, gpu_info, wall_ms
from sod100k_b200 import checkpoints, compiler, engine, runtime
from sod100k_b200.data import SalImages
from sod100k_b200.salmetric import SalMetric
from tests import sk_native as SN
from tests import sk_resize as SK


def seeded_set(n, seed):
    rng = np.random.default_rng(seed)
    sizes = []
    for _ in range(n):
        r = rng.random()
        if r < 0.35:
            sizes.append((300, 400))
        elif r < 0.55:
            sizes.append((400, 300))
        elif r < 0.7:
            v = int(rng.integers(180, 401))
            sizes.append((400, v) if rng.random() < 0.5 else (v, 400))
        else:
            sizes.append(tuple(int(v) for v in rng.integers(180, 521, size=2)))
    imgs = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in sizes]
    masks = [((rng.random((h, w)) > 0.7) * 255).astype(np.uint8) for h, w in sizes]
    return sizes, imgs, masks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=300)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=16, help="images in the host restatement's timing")
    ap.add_argument("--plan-sample", type=int, default=4, help="padded sizes whose first-use cost is split into its parts")
    ap.add_argument("--dtype", default="fp16")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("native_eval.py measures on the GPU; no CUDA device visible")
    name, power = gpu_info()
    sizes, imgs, masks = seeded_set(a.images, 2025)
    N = len(imgs)
    padded = sorted({engine.native_size(h, w) for h, w in sizes})
    m, cfg, sd = checkpoints.build_from_npz("csnet-L-x2")
    m.cuda().eval().set_precision(a.dtype)
    eng = m.engine()
    eng.freeze(True)
    eng.native_plan_budget = 1 << 40                 # the warm timings keep every native plan resident
    ds = SalImages(imgs, masks)
    dev = torch.device("cuda", 0)
    res = {"metric": "native_eval", "gpu": name, "power_limit": power, "model": "csnet-L-x2", "dtype": a.dtype, "images": N,
           "batch": a.batch, "padded_sizes": len(padded), "pixels_M": sum(h * w for h, w in sizes) / 1e6, "steps": a.steps}

    with torch.no_grad():
        # first use: one plan per padded size
        t0 = time.perf_counter()
        scores = ds.evaluate(m, size=None, batch=a.batch)
        first_s = time.perf_counter() - t0
        res["resident_native_arena_MB"] = sum(p.arena_bytes for p in eng._native_plans.values()) / 1e6
        # warm: every plan resident
        ev_ms, _ = wall_ms(lambda: ds.evaluate(m, size=None, batch=a.batch), a.steps, a.warmup)
        counts = (np.zeros((N, 256), np.int64), np.ones((N, 256), np.int64), np.zeros(N, np.int64), np.full(N, 1000))
        red_ms, _ = wall_ms(lambda: SalMetric().add_images(*counts), a.steps, a.warmup)
        dimgs = [torch.from_numpy(im).cuda() for im in imgs]
        fc_ms, _ = wall_ms(lambda: eng.forward_images_u8(dimgs, size=None, batch=a.batch), a.steps, a.warmup)
        fh_ms, _ = wall_ms(lambda: eng.forward_images_u8(imgs, size=None, batch=a.batch), a.steps, a.warmup)
        res.update(evaluate_ms=ev_ms, evaluate_img_s=N / ev_ms * 1e3, host_reduction_ms=red_ms,
                   forward_cuda_ms=fc_ms, forward_cuda_img_s=N / fc_ms * 1e3, forward_host_ms=fh_ms, forward_host_img_s=N / fh_ms * 1e3,
                   max_f=scores["max_f"], mae=scores["mae"])
        res["first_pass_s"] = first_s
        res["first_pass_plan_s_per_size"] = (first_s - ev_ms / 1e3) / len(padded)

        # first-use cost split on a sample of sizes: compile, create, first run against a warm run
        parts = []
        per_size = {s: sum(1 for h, w in sizes if engine.native_size(h, w) == s) for s in padded}
        for (H, W) in sorted(padded, key=lambda s: -per_size[s])[:a.plan_sample]:
            n = min(a.batch, per_size[(H, W)])
            t0 = time.perf_counter()
            prog = compiler.compile_csnet(m.layer_config, eng._state(), H, W, eng.dtype)
            t1 = time.perf_counter()
            plan = runtime.Plan(prog, max_batch=n, device=0)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            x = torch.zeros((n, 3, H, W), dtype=torch.float32, device=dev)
            plan.forward(x)
            torch.cuda.synchronize()
            t3 = time.perf_counter()
            warm, _ = wall_ms(lambda: plan.forward(x), 5, 1)
            plan.close()
            parts.append({"H": H, "W": W, "images": per_size[(H, W)], "batch": n, "compile_ms": (t1 - t0) * 1e3, "create_ms": (t2 - t1) * 1e3,
                          "first_run_ms": (t3 - t2) * 1e3, "warm_run_ms": warm})
        res["plan_cost_sample"] = parts

        # the same set at the fixed network size
        ds.evaluate(m, size=(224, 224), batch=a.batch)
        f_ev_ms, _ = wall_ms(lambda: ds.evaluate(m, size=(224, 224), batch=a.batch), a.steps, a.warmup)
        f_fc_ms, _ = wall_ms(lambda: eng.forward_images_u8(dimgs, size=(224, 224)), a.steps, a.warmup)
        stream = torch.cuda.current_stream().cuda_stream
        z = torch.randn((N, 1, 224, 224), generator=torch.Generator().manual_seed(5)).cuda()
        yd = torch.empty(ds.m.numel(), dtype=torch.uint8, device=dev)
        ha = torch.empty((N, 256), dtype=torch.int32, device=dev)
        hp, ad = torch.empty_like(ha), torch.empty(N, dtype=torch.int64, device=dev)
        zc = torch.full_like(z, -10.0)               # every pixel in bin 0, as a map's background: the most contended case
        k_out, k_eval, k_eval_bg = event_ms([
            lambda: runtime.resize_logits_to_u8(z.data_ptr(), N, 224, 224, ds.geom.data_ptr(), yd.data_ptr(), stream),
            lambda: runtime.salmetric_images_u8(z.data_ptr(), N, 224, 224, ds.geom.data_ptr(), ds.m.data_ptr(), 0, ha.data_ptr(),
                                                hp.data_ptr(), ad.data_ptr(), stream),
            lambda: runtime.salmetric_images_u8(zc.data_ptr(), N, 224, 224, ds.geom.data_ptr(), ds.m.data_ptr(), 0, ha.data_ptr(),
                                                hp.data_ptr(), ad.data_ptr(), stream)], 20, 3)
        res["fixed_224"] = {"evaluate_ms": f_ev_ms, "evaluate_img_s": N / f_ev_ms * 1e3,
                            "forward_cuda_ms": f_fc_ms, "forward_cuda_img_s": N / f_fc_ms * 1e3,
                            "kernel_ms": {"resize_logits_to_u8": k_out, "salmetric_images_u8": k_eval,
                                          "salmetric_images_u8_one_bin": k_eval_bg}}

        # the reference's host loop on a sample (its model call replaced by the engine's host call at the padded size)
        S = min(a.sample, N)
        for im in imgs[:S]:                             # plans and host staging of the sample's sizes, outside the timing
            H, W = SN.padded_size(*im.shape[:2])
            eng.forward_host(torch.empty((1, 3, H, W), dtype=torch.float32).pin_memory())
        t_in = t_net = t_out = 0.0
        maps = []
        for im in imgs[:S]:
            t0 = time.perf_counter()
            H, W = SN.padded_size(*im.shape[:2])
            v = im.astype(np.float64) / 255.0
            if (H, W) != im.shape[:2]:
                v = SK.resize(v, (H, W))
            x = torch.from_numpy(np.transpose((v - np.asarray(SK.IMAGENET_MEAN)) / np.asarray(SK.IMAGENET_STD), (2, 0, 1))[None]
                                 .astype(np.float32))
            t1 = time.perf_counter()
            z = eng.forward_host(x)
            t2 = time.perf_counter()
            maps.append((SK.resize(torch.sigmoid(z)[0, 0].numpy(), im.shape[:2]) * 255).astype(np.uint8))
            t3 = time.perf_counter()
            t_in, t_net, t_out = t_in + t1 - t0, t_net + t2 - t1, t_out + t3 - t2
        t0 = time.perf_counter()
        OS.evaluate(maps, masks[:S])
        t_metric = time.perf_counter() - t0
        total = t_in + t_net + t_out + t_metric
        res["reference_sample"] = {"images": S, "img_s": S / total,
                                   "ms_per_img": {"resize_in": t_in / S * 1e3, "network_host_call": t_net / S * 1e3,
                                                  "resize_out": t_out / S * 1e3, "salmetric_numpy": t_metric / S * 1e3}}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
