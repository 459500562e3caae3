"""CSF+Res2Net training with fp32 and bf16 activation storage (net.train_storage), alternated in one process.

At 352 x 352, batch 1 and batch 8 (8 images of one size from SalImages.csf_train_batch), synthetic seeded weights, net.eval() as
solver.train keeps it.  Per storage and batch, over `--rounds` alternations of `--steps` steps each after `--warmup`:
  backbone_fwd_ms / head_fwd_ms / head_bwd_ms / backbone_bwd_ms   CUDA events around each part of a step (sum-BCE, backward), median
  device_ms                                                       their sum
  wall_ms                                                         host clock around whole CSFTrainer-style steps, each synchronised
  peak_mib                                                        torch.cuda.max_memory_allocated over the storage's steps
In a separate profiled run per storage and batch (torch.profiler, CUDA activities): the head GEMM kernels' time (gemm_bf16_kernel or
gemm_f32_kernel, and with their split-K merges) and their achieved TFLOP/s, from the head's forward, data-gradient and
weight-gradient FLOPs (scripts/csf_train_time.head_gemm_flops) over that time.  Prints one JSON line with the GPU's name and power
limit (read-only query)."""
import argparse
import collections
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

from scripts.csf_train_time import head_gemm_flops
from scripts.images_e2e import gpu_info
from sod100k_b200 import modular_r, synth
from sod100k_b200.data import SalImages
from sod100k_b200.networks import csf_res2net
from sod100k_b200.train_ops import BceSumFn

GEMM = {"fp32": "gemm_f32_kernel", "bf16": "gemm_bf16_kernel"}
MERGE = {"fp32": "gemm_merge_kernel", "bf16": "gemm_bf16_merge_kernel"}


def backbone(m, x, storage):
    if storage == "bf16":
        with torch.autocast("cuda", dtype=torch.bfloat16):
            return [f.to(torch.bfloat16).contiguous() for f in m.base(x)]
    return m.base(x)


def step_parts(m, x, t, head_params, storage):
    """One step as CSFNet.forward runs it in training, cut into four timed parts."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    ev[0].record()
    feats = backbone(m, x, storage)
    ev[1].record()
    y = modular_r.csf_head(m, feats, x.shape[2:])
    loss = BceSumFn.apply(y, t, 10)
    ev[2].record()
    g = torch.autograd.grad(loss, list(feats) + head_params, retain_graph=True)
    ev[3].record()
    torch.autograd.backward(feats, g[:4])
    ev[4].record()
    return ev


def whole_step(m, x, t):
    with torch.enable_grad():
        BceSumFn.apply(m(x), t, 10).backward()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("csf_train_bf16.py measures on the GPU; no CUDA device is visible")
    m0 = csf_res2net.build_model()
    shapes = {k: tuple(v.shape) for k, v in m0.state_dict().items()}
    sd = {k: torch.from_numpy(v) for k, v in synth.synth_state_r(shapes, 21).items()}
    nets = {}
    for storage in ("fp32", "bf16"):
        m = csf_res2net.build_model()
        m.load_state_dict(sd)
        m.cuda().eval()
        m.train_storage = storage
        nets[storage] = m
    h = w = 352
    g = np.random.default_rng(3)
    ds = SalImages([g.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(8)],
                   [(g.random((h, w)) > 0.5).astype(np.uint8) * 255 for _ in range(8)])
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power, "h": h, "w": w, "steps": a.steps, "rounds": a.rounds, "cases": []}
    for n in [int(b) for b in a.batches.split(",")]:
        x, t = ds.csf_train_batch(list(range(n)))
        parts = collections.defaultdict(list)
        walls = collections.defaultdict(list)
        peak = {}
        for r in range(a.rounds):
            for storage in ("fp32", "bf16"):
                m = nets[storage]
                hp = [p for k, p in m.named_parameters() if not k.startswith("base.") and p.requires_grad]
                torch.cuda.reset_peak_memory_stats()
                for it in range(a.warmup + a.steps):
                    ev = step_parts(m, x, t, hp, storage)
                    torch.cuda.synchronize()
                    if it >= a.warmup:
                        parts[storage].append([ev[k].elapsed_time(ev[k + 1]) for k in range(4)])
                    m.zero_grad(set_to_none=True)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(a.steps):
                    whole_step(m, x, t)
                    m.zero_grad(set_to_none=True)
                torch.cuda.synchronize()
                walls[storage].append((time.perf_counter() - t0) * 1e3 / a.steps)
                peak[storage] = max(peak.get(storage, 0), torch.cuda.max_memory_allocated() / 2 ** 20)
        from torch.profiler import ProfilerActivity, profile

        flops = 3 * n * head_gemm_flops(h, w)
        for storage in ("fp32", "bf16"):
            m = nets[storage]
            hp = [p for k, p in m.named_parameters() if not k.startswith("base.") and p.requires_grad]
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    step_parts(m, x, t, hp, storage)
                    m.zero_grad(set_to_none=True)
                torch.cuda.synchronize()
            gemm_ms = merge_ms = 0.0
            for e in prof.key_averages():
                if GEMM[storage] in e.key:
                    gemm_ms += e.device_time_total / 3 / 1000.0
                elif MERGE[storage] in e.key:
                    merge_ms += e.device_time_total / 3 / 1000.0
            p = np.median(np.array(parts[storage]), axis=0)
            case = dict(batch=n, storage=storage, backbone_fwd_ms=p[0], head_fwd_ms=p[1], head_bwd_ms=p[2], backbone_bwd_ms=p[3],
                        device_ms=float(p.sum()), wall_ms_per_round=walls[storage], wall_ms=float(np.median(walls[storage])),
                        peak_mib=peak[storage], gemm_ms=gemm_ms, gemm_merge_ms=merge_ms, gemm_flops=flops,
                        gemm_tflops=flops / (gemm_ms * 1e-3) / 1e12, gemm_tflops_with_merge=flops / ((gemm_ms + merge_ms) * 1e-3) / 1e12)
            res["cases"].append(case)
            print(json.dumps(case), file=sys.stderr)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
