"""The CSNet training step with fp32 and with bf16 activation storage (Trainer(storage=...)), csnet-L-x2 at 224 x 224 on one GPU.

Runs, in one process, on seeded synthetic batches:
  * fp32 and bf16 at batch 256 without recompute, alternated for --rounds rounds;
  * bf16 at batch 512 without recompute;
  * bf16 at batch 1024 with ILBlock recompute (SURVEY config c3's batch);
  * one torch.profiler step per storage at batch 256 (a run of its own), splitting the step's kernel time between the FP32-pipe-bound
    convolution kernels (conv1x1 / conv_fwd / conv_wgrad) and the bandwidth-bound ones (BatchNorm, depthwise, pooling, resampling,
    the ordered partial merges); the rest (BCE, Adam, ATen adds and fills) is reported as "other".
Per run: img/s from CUDA events around `--steps` back-to-back steps after `--warmup` (the device is synchronised before the first
event and before the events are read), torch.cuda.max_memory_allocated, and the median SM clock sampled by nvidia-smi during the timed steps.  Prints one JSON line
with the card's name and power limit (read-only nvidia-smi queries), and writes it to --out if given."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch

from bench import ClockSampler
from scripts.images_e2e import gpu_info
from sod100k_b200 import checkpoints, synth
from sod100k_b200.trainer import Trainer

CONV = ("conv1x1", "conv_fwd", "conv_wgrad", "tr_mix")
BANDWIDTH = ("bn_", "dw3", "pool", "resample_bwd", "reduce_partials")


def run(storage, batch, recompute, steps, warmup, size=224, profile=False):
    model, _, _ = checkpoints.build_from_npz("csnet-L-x2")
    model.cuda()
    tr = Trainer(model, lr=1e-4, weight_decay=5e-3, flops_weight=3.0, recompute=recompute, storage=storage)
    x = torch.from_numpy(synth.randn_images(batch, size, size, 1234)).cuda()
    t = torch.from_numpy(synth.random_masks(batch, size, size, 1236)).cuda()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    for _ in range(warmup):
        tr.step(x, t)
    torch.cuda.synchronize()
    rec = {"storage": storage, "batch": batch, "recompute": recompute}
    if profile:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            tr.step(x, t)
            torch.cuda.synchronize()
        split = {"conv_fp32_pipe": 0.0, "bandwidth": 0.0, "other": 0.0}
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            us = e.time_range.elapsed_us()
            name = e.name
            key = "conv_fp32_pipe" if any(k in name for k in CONV) else "bandwidth" if any(k in name for k in BANDWIDTH) else "other"
            split[key] += us / 1e3
        total = sum(split.values())
        rec["kernel_ms"] = {k: round(v, 2) for k, v in split.items()}
        rec["kernel_share"] = {k: round(v / total, 4) for k, v in split.items()}
    else:
        clocks = ClockSampler(0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            tr.step(x, t)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        clk = clocks.stop()
        rec.update({"img_per_s": round(batch * steps / (ms * 1e-3), 1), "ms_per_step": round(ms / steps, 2), "steps": steps, "warmup": warmup,
                    "peak_memory_GiB": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), "sm_mhz": clk.get("sm_mhz"),
                    "clock_reasons": clk.get("reasons")})
    del tr, model, x, t
    torch.cuda.empty_cache()
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_bf16.py measures on the GPU; no CUDA device found")
    name, power = gpu_info()
    out = {"gpu": name, "power_limit": power, "model": "csnet-L-x2", "size": 224, "flops_weight": 3.0, "b256": [], "runs": []}
    for _ in range(a.rounds):
        for storage in ("fp32", "bf16"):
            out["b256"].append(run(storage, 256, False, a.steps, a.warmup))
    for storage in ("fp32", "bf16"):
        r = [v["img_per_s"] for v in out["b256"] if v["storage"] == storage]
        out[f"b256_{storage}_median_img_per_s"] = statistics.median(r)
        out[f"b256_{storage}_peak_memory_GiB"] = max(v["peak_memory_GiB"] for v in out["b256"] if v["storage"] == storage)
    out["runs"].append(run("bf16", 512, False, a.steps, a.warmup))
    out["runs"].append(run("bf16", 1024, True, 3, 1))
    out["profile_b256"] = [run(s, 256, False, 1, a.warmup, profile=True) for s in ("fp32", "bf16")]
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
