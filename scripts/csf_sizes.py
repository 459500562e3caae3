"""CSF+Res2Net one image at a time at each image's own size (CSF+Res2Net/solver.py:test), on the engine against eager ATen.

Workload: seeded images at ECSSD's sizes (400 x 300, 300 x 400) and `--spread` more with h, w drawn from [180, 520], batch 1, seeded
synthetic weights, fp32 and fp16.  Per size and precision, with every plan already built (the first call at a size compiles the
head program and creates its plan; that cost is reported separately as first_call_ms):
  model_ms            model(x): the backbone (torch / cuDNN) and the head program; median of CUDA-event times
  backbone_ms         model.backbone(x) alone; head_ms = model_ms - backbone_ms
  resize_share        the RESIZE ops' share of the head's device time (csnet_plan_profile, one event per op)
  kernels             how many ops run on each kernel (csnet_plan_op_kernel); ops on mix_generic_kernel are listed with their time
  oracle_ms           the same image through oracle/csf_res2net_oracle.py's forward on the GPU (eager ATen, fp32): the baseline
  max_abs_vs_oracle   |engine - oracle| on that image
Prints one JSON line with the GPU's name and power limit (read-only nvidia-smi query)."""
import argparse
import collections
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

from oracle import csf_res2net_oracle as R
from scripts.images_e2e import event_ms, gpu_info
from sod100k_b200 import ir, synth
from sod100k_b200.networks import csf_res2net


def sizes(spread, seed):
    rng = np.random.default_rng(seed)
    return [(400, 300), (300, 400)] + [tuple(int(v) for v in rng.integers(180, 521, size=2)) for _ in range(spread)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spread", type=int, default=6)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=2024)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("csf_sizes.py measures on the GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    m = csf_res2net.build_model()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    sd = {k: torch.from_numpy(v) for k, v in synth.synth_state_r(shapes, 21).items()}
    m.load_state_dict(sd)
    m.cuda().eval()
    sd_dev = {k: v.cuda() for k, v in sd.items()}
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power, "steps": a.steps, "warmup": a.warmup, "cases": []}
    hw = sizes(a.spread, a.seed)
    with torch.no_grad():
        for i, (h, w) in enumerate(hw):
            x = torch.from_numpy(synth.randn_images(1, h, w, a.seed + i)).cuda()
            oracle_ms = event_ms([lambda: R.csfnet_forward(sd_dev, x)], a.steps, a.warmup)[0]
            y_ref = R.csfnet_forward(sd_dev, x)
            for dtype in ("fp32", "fp16"):
                m.set_precision(dtype)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                y = m(x)
                torch.cuda.synchronize()
                first = (time.perf_counter() - t0) * 1e3
                model_ms, backbone_ms = event_ms([lambda: m(x), lambda: m.backbone(x)], a.steps, a.warmup)
                plan = m._plans[(h, w, dtype, 0)]
                feats = m.backbone(x)
                out = torch.empty((1, 1, h, w), device="cuda")
                ptrs = [f.data_ptr() for f in feats] + [out.data_ptr()]
                per_op = np.median([plan.profile(1, ptrs, torch.cuda.current_stream().cuda_stream) for _ in range(a.steps)], axis=0)
                ops = plan.prog.ops
                kern = [plan.op_kernel(k) for k in range(len(ops))]
                resize_ms = float(sum(t for o, t in zip(ops, per_op) if o.kind == ir.OP_RESIZE))
                generic = {o.name: round(float(t), 4) for o, k, t in zip(ops, kern, per_op) if k.startswith("mix_generic")}
                res["cases"].append({
                    "h": h, "w": w, "dtype": dtype, "model_ms": model_ms, "backbone_ms": backbone_ms, "head_ms": model_ms - backbone_ms,
                    "head_profiled_ms": float(per_op.sum()), "resize_ms": resize_ms, "resize_share": resize_ms / float(per_op.sum()),
                    "kernels": dict(collections.Counter(kern)), "mix_generic_ops_ms": generic,
                    "mix_generic_ms": float(sum(generic.values())), "first_call_ms": first, "oracle_ms": oracle_ms,
                    "max_abs_vs_oracle": float((y - y_ref).abs().max())})
    for dtype in ("fp32", "fp16"):
        cs = [c for c in res["cases"] if c["dtype"] == dtype]
        res[f"mean_{dtype}"] = {k: float(np.mean([c[k] for c in cs])) for k in
                                ("model_ms", "backbone_ms", "head_ms", "resize_ms", "resize_share", "mix_generic_ms", "oracle_ms",
                                 "first_call_ms")}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
