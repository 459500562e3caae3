"""CSF+Res2Net training step time at batch 1 (CSF+Res2Net/solver.py:train: one image at its own size, net.eval()), fp32.

Sizes: 352 x 352 and csf_sizes.py's eight (400 x 300, 300 x 400 and six seeded ones).  Per size:
  backbone_fwd_ms / head_fwd_ms / head_bwd_ms / backbone_bwd_ms   CUDA events around each part of one step (sum-BCE / 2, backward), median
  step_ms                                                         their sum
  oracle_ms_tf32_off / oracle_ms_default                          the same step through oracle/csf_res2net_oracle.py on eager ATen autograd
                                                                  with torch.backends.cudnn.allow_tf32 False, and at torch's default (True)
In a separate profiled run at 352 x 352 (torch.profiler, CUDA activities): the head's kernels by total time, and the fp32 GEMM kernels'
achieved FLOP/s (the head's forward, data-gradient and weight-gradient FLOPs, from its shapes, over the gemm_f32 kernels' time) against
the 67 TFLOP/s fp32 data-sheet rate of an H100 SXM.  Prints one JSON line with the GPU's name and power limit (read-only query)."""
import argparse
import collections
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch
import torch.nn.functional as F

from oracle import csf_res2net_oracle as R
from scripts.csf_sizes import sizes
from scripts.images_e2e import gpu_info
from sod100k_b200 import compiler_r, modular_r, splits, synth
from sod100k_b200.networks import csf_res2net

FP32_PEAK = 67e12


def head_gemm_flops(h, w):
    """Multiply-adds x 2 of every head convolution at an h x w input, forward only (data and weight gradients: the same again each)."""
    dims = compiler_r.res2net_feat_dims(h, w)
    ci, co = splits.cuts(3840, compiler_r.FUSE_IN_SPLIT), splits.cuts(1408, compiler_r.FUSE_OUT_SPLIT)
    f = 0
    for j in range(4):
        for i in range(4):
            hw = dims[j] if i <= j else dims[i]                      # down paths convolve at j, up paths at i
            f += 2 * (co[j + 1] - co[j]) * (ci[i + 1] - ci[i]) * hw[0] * hw[1]
    for j in range(4):
        c = co[j + 1] - co[j]
        f += 2 * c * c * 9 * dims[j][0] * dims[j][1]                   # five dilated 3x3 convs, c in and c out together
        f += 2 * 1408 * c * dims[j][0] * dims[j][1]                    # fuse1x1 path j at branch j's size
    f += 2 * 1408 * dims[0][0] * dims[0][1]                            # cls_layer
    return f


def step_parts(m, x, lab, head_params):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    ev[0].record()
    feats = m.base(x)
    ev[1].record()
    y = modular_r.csf_head(m, feats, x.shape[2:])
    loss = F.binary_cross_entropy_with_logits(y, lab, reduction="sum") / 2
    ev[2].record()
    g = torch.autograd.grad(loss, list(feats) + head_params, retain_graph=True)
    ev[3].record()
    torch.autograd.backward(feats, g[:4])
    ev[4].record()
    for p, gp in zip(head_params, g[4:]):
        p.grad = gp
    return ev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--spread", type=int, default=6)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("csf_train_time.py measures on the GPU; no CUDA device is visible")
    m = csf_res2net.build_model()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    sd = {k: torch.from_numpy(v) for k, v in synth.synth_state_r(shapes, 21).items()}
    m.load_state_dict(sd)
    m.cuda().eval()
    head_params = [p for k, p in m.named_parameters() if not k.startswith("base.") and p.requires_grad]
    names = [k for k, p in m.named_parameters() if p.requires_grad]
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power, "steps": a.steps, "cases": []}
    for i, (h, w) in enumerate([(352, 352)] + sizes(a.spread, 2024)):
        x = torch.from_numpy(synth.randn_images(1, h, w, 2024 + i)).cuda()
        lab = (torch.rand((1, 1, h, w), device="cuda") > 0.5).float()
        times = []
        for it in range(a.warmup + a.steps):
            ev = step_parts(m, x, lab, head_params)
            torch.cuda.synchronize()
            if it >= a.warmup:
                times.append([ev[k].elapsed_time(ev[k + 1]) for k in range(4)])
            m.zero_grad(set_to_none=True)
        t = np.median(np.array(times), axis=0)
        case = dict(h=h, w=w, backbone_fwd_ms=t[0], head_fwd_ms=t[1], head_bwd_ms=t[2], backbone_bwd_ms=t[3], step_ms=float(t.sum()))
        sd_dev = {k: v.detach().clone().cuda() for k, v in m.state_dict().items()}
        ps = [sd_dev[k].requires_grad_(True) for k in names]

        def oracle_step():
            loss = F.binary_cross_entropy_with_logits(R.csfnet_forward(sd_dev, x), lab, reduction="sum") / 2
            torch.autograd.grad(loss, ps)
        for tf32 in (False, True):
            old = torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = tf32
            for _ in range(a.warmup):
                oracle_step()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                oracle_step()
            e1.record()
            torch.cuda.synchronize()
            torch.backends.cudnn.allow_tf32 = old
            case["oracle_ms_default" if tf32 else "oracle_ms_tf32_off"] = e0.elapsed_time(e1) / a.steps
        res["cases"].append(case)
        print(json.dumps(case), file=sys.stderr)
    # profiled run at 352 x 352
    from torch.profiler import ProfilerActivity, profile

    x = torch.from_numpy(synth.randn_images(1, 352, 352, 7)).cuda()
    lab = (torch.rand((1, 1, 352, 352), device="cuda") > 0.5).float()
    step_parts(m, x, lab, head_params)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            step_parts(m, x, lab, head_params)
        torch.cuda.synchronize()
    per = collections.Counter()
    for e in prof.key_averages():
        if e.device_time_total > 0:
            per[e.key] += e.device_time_total / 3 / 1000.0
    ours = {k: v for k, v in per.items() if "csnet::" in k or "bias_grad" in k}   # the head's kernels (the backbone's are cuDNN's)
    gemm_ms = sum(v for k, v in ours.items() if "g32::gemm_f32_kernel" in k)
    flops = 3 * head_gemm_flops(352, 352)
    res["profile_352"] = {"head_kernels_total_ms": sum(ours.values()), "head_kernels_ms": dict(sorted(((k[:120], round(v, 4)) for k, v in ours.items()), key=lambda kv: -kv[1])),
                          "gemm_ms": gemm_ms, "gemm_flops": flops, "gemm_tflops": flops / (gemm_ms * 1e-3) / 1e12,
                          "gemm_share_of_fp32_datasheet": flops / (gemm_ms * 1e-3) / FP32_PEAK}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
