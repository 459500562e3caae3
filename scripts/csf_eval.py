"""CSF+Res2Net test-set evaluation on the device (CSF+Res2Net/solver.py:test, then SalMetric), fp32 and fp16.

Workload: native_eval.seeded_set, the same size mix as the CSNet measurement (most images at ECSSD's 300 x 400 and 400 x 300, the rest
with h or w drawn from [180, 520]), seeded synthetic weights (synth.synth_state_r, seed 21).  CSF+Res2Net runs every image at its exact
size, so every distinct size is one head plan.  Per precision:
  first_pass        the first SalImages.evaluate of a fresh net at batch 16: the same work plus one plan compile and create per exact
                    size; plan_cost_sample splits that cost on a sample of sizes into compile (compiler_r.compile_csf_head) and create
                    (runtime.Plan)
  evaluate          SalImages.evaluate at batch 1 / 4 / 8 / 16 with every plan resident (wall time ending in the host reduction)
  forward_images    CSFNet.forward_images_u8 at batch 16 with CUDA tensors in, and with numpy images in (pinned staging, maps back)
  arena_MB          one plan's arena at 300 x 400 for max_batch 1 / 4 / 8 / 16
  kernels_us        CUDA events around csnet_csf_input_u8, csnet_csf_maps_u8 and csnet_salmetric_csf_u8 on 16 images at 300 x 400, and
                    their share of one such run (input, backbone, head and counting)
  reference_sample  solver.test restated on the host for a sample: numpy load_image_test, net(x) at batch 1, sigmoid, .cpu(), 255 *,
                    rint, then the numpy SalMetric (oracle/salmetric.py)
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

from oracle import salmetric as OS
from scripts.images_e2e import event_ms, gpu_info, wall_ms
from scripts.native_eval import seeded_set
from sod100k_b200 import compiler_r, runtime, synth
from sod100k_b200.data import SalImages
from sod100k_b200.networks import csf_res2net
from tests import csf_ref

BATCHES = (1, 4, 8, 16)


def clocks():
    """The SM clock now and its maximum (read-only query)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out
    except Exception as e:                           # the timings stand without it
        return f"unknown ({e})"


def build_net():
    m = csf_res2net.build_model()
    sd = synth.synth_state_r({k: tuple(v.shape) for k, v in m.state_dict().items()}, 21)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    m = m.cuda().eval()
    m.plan_budget = 1 << 40                          # the warm timings keep every plan resident
    return m


def kernel_times(m, steps, warmup):
    """Device time of the three calls on 16 images at 300 x 400, and of one whole run of those images."""
    n, H, W = 16, 300, 400
    rng = np.random.default_rng(3)
    dev = torch.device("cuda", 0)
    x = torch.from_numpy(rng.integers(0, 256, size=n * H * W * 3, dtype=np.uint8)).to(dev)
    msk = torch.from_numpy(((rng.random(n * H * W) > 0.7) * 255).astype(np.uint8)).to(dev)
    g = torch.from_numpy(runtime.image_geometry([(H, W)] * n).view(np.uint8)).to(dev)
    xin = torch.empty((n, 3, H, W), device=dev)
    z = torch.randn((n, 1, H, W), generator=torch.Generator().manual_seed(5)).to(dev)
    y = torch.empty(n * H * W, dtype=torch.uint8, device=dev)
    ha = torch.empty((n, 256), dtype=torch.int32, device=dev)
    hp, ad = torch.empty_like(ha), torch.empty(n, dtype=torch.int64, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    mean, std = csf_res2net.CSFNet.IMAGENET_MEAN, csf_res2net.CSFNet.IMAGENET_STD

    def count(logits, a, b, H_, W_, g_run):
        runtime.salmetric_csf_u8(logits.data_ptr(), b - a, H_, W_, g_run, msk.data_ptr(), 0, ha.data_ptr(), hp.data_ptr(), ad.data_ptr(), s)

    t_in, t_maps, t_count, t_run = event_ms([
        lambda: runtime.csf_input_u8(x.data_ptr(), g.data_ptr(), n, H, W, mean, std, xin.data_ptr(), s),
        lambda: runtime.csf_maps_u8(z.data_ptr(), n, H, W, g.data_ptr(), y.data_ptr(), s),
        lambda: runtime.salmetric_csf_u8(z.data_ptr(), n, H, W, g.data_ptr(), msk.data_ptr(), 0, ha.data_ptr(), hp.data_ptr(),
                                         ad.data_ptr(), s),
        lambda: m.run_packed_images(x, g, [(0, n, H, W)], mean, std, count)], steps, warmup)
    return {"images": n, "H": H, "W": W, "csf_input_u8_us": t_in * 1e3, "csf_maps_u8_us": t_maps * 1e3,
            "salmetric_csf_u8_us": t_count * 1e3, "run_ms": t_run, "input_and_count_share_of_run": (t_in + t_count) / t_run,
            "input_GB_s": n * H * W * 15 / (t_in * 1e-3) / 1e9}


def reference_sample(m, imgs, masks):
    t_in = t_net = t_out = 0.0
    maps = []
    for im in imgs:
        t0 = time.perf_counter()
        x = torch.from_numpy(np.ascontiguousarray(csf_ref.load_image_test(im))[None]).cuda()
        t1 = time.perf_counter()
        with torch.no_grad():
            preds = m(x)
        pred = np.squeeze(torch.sigmoid(preds).cpu().numpy())
        t2 = time.perf_counter()
        maps.append(csf_ref.map_bytes(pred))
        t3 = time.perf_counter()
        t_in, t_net, t_out = t_in + t1 - t0, t_net + t2 - t1, t_out + t3 - t2
    t0 = time.perf_counter()
    OS.evaluate(maps, masks)
    t_metric = time.perf_counter() - t0
    S = len(imgs)
    return {"images": S, "img_s": S / (t_in + t_net + t_out + t_metric),
            "ms_per_img": {"load_image_test": t_in / S * 1e3, "net_sigmoid_cpu": t_net / S * 1e3, "map_bytes": t_out / S * 1e3,
                           "salmetric_numpy": t_metric / S * 1e3}}


def run(dtype, sizes, imgs, masks, a):
    m = build_net().set_precision(dtype)
    ds = SalImages(imgs, masks)
    exact = sorted(set(sizes))
    N = len(imgs)
    res = {"distinct_sizes": len(exact)}
    with torch.no_grad():
        t0 = time.perf_counter()
        scores = ds.evaluate(m, batch=16)
        torch.cuda.synchronize()
        first_s = time.perf_counter() - t0
        ev = {}
        for b in sorted(BATCHES, reverse=True):      # largest first: the plans made at batch 16 serve the smaller batches
            ms, _ = wall_ms(lambda: ds.evaluate(m, batch=b), a.steps, a.warmup)
            ev[b] = {"ms": ms, "img_s": N / ms * 1e3}
        res.update(max_f=scores["max_f"], mae=scores["mae"], first_pass_s=first_s,
                   first_pass_plan_s_per_size=(first_s - ev[16]["ms"] / 1e3) / len(exact),
                   evaluate={str(b): ev[b] for b in BATCHES})
        dimgs = [torch.from_numpy(im).cuda() for im in imgs]
        fc, _ = wall_ms(lambda: m.forward_images_u8(dimgs, batch=16), a.steps, a.warmup)
        fh, _ = wall_ms(lambda: m.forward_images_u8(imgs, batch=16), a.steps, a.warmup)
        res["forward_images"] = {"cuda_ms": fc, "cuda_img_s": N / fc * 1e3, "numpy_ms": fh, "numpy_img_s": N / fh * 1e3}

        # plan cost per size, and the arena per plan at each batch, at 300 x 400
        feats = {}
        parts = []
        for (h, w) in exact[:a.plan_sample]:
            x = torch.zeros((1, 3, h, w), device="cuda")
            feats[(h, w)] = [tuple(f.shape[1:]) for f in m.backbone(x)]
            t0 = time.perf_counter()
            prog = compiler_r.compile_csf_head(m.head_state(), feats[(h, w)], h, w, dtype)
            t1 = time.perf_counter()
            plan = runtime.Plan(prog, max_batch=16, device=0)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            plan.close()
            parts.append({"h": h, "w": w, "compile_ms": (t1 - t0) * 1e3, "create_ms": (t2 - t1) * 1e3})
        res["plan_cost_sample"] = parts
        fd = [tuple(f.shape[1:]) for f in m.backbone(torch.zeros((1, 3, 300, 400), device="cuda"))]
        prog = compiler_r.compile_csf_head(m.head_state(), fd, 300, 400, dtype)
        arena = {}
        for b in BATCHES:
            plan = runtime.Plan(prog, max_batch=b, device=0)
            arena[str(b)] = plan.arena_bytes / 1e6
            plan.close()
        res["arena_MB_300x400"] = arena
        res["kernels"] = kernel_times(m, 20, 3)
        S = min(a.sample, N)
        csf_ref.solver_test(m, imgs[:S])              # the sample's plans at batch 1, outside the timing
        res["reference_sample"] = reference_sample(m, imgs[:S], masks[:S])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=48)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=16, help="images in the host restatement's timing")
    ap.add_argument("--plan-sample", type=int, default=3, help="exact sizes whose plan cost is split into compile and create")
    ap.add_argument("--dtypes", default="fp32,fp16")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("csf_eval.py measures on the GPU; no CUDA device visible")
    name, power = gpu_info()
    sizes, imgs, masks = seeded_set(a.images, 2025)
    res = {"metric": "csf_eval", "gpu": name, "power_limit": power, "clocks": clocks(), "model": "csf_res2net (synthetic weights)",
           "images": len(imgs), "pixels_M": sum(h * w for h, w in sizes) / 1e6, "steps": a.steps}
    for dtype in a.dtypes.split(","):
        res[dtype] = run(dtype, sizes, imgs, masks, a)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
