"""GPU check of the streaming ILBlock kernel (csrc/il_stream.cuh): every qualifying block fused in isolation, the streaming
kernel against the all-generic program (same inputs bit for bit), for several batch sizes / image sizes, then per-op times of the
full fp16 program with the streaming kernel on and off.  Needs a GPU:  python scripts/ils_check.py [--time]"""
import os
import sys
import json

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from sod100k_b200 import compiler, runtime, synth, checkpoints


def plan(prog, nb, ils, min_chunks=0):
    os.environ["CSNET_ILS"] = "1" if ils else "0"
    os.environ["CSNET_ILS_MIN_CHUNKS"] = str(min_chunks)
    return runtime.Plan(prog, max_batch=nb)


def check(tag, h, w, nb, seed=31):
    cfg, sd = checkpoints.load_npz(tag)
    sd = {k: torch.from_numpy(v) for k, v in sd.items()}
    x = torch.from_numpy(synth.randn_images(nb, h, w, seed)).cuda()
    base = compiler.compile_csnet(cfg, sd, h, w, "fp16", reuse_arena=False, fuse=False, tensor_core=False)
    p0 = plan(base, nb, False)
    p0.forward(x)
    full = compiler.compile_csnet(cfg, sd, h, w, "fp16", fuse=True)
    names = [o.name for o in full.ops if o.kind == 3]
    worst = 0.0
    for name in names:
        prog = compiler.compile_csnet(cfg, sd, h, w, "fp16", reuse_arena=False, fuse={name}, tensor_core=False)
        for ils in (True, False):
            p1 = plan(prog, nb, ils)
            p1.forward(x)
            torch.cuda.synchronize()
            for b in (0, 1):
                key = f"{name}/{b}"
                if key not in prog.taps:
                    continue
                ref = p0.read_tensor(base.taps[key], nb)
                got = p1.read_tensor(prog.taps[key], nb)
                err = (got - ref).abs()
                rel = err.max().item() / max(1.0, ref.abs().max().item())
                bad = int((err > 4e-3 * max(1.0, ref.abs().max().item())).sum().item())
                print(f"{tag} {h}x{w} bs{nb} {key:14s} {'stream' if ils else 'tiled '} rel err {rel:.2e} bad {bad} finite {bool(torch.isfinite(got).all())}", flush=True)
                if ils:
                    worst = max(worst, rel)
                    if bad:
                        idx = torch.nonzero(err > 4e-3 * max(1.0, ref.abs().max().item()))[:8].tolist()
                        print("   first bad (n, c, y, x):", idx, flush=True)
            p1.close()
    p0.close()
    return worst


def timing(batch=256):
    cfg, sd = checkpoints.load_npz("csnet-L-x2")
    sd = {k: torch.from_numpy(v) for k, v in sd.items()}
    x = torch.from_numpy(synth.randn_images(8, 224, 224, 7)).cuda().repeat(batch // 8, 1, 1, 1)
    prog = compiler.compile_csnet(cfg, sd, 224, 224, "fp16")
    out = {}
    for ils in (False, True):
        p = plan(prog, batch, ils, 592)
        y = torch.empty((batch, 1, 224, 224), dtype=torch.float32, device="cuda")
        for _ in range(3):
            p.run(batch, [x.data_ptr(), y.data_ptr()], torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        ms = np.median(np.array([p.profile(batch, [x.data_ptr(), y.data_ptr()], torch.cuda.current_stream().cuda_stream) for _ in range(5)]), axis=0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            p.run(batch, [x.data_ptr(), y.data_ptr()], torch.cuda.current_stream().cuda_stream)
        e1.record()
        torch.cuda.synchronize()
        step = e0.elapsed_time(e1) / 10
        print(f"ILS={int(ils)}: step {step:.3f} ms = {batch / step * 1e3:.0f} img/s", flush=True)
        for o, t in zip(prog.ops, ms):
            if o.kind == 3:
                print(f"   {o.name:12s} {t:.3f} ms", flush=True)
        out[f"ils{int(ils)}"] = {"step_ms": step, "ops": {o.name: float(t) for o, t in zip(prog.ops, ms)}}
        out[f"y{int(ils)}"] = y.clone()
        p.close()
    d = (torch.sigmoid(out["y0"]) - torch.sigmoid(out["y1"])).abs().max().item()
    print(f"max |sigmoid(tiled) - sigmoid(stream)| over the batch: {d:.3e}", flush=True)
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump({k: v for k, v in out.items() if k.startswith("ils")}, open("gpurun_out/ils_timing.json", "w"), indent=1)


if __name__ == "__main__":
    w = 0.0
    w = max(w, check("csnet-L-x2", 224, 224, 3))
    w = max(w, check("csnet-L-x2", 96, 160, 5))
    w = max(w, check("csnet-L-x1", 128, 64, 2))
    print("worst streaming rel err", w, flush=True)
    if "--time" in sys.argv:
        timing()
