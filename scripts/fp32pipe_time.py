"""Per-op device times of the ops that run on the FP32 pipe in the bench program (csnet-L-x2, 224x224, fp16, batch 256): the
MSBlock dilated paths (msd_kernel; the 28-wide one runs on mix_tc_kernel) and the stage-3 ILBlocks (il_block_kernel), with the
step total and each kernel's sum.

    python scripts/fp32pipe_time.py [--lib PATH] [--passes P] [--json OUT]

Each op's time is the minimum over P profiled runs (CUDA events around every launch).  Next to it: the FP32-pipe
multiply-adds it needs (the MS paths' 3x3 taps; the ILBlocks' two depthwise 3x3 layers, their 1x1 GEMMs run on tensor
cores) against 128 FMA / clock / SM at the sampled SM clock, and its algorithmic bytes (bench.py's op_bytes) against the
H100 SXM data-sheet HBM bandwidth.  `--lib` loads another build of libcsnet_b200.so, so that two builds can be timed in
alternating processes on the same inputs.
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

_spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
bench = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(bench)

from sod100k_b200 import checkpoints, compiler, ir, runtime, synth  # noqa: E402

MODEL, SIZE, BATCH = "csnet-L-x2", 224, 256
FMA_PER_CLK_SM = 128


def fp32_macs(prog, op, n):
    """Multiply-adds of one op launch that run on the FP32 pipe."""
    if op.kind == ir.OP_ILBLOCK:                          # two depthwise 3x3 layers on each output branch
        return n * sum(2 * 9 * prog.tensors[t].C * prog.tensors[t].H * prog.tensors[t].W for t in op.dsts)
    d = prog.tensors[op.dst]                             # dilated 3x3 paths of an MSBlock
    return n * sum(9 * q.cin * q.cout * d.H * d.W for q in op.paths)


def selected(prog):
    return [i for i, o in enumerate(prog.ops)
            if ".ms.convs." in o.name or (o.kind == ir.OP_ILBLOCK and o.name.startswith("stage3."))]


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                              capture_output=True, text=True, timeout=10).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return ""


class ClockSampler(threading.Thread):
    """SM clock samples (nvidia-smi, every ~100 ms) while the timed passes run."""

    def __init__(self):
        super().__init__(daemon=True)
        self.mhz, self.stop = [], threading.Event()

    def run(self):
        while not self.stop.is_set():
            try:
                self.mhz.append(float(smi("clocks.sm")))
            except ValueError:
                pass
            self.stop.wait(0.1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", help="libcsnet_b200.so to load instead of the in-tree build")
    ap.add_argument("--passes", type=int, default=10)
    ap.add_argument("--json", help="also write the numbers to this file")
    a = ap.parse_args()

    import numpy as np
    import torch

    cfg, sd = checkpoints.load_npz(MODEL)
    prog = compiler.compile_csnet(cfg, {k: torch.from_numpy(v) for k, v in sd.items()}, SIZE, SIZE, "fp16")
    sel = selected(prog)
    if a.lib:
        runtime.LIB_PATH = os.path.abspath(a.lib)          # the library Plan loads
    runtime.load_library()
    plan = runtime.Plan(prog, max_batch=BATCH)
    x = torch.from_numpy(synth.randn_images(8, SIZE, SIZE, 7)).cuda().repeat(BATCH // 8, 1, 1, 1)
    y = torch.empty((BATCH, 1, SIZE, SIZE), dtype=torch.float32, device="cuda")
    ptrs, st = [x.data_ptr(), y.data_ptr()], torch.cuda.current_stream().cuda_stream
    for _ in range(3):
        plan.run(BATCH, ptrs, st)
    torch.cuda.synchronize()

    clocks = ClockSampler()
    clocks.start()
    ms = np.min(np.array([plan.profile(BATCH, ptrs, st) for _ in range(a.passes)]), axis=0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    steps = []
    for _ in range(a.passes):
        e0.record()
        plan.run(BATCH, ptrs, st)
        e1.record()
        torch.cuda.synchronize()
        steps.append(e0.elapsed_time(e1))
    clocks.stop.set()
    clocks.join()

    props = torch.cuda.get_device_properties(0)
    mhz = float(np.median(clocks.mhz)) if clocks.mhz else float("nan")
    fp32_gmacs = props.multi_processor_count * FMA_PER_CLK_SM * mhz * 1e-3
    print(f"{props.name}, power limit {smi('power.limit')} W, SM clock {mhz:.0f} MHz (median of {len(clocks.mhz)} samples), "
          f"{props.multi_processor_count} SMs; library {runtime.LIB_PATH}")
    print(f"{MODEL} {SIZE}x{SIZE} fp16 batch {BATCH}: step {min(steps):.3f} ms (min of {a.passes}), sum of op minima {ms.sum():.3f} ms")
    print(f"FP32 pipe {fp32_gmacs:.0f} GMAC/s at that clock, HBM {bench.H100_HBM_GBS:.0f} GB/s (data sheet)")
    print(f"{'op':26s} {'kernel':38s} {'ms':>7s} {'GMAC':>6s} {'GMAC/s':>7s} {'%FP32':>6s} {'GB':>6s} {'GB/s':>6s} {'%HBM':>5s}")

    def line(name, kernel, t, mac, nb):
        gmacs, gbs = mac / 1e9 / (t * 1e-3), nb / 1e9 / (t * 1e-3)
        print(f"{name:26s} {kernel[:38]:38s} {t:7.3f} {mac / 1e9:6.2f} {gmacs:7.0f} {100 * gmacs / fp32_gmacs:5.1f}% "
              f"{nb / 1e9:6.3f} {gbs:6.0f} {100 * gbs / bench.H100_HBM_GBS:4.1f}%")

    rows, groups = [], {}
    for i in sel:
        o = prog.ops[i]
        mac, nb = fp32_macs(prog, o, BATCH), bench.op_bytes(prog, o, BATCH)
        line(o.name, plan.op_kernel(i), ms[i], mac, nb)
        rows.append({"op": o.name, "kernel": plan.op_kernel(i), "ms": float(ms[i]), "gmac": mac / 1e9, "gb": nb / 1e9})
        g = groups.setdefault(plan.op_kernel(i).split(" ")[0], [0.0, 0, 0])
        g[0] += float(ms[i]); g[1] += mac; g[2] += nb
    for k, (t, mac, nb) in groups.items():
        line(f"[sum {k}]", "", t, mac, nb)
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"gpu": props.name, "power_limit_w": smi("power.limit"), "sm_mhz": mhz, "lib": runtime.LIB_PATH,
                       "step_ms": min(steps), "ops": rows, "groups": {k: {"ms": v[0], "gmac": v[1] / 1e9, "gb": v[2] / 1e9}
                                                                         for k, v in groups.items()}}, f, indent=1)
    plan.close()


if __name__ == "__main__":
    main()
