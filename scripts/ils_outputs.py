"""Write the fp16 logits of csnet-L-x1 at 224x224 and csnet-L-x2 at 512x512 on seeded inputs, for a byte comparison of two
builds of the native library (a kernel change that keeps every FMA and its order must leave them bit-identical).

    python scripts/ils_outputs.py OUT_DIR      -> OUT_DIR/<model>_<size>.npy (float32 logits), and which kernel ran each op
    python scripts/ils_outputs.py --compare DIR_A DIR_B     -> max |difference| and the count of differing elements

The batches (256 at 224x224, 64 at 512x512) are large enough that the plan puts every 1x1-kind ILBlock and the stem on the
streaming kernel, as at the bench shape; the script fails if an ILBlock of stages 0-2 runs elsewhere.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

CASES = [("csnet-L-x1", 224, 256), ("csnet-L-x2", 512, 64)]
ILS = "il_stream_kernel (TMA + wgmma)"


def write(out):
    import collections

    import torch

    from sod100k_b200 import checkpoints, compiler, runtime, synth

    os.makedirs(out, exist_ok=True)
    st = torch.cuda.current_stream().cuda_stream
    for model, size, batch in CASES:
        cfg, sd = checkpoints.load_npz(model)
        sd = {k: torch.from_numpy(v) for k, v in sd.items()}
        x = torch.from_numpy(synth.randn_images(batch, size, size, 4321)).cuda()
        prog = compiler.compile_csnet(cfg, sd, size, size, "fp16")
        p = runtime.Plan(prog, max_batch=batch)
        kernels = [p.op_kernel(i) for i in range(len(prog.ops))]
        print(f"{model} {size}x{size} batch {batch}: {dict(collections.Counter(kernels))}")
        # the ILBlocks of stages 0-2 (stage 3 at 224 is 56 wide: not a streaming shape)
        off = [o.name for o, k in zip(prog.ops, kernels) if o.kind == 3 and o.name[:7] in ("stage0.", "stage1.", "stage2.") and k != ILS]
        if off:
            sys.exit(f"{model} {size}x{size}: ILBlock ops not on the streaming kernel: {off}")
        y = torch.empty((batch, 1, size, size), dtype=torch.float32, device="cuda")
        p.run(batch, [x.data_ptr(), y.data_ptr()], st)
        torch.cuda.synchronize()
        np.save(os.path.join(out, f"{model}_{size}.npy"), y.cpu().numpy())
        p.close()


def compare(a, b):
    same = True
    for model, size, _ in CASES:
        ya, yb = (np.load(os.path.join(d, f"{model}_{size}.npy")) for d in (a, b))
        diff = int((ya.view(np.uint32) != yb.view(np.uint32)).sum())
        print(f"{model} {size}x{size}: {diff} of {ya.size} elements differ, max |diff| {np.abs(ya - yb).max():.3e}")
        same = same and diff == 0
    return same


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?")
    ap.add_argument("--compare", nargs=2, metavar=("DIR_A", "DIR_B"))
    a = ap.parse_args()
    if a.compare:
        sys.exit(0 if compare(*a.compare) else 1)
    write(a.out)
