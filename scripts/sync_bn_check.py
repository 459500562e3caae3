"""torchrun --nproc-per-node 2 scripts/sync_bn_check.py [--steps K] — synchronized BatchNorm on 2 GPUs (NCCL).

dp_check.py with BatchNorm in training mode and the model converted by nn.SyncBatchNorm.convert_sync_batchnorm:
  1. each rank back-propagates its shard of the global batch; the flat gradient bucket is all-reduced (mean) and rank 0
     compares it with the single-process gradient of the whole batch (unconverted model): max |diff| / max |g| per tensor;
  2. one Trainer step on the converted model must leave both ranks with bit-identical parameters and running statistics;
  3. Trainer.step time at batch 256 per GPU (csnet-L-x2, 224 x 224), fp32 and bf16 storage, converted against unconverted,
     the two alternated in rounds; rank 0 prints the median step time of each and the spread over the rounds."""
import argparse
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, torch.distributed as dist, torch.nn as nn
from sod100k_b200 import checkpoints, synth, train_ops as T
from sod100k_b200.trainer import FlatGrads, Trainer

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10, help="timed steps per round")
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--batch", type=int, default=256, help="images per GPU in the timing")
args = ap.parse_args()

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
per = 2
x = torch.from_numpy(synth.randn_images(per * world, 64, 64, 5)).cuda()
t = torch.from_numpy(synth.random_masks(per * world, 64, 64, 6)).cuda()


def model(convert):
    m, _, _ = checkpoints.build_from_npz("csnet-L-x2")
    if convert:
        m = nn.SyncBatchNorm.convert_sync_batchnorm(m)
    return m.cuda().train()


def grads_of(m, xb, tb):
    flat = FlatGrads(m.parameters())
    loss = T.BceFn.apply(m(xb), tb)
    loss.backward()
    assert flat.intact()
    return flat


sh = slice(rank * per, (rank + 1) * per)
flat = grads_of(model(True), x[sh], t[sh])
flat.all_reduce_mean()
ok = True
if rank == 0:
    ref_model = model(False)
    ref = grads_of(ref_model, x, t)
    err, off = 0.0, 0
    for p in ref_model.parameters():
        g, gr = flat.bucket[off:off + p.numel()], ref.bucket[off:off + p.numel()]
        off += p.numel()
        s = gr.abs().max().item()
        if s > 0:
            err = max(err, (g - gr).abs().max().item() / s)
    print(f"sync_bn_check: world={world} max over tensors of max |allreduced - single-process| / max|g| = {err:.3e}")
    ok = err <= 1e-3
m = model(True)
Trainer(m, lr=1e-4).step(x[sh], t[sh])
vec = torch.cat([v.detach().double().reshape(-1) for v in list(m.parameters()) + list(m.buffers())])
others = [torch.empty_like(vec) for _ in range(world)]
dist.all_gather(others, vec)
same = all(torch.equal(o, others[0]) for o in others)
if rank == 0:
    print("sync_bn_check: parameters and running statistics identical across ranks after one step:", same)

# ---- step time at batch `args.batch` per GPU, converted against unconverted, alternated ---------------------------------------
xb = torch.from_numpy(synth.randn_images(args.batch, 224, 224, 7 + rank)).cuda()
tb = torch.from_numpy(synth.random_masks(args.batch, 224, 224, 8 + rank)).cuda()
if rank == 0:
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(local)],
                         capture_output=True, text=True).stdout.strip()
    print(f"sync_bn_check: timing on {world} x {gpu}, batch {args.batch} per GPU, 224 x 224, {args.rounds} rounds x {args.steps} steps")
for storage in ("fp32", "bf16"):
    trainers = {c: Trainer(model(c), lr=1e-4, storage=storage) for c in (False, True)}
    for tr in trainers.values():                                   # warm-up: plans, workspaces, NCCL communicators
        for _ in range(2):
            tr.step(xb, tb)
    times = {False: [], True: []}
    for _ in range(args.rounds):
        for c in (False, True):
            torch.cuda.synchronize()
            dist.barrier()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                trainers[c].step(xb, tb)
            torch.cuda.synchronize()
            times[c].append((time.perf_counter() - t0) / args.steps * 1e3)
    if rank == 0:
        med = {c: statistics.median(v) for c, v in times.items()}
        print(f"sync_bn_check: {storage}: unconverted {med[False]:.1f} ms/step (rounds {min(times[False]):.1f}-{max(times[False]):.1f}), "
              f"SyncBatchNorm {med[True]:.1f} ms/step (rounds {min(times[True]):.1f}-{max(times[True]):.1f}), "
              f"overhead {100 * (med[True] / med[False] - 1):+.1f} %")
    del trainers
    torch.cuda.empty_cache()
if rank == 0:
    print("sync_bn_check:", "PASS" if (ok and same) else "FAIL")
dist.destroy_process_group()
sys.exit(0 if (ok and same) else 1)
