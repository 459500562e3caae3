"""Per-op times of the fp16 bs-256 program (streaming ILBlock kernel on)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from sod100k_b200 import compiler, runtime, synth, checkpoints
batch = int(sys.argv[1]) if len(sys.argv) > 1 else 256
cfg, sd = checkpoints.load_npz("csnet-L-x2")
sd = {k: torch.from_numpy(v) for k, v in sd.items()}
x = torch.from_numpy(synth.randn_images(8, 224, 224, 7)).cuda().repeat(batch // 8, 1, 1, 1)
prog = compiler.compile_csnet(cfg, sd, 224, 224, "fp16")
p = runtime.Plan(prog, max_batch=batch)
y = torch.empty((batch, 1, 224, 224), dtype=torch.float32, device="cuda")
st = torch.cuda.current_stream().cuda_stream
for _ in range(3):
    p.run(batch, [x.data_ptr(), y.data_ptr()], st)
torch.cuda.synchronize()
ms = np.median(np.array([p.profile(batch, [x.data_ptr(), y.data_ptr()], st) for _ in range(5)]), axis=0)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(10):
    p.run(batch, [x.data_ptr(), y.data_ptr()], st)
e1.record(); torch.cuda.synchronize()
step = e0.elapsed_time(e1) / 10
print(f"step {step:.3f} ms = {batch / step * 1e3:.0f} img/s; sum of ops {ms.sum():.3f}")
for o, t in sorted(zip(prog.ops, ms), key=lambda ot: -ot[1])[:int(os.environ.get("TOP", "24"))]:
    print(f"   {o.name:34s} kind {o.kind} {t:.3f} ms")
