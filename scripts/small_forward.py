"""Tiny forwards for compute-sanitizer runs: fp32 generic path, fp16 / bf16 fused path at two sizes (boundary tiles only and
interior + boundary tiles), the pipelined host call, and the device SalMetric."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from sod100k_b200 import checkpoints, synth, salmetric
for tag, dt, hw in (("csnet-L-x2", "fp32", (64, 96)), ("csnet-L-x1", "fp16", (64, 96)), ("csnet-L-x2", "fp16", (224, 224)),
                    ("csnet-L-x2", "bf16", (96, 160))):
    m, cfg, sd = checkpoints.build_from_npz(tag)
    m.cuda().eval().set_precision(dt)
    with torch.no_grad():
        y = m(torch.from_numpy(synth.randn_images(2, hw[0], hw[1], 5)).cuda())
    torch.cuda.synchronize()
    print(tag, dt, hw, float(y.mean()))
# 12 images at 224 x 224: enough row chunks for the streaming TMA / wgmma kernels (il_stream, mix_stream) to be selected
m, cfg, sd = checkpoints.build_from_npz("csnet-L-x2")
m.cuda().eval().set_precision("fp16")
with torch.no_grad():
    y = m(torch.from_numpy(synth.randn_images(12, 224, 224, 7)).cuda())
    y8 = m.engine().forward_host_u8(torch.randint(0, 256, (12, 224, 224, 3), dtype=torch.uint8))
torch.cuda.synchronize()
print("streaming", float(y.mean()), int(y8.sum()))
with torch.no_grad():
    x = torch.from_numpy(synth.randn_images(70, 64, 64, 6)).pin_memory()
    y = m.engine().forward_host(x)
torch.cuda.synchronize()
sm = salmetric.SalMetric()
sm.update(torch.rand(3, 1, 40, 56, device="cuda"), (torch.rand(3, 1, 40, 56, device="cuda") > 0.5).to(torch.uint8) * 255)
print("salmetric", sm.compute()["max_f"])
