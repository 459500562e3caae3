"""Per-model engine state: compiled programs and device plans, keyed by input size / precision, refreshed
when parameters change.  This is the host logic between the `nn.Module` surface and the C ABI."""
from __future__ import annotations

import os
from typing import Dict, Tuple

import torch

from . import compiler, ir, runtime


def _has_hooks(model) -> bool:
    """True if any descendant carries a forward (pre-)hook: those callers expect sub-module __call__s."""
    for m in model.modules():
        if m is model:
            continue
        if m._forward_hooks or m._forward_pre_hooks:
            return True
    return False


_PROBES = {}


def param_version(tensors, epoch: int = 0, owner=None) -> int:
    """Version stamp of a parameter set: torch's in-place counters and storage addresses (cheap, catches optimizer steps,
    load_state_dict, .to()) PLUS a value checksum computed on the device — writes through `.data` (`m.weight.data.normal_()`,
    pruning masks `w.data.mul_(mask)`, manual BN-statistic edits) do not bump `_version`, and the reference's own callers
    use them (weights_init, finetune).  The checksum is the dot product of all floating-point values with a fixed
    pseudo-random probe vector: one concatenation + one dot + one scalar read per call; `freeze()` skips it."""
    h = runtime.PARAM_EPOCH * 1000003 + epoch
    fl = []
    for t in tensors:
        h = (h * 1000003 + t._version * 31 + t.data_ptr()) & 0xFFFFFFFFFFFF
        if t.is_floating_point() and t.numel() > 0 and t.is_cuda:
            fl.append(t.detach().reshape(-1).float())
    if fl:
        flat = torch.cat(fl)
        key = (flat.numel(), flat.device)
        probe = _PROBES.get(key)
        if probe is None:
            g = torch.Generator(device="cpu").manual_seed(0x5EED)
            probe = _PROBES[key] = (torch.rand(flat.numel(), generator=g) + 0.5).to(flat.device)
        c = torch.stack([torch.dot(flat, probe), flat.abs().sum()]).tolist()
        h = (h * 1000003 + hash((c[0], c[1]))) & 0xFFFFFFFFFFFF
    return h


class ModelEngine:
    def __init__(self, model):
        self.model = model
        self.dtype = os.environ.get("CSNET_B200_DTYPE", "fp32")
        self._plans: Dict[Tuple, runtime.Plan] = {}
        self._plan_version: Dict[Tuple, int] = {}
        self.frozen = False
        self._epoch = 0

    def set_precision(self, dtype: str):
        if dtype not in ir.DTYPE_NAMES:
            raise ValueError(f"unknown precision {dtype!r}")
        self.dtype = dtype

    def freeze(self, flag: bool = True):
        """Skip the per-call parameter-version scan (weights will not change; latency-critical serving)."""
        self.frozen = flag

    def invalidate(self):
        """Force the next forward to re-fold the parameters (after writes the automatic checks cannot see)."""
        self._epoch += 1

    def _version(self) -> int:
        return param_version(list(self.model.parameters()) + list(self.model.buffers()), self._epoch, self)

    def _state(self):
        return {k: v.detach().cpu() for k, v in self.model.state_dict().items()}

    def plan_for(self, N: int, H: int, W: int, device: torch.device) -> runtime.Plan:
        key = (H, W, self.dtype, device.index or 0)
        plan = self._plans.get(key)
        if plan is not None and self.frozen and plan.max_batch >= N:
            return plan
        ver = self._version()
        if plan is None or plan.max_batch < N:
            prog = compiler.compile_csnet(self.model.layer_config, self._state(), H, W, self.dtype)
            if plan is not None:
                plan.close()
            plan = runtime.Plan(prog, max_batch=N, device=key[3])
            self._plans[key] = plan
        elif self._plan_version.get(key) != ver:
            prog = compiler.compile_csnet(self.model.layer_config, self._state(), H, W, self.dtype)
            if prog.signature() == plan.prog.signature():
                plan.set_blob(prog.blob, torch.cuda.current_stream(device).cuda_stream)
                plan.prog = prog
            else:
                # new weights changed the program itself (a 16-bit overflow veto, a fused block falling back, ...): the kernel
                # choices frozen at plan creation no longer fit -> rebuild the plan
                max_batch = plan.max_batch
                plan.close()
                plan = runtime.Plan(prog, max_batch=max_batch, device=key[3])
                self._plans[key] = plan
        self._plan_version[key] = ver
        return plan

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"expected input [N,3,H,W], got {tuple(x.shape)}")
        if not x.is_cuda:
            raise runtime.EngineError("CSNet (CUDA engine) needs a CUDA input; call model.cuda() / input.cuda() "
                                      "as the reference's test.py does — there is no CPU path")
        if self.model.training:
            from . import modular

            return modular.csnet_forward(self.model, x)
        needs_graph = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.model.parameters()))
        if _has_hooks(self.model) or (needs_graph and getattr(self.model, "frozen_bn_training", False)):
            # sub-module hooks, or training with the net kept in eval mode (frozen BatchNorm, as CSF+Res2Net/solver.py
            # does): run module by module so hooks fire and autograd sees every piece
            from . import modular

            return modular.csnet_forward(self.model, x)
        N, _, H, W = x.shape
        return self.plan_for(N, H, W, x.device).forward(x)

    def forward_host(self, x_host: torch.Tensor, out: torch.Tensor = None, device: int = 0) -> torch.Tensor:
        """End-to-end call on HOST tensors (float32 [N,3,H,W], ideally pinned): H2D, program, D2H, synchronised.
        Mirrors CSNet/test.py:86-93 (`.cuda()` ... `.cpu()`) in one C-ABI call."""
        if x_host.is_cuda or x_host.dtype != torch.float32:
            raise ValueError("forward_host takes a float32 host tensor")
        x_host = x_host.contiguous()
        N, _, H, W = x_host.shape
        dev = torch.device("cuda", device)
        plan = self.plan_for(N, H, W, dev)
        if out is None:
            out = torch.empty((N, 1, H, W), dtype=torch.float32, pin_memory=True)
        plan.run_host(N, x_host.data_ptr(), out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
        return out

    IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)          # CSNet/test.py:68-69

    def forward_host_u8(self, x_u8: torch.Tensor, out: torch.Tensor = None, device: int = 0, mean=IMAGENET_MEAN, std=IMAGENET_STD) -> torch.Tensor:
        """uint8 images in, uint8 saliency maps out, host to host (CSNet/test.py:72-98 without its resizes): x_u8 is [N,H,W,3] uint8
        (ideally pinned) as io.imread returns it; normalisation, the network, sigmoid and the *255 quantisation run on the device."""
        if x_u8.is_cuda or x_u8.dtype != torch.uint8 or x_u8.dim() != 4 or x_u8.shape[-1] != 3:
            raise ValueError("forward_host_u8 takes a uint8 host tensor [N, H, W, 3]")
        x_u8 = x_u8.contiguous()
        N, H, W, _ = x_u8.shape
        dev = torch.device("cuda", device)
        plan = self.plan_for(N, H, W, dev)
        if out is None:
            out = torch.empty((N, H, W), dtype=torch.uint8, pin_memory=True)
        plan.run_host_u8(N, x_u8.data_ptr(), out.data_ptr(), mean, std, torch.cuda.current_stream(dev).cuda_stream)
        return out
