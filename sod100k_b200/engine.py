"""Per-model engine state: compiled programs and device plans, keyed by input size / precision, refreshed
when parameters change.  This is the host logic between the `nn.Module` surface and the C ABI."""
from __future__ import annotations

import os
from collections import OrderedDict
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
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

NATIVE_PLAN_BUDGET = 2 << 30        # bytes of arena the native-size plans of one engine may keep resident between calls


def native_size(h: int, w: int) -> Tuple[int, int]:
    """The network input of an h x w image when CSNet/test.py runs with TEST.IMAGE_H = 0 (test.py:75-84): the image itself when h and
    w are multiples of 16, else resized to (ceil(h / 16) * 16, ceil(w / 16) * 16)."""
    if h % 16 or w % 16:
        return (h + 15) // 16 * 16, (w + 15) // 16 * 16
    return h, w


def image_runs(sizes: Sequence, size: Optional[Tuple[int, int]], batch: Optional[int]):
    """How forward_images_u8 and SalImages.evaluate cut a set of (h, w) images into network runs.  Returns (order, runs): `order` lists
    the images in run order, and each run (a, b, H, W) takes order[a:b] at the network size H x W.  size=(H, W) keeps the input order
    and runs everything at that size; size=None groups the images by native_size, in ascending padded size so that one pass meets each
    size once.  No run holds more than `batch` images (None: no limit)."""
    if batch is not None and int(batch) < 1:
        raise ValueError(f"batch must be at least 1, got {batch}")
    hw = [(int(h), int(w)) for h, w in sizes]
    net = [native_size(h, w) for h, w in hw] if size is None else [(int(size[0]), int(size[1]))] * len(hw)
    order = sorted(range(len(hw)), key=lambda i: net[i]) if size is None else list(range(len(hw)))
    step = len(hw) if batch is None else int(batch)
    runs: List[Tuple[int, int, int, int]] = []
    a = 0
    while a < len(order):
        H, W = net[order[a]]
        b = a
        while b < len(order) and b - a < step and net[order[b]] == (H, W):
            b += 1
        runs.append((a, b, H, W))
        a = b
    return order, runs


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


def trim_plans(plans: "OrderedDict[Tuple, runtime.Plan]", budget: int, versions: Dict[Tuple, int], keep: Optional[Tuple] = None) -> None:
    """Close plans of an LRU cache (least recently used first; keys (H, W, dtype, device, ...)) until their arenas
    (csnet_plan_arena_bytes) fit `budget` bytes, dropping their parameter versions too.  The plan of key `keep`, if given, stays."""
    total = sum(p.arena_bytes for p in plans.values())
    if total <= budget:
        return
    for dev in {k[3] for k in plans}:
        torch.cuda.synchronize(dev)                      # work queued on a plan's arena or graphs ends before the plan goes
    for key in [k for k in plans if k != keep]:
        if total <= budget:
            break
        plan = plans.pop(key)
        total -= plan.arena_bytes
        versions.pop(key, None)
        plan.close()


class ModelEngine:
    def __init__(self, model):
        self.model = model
        self.dtype = os.environ.get("CSNET_B200_DTYPE", "fp32")
        self._plans: Dict[Tuple, runtime.Plan] = {}
        self._plan_version: Dict[Tuple, int] = {}
        self.frozen = False
        self._epoch = 0
        self._pinned_images = None          # forward_images_u8's packed host input, reused across calls
        self._native_plans: "OrderedDict[Tuple, runtime.Plan]" = OrderedDict()     # least recently used first
        self.native_plan_budget = NATIVE_PLAN_BUDGET

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
        return self._plan_in(self._plans, (H, W, self.dtype, device.index or 0), N)

    def _plan_in(self, plans: Dict[Tuple, runtime.Plan], key: Tuple, N: int) -> runtime.Plan:
        """The plan of `key` = (H, W, dtype, device, ...) in `plans` for a batch of N, created, refreshed after a parameter change,
        or rebuilt when N outgrows it."""
        H, W, dev = key[0], key[1], key[3]
        plan = plans.get(key)
        if plan is not None and self.frozen and plan.max_batch >= N:
            return plan
        ver = self._version()
        if plan is None or plan.max_batch < N:
            prog = compiler.compile_csnet(self.model.layer_config, self._state(), H, W, self.dtype)
            if plan is not None:
                plan.close()
            plan = runtime.Plan(prog, max_batch=N, device=dev)
            plans[key] = plan
        elif self._plan_version.get(key) != ver:
            prog = compiler.compile_csnet(self.model.layer_config, self._state(), H, W, self.dtype)
            if prog.signature() == plan.prog.signature():
                plan.set_blob(prog.blob, torch.cuda.current_stream(dev).cuda_stream)
                plan.prog = prog
            else:
                # new weights changed the program itself (a 16-bit overflow veto, a fused block falling back, ...): the kernel
                # choices frozen at plan creation no longer fit -> rebuild the plan
                max_batch = plan.max_batch
                plan.close()
                plan = runtime.Plan(prog, max_batch=max_batch, device=dev)
                plans[key] = plan
        self._plan_version[key] = ver
        return plan

    def native_plan(self, N: int, H: int, W: int, device: torch.device) -> runtime.Plan:
        """plan_for for the padded sizes of `forward_images_u8(size=None)`: these plans live in a cache of their own whose arenas
        `trim_native_plans` keeps within `native_plan_budget` bytes, so a test set of many image sizes does not keep one arena per
        size on the device.  The fixed-size plans of plan_for are not part of it."""
        key = (H, W, self.dtype, device.index or 0, "native")
        plan = self._plan_in(self._native_plans, key, N)
        self._native_plans.move_to_end(key)
        return plan

    def trim_native_plans(self) -> None:
        """Close native-size plans, least recently used first, until their arenas (csnet_plan_arena_bytes) fit the budget."""
        trim_plans(self._native_plans, self.native_plan_budget, self._plan_version)

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

    @staticmethod
    def _image_u8(im, i: int) -> torch.Tensor:
        if isinstance(im, np.ndarray):
            im = torch.from_numpy(np.ascontiguousarray(im))
        if not isinstance(im, torch.Tensor) or im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3:
            raise ValueError(f"image {i}: expected a uint8 [h, w, 3] array or tensor, got "
                             f"{getattr(im, 'dtype', type(im).__name__)} {tuple(getattr(im, 'shape', ()))}")
        if not (1 <= im.shape[0] <= 32767 and 1 <= im.shape[1] <= 32767):
            raise ValueError(f"image {i}: h and w must lie in [1, 32767], got {tuple(im.shape[:2])}")
        return im.contiguous()

    def forward_images_u8(self, images, size=(224, 224), device: int = 0, mean=IMAGENET_MEAN, std=IMAGENET_STD, batch: int = None):
        """CSNet/test.py:71-98 for a batch of images of any sizes, both skimage resizes included: each uint8 [h, w, 3] image is
        resized to its network size (skimage >= 0.19 `resize(..., mode='reflect', anti_aliasing=False)`), normalised, run through the
        network, and its sigmoid map resized back to (h, w) and quantised to uint8.  Returns the uint8 [h_i, w_i] maps in input order.

        size=(H, W) is test.py with TEST.IMAGE_H / IMAGE_W set: every image goes in at H x W.  size=None is TEST.IMAGE_H = 0: every
        image goes in at its own size, resized to native_size(h, w) (the next multiples of 16) only when h or w is not a multiple of
        16.  The images are then grouped by that size, one plan per size from a cache bounded by `native_plan_budget`.  No network
        run takes more than `batch` images (None: all images of one size in one run).

        `images` are numpy arrays or CPU tensors (the host path: packed into a pinned buffer that is reused across calls, one
        synchronised C call per run on plan `device`, the maps are views of one pinned buffer) or all CUDA tensors on one device (the
        device path: the resizes run around the network on the current stream, no host copies of pixels or maps)."""
        imgs = [self._image_u8(im, i) for i, im in enumerate(images)]
        if not imgs:
            return []
        if len({t.device for t in imgs}) > 1:
            raise ValueError("forward_images_u8 takes host images or CUDA images of one device, not a mix")
        order, runs = image_runs([t.shape[:2] for t in imgs], size, batch)
        imgs = [imgs[i] for i in order]
        geom = runtime.image_geometry([t.shape[:2] for t in imgs])
        hw = (geom["h"].astype(np.int64) * geom["w"]).tolist()
        total = sum(hw)
        if imgs[0].is_cuda:
            dev = imgs[0].device
            x = torch.cat([t.reshape(-1) for t in imgs])
            g = torch.from_numpy(geom.view(np.uint8)).to(dev)
            y = torch.empty(total, dtype=torch.uint8, device=dev)
            stream = torch.cuda.current_stream(dev).cuda_stream

            def store(logits, a, b, H, W, g_run):
                runtime.resize_logits_to_u8(logits.data_ptr(), b - a, H, W, g_run, y.data_ptr(), stream)

            self.run_packed_images(x, g, runs, size is None, mean, std, store)
        else:
            dev = torch.device("cuda", device)
            if self._pinned_images is None or self._pinned_images.numel() < 3 * total:
                self._pinned_images = torch.empty(3 * total, dtype=torch.uint8, pin_memory=True)
            x = self._pinned_images[:3 * total]
            torch.cat([t.reshape(-1) for t in imgs], out=x)
            y = torch.empty(total, dtype=torch.uint8, pin_memory=True)
            for k, (a, b, H, W) in enumerate(runs):
                plan = self.native_plan(b - a, H, W, dev) if size is None else self.plan_for(b - a, H, W, dev)
                g = geom[a:b].copy()
                base, n_px = int(g["dst_off"][0]), sum(hw[a:b])
                g["src_off"] -= 3 * base
                g["dst_off"] -= base
                plan.run_host_images_u8(b - a, x.data_ptr() + 3 * base, 3 * n_px, g, y.data_ptr() + base, n_px, mean, std,
                                        torch.cuda.current_stream(dev).cuda_stream)
                if size is None and (k + 1 == len(runs) or runs[k + 1][2:] != (H, W)):
                    self.trim_native_plans()
        offs = geom["dst_off"].tolist()
        maps = [None] * len(imgs)
        for i, o, n, t in zip(order, offs, hw, imgs):
            maps[i] = y[o:o + n].view(t.shape[0], t.shape[1])
        return maps

    def run_packed_images(self, x_packed: torch.Tensor, geom_dev: torch.Tensor, runs, native: bool, mean, std, consume) -> None:
        """The device side of forward_images_u8 for packed uint8 images on one device: for each run (a, b, H, W) of image_runs, entries
        a..b-1 of the device geometry table `geom_dev` are resized to H x W (csnet_resize_u8_to_input) and run through the plan of
        that size (native_plan when `native`, else plan_for), then consume(logits, a, b, H, W, geometry address of entry a) takes the
        logits, on the current stream.  Native-size plans are trimmed to the budget after each size."""
        dev = x_packed.device
        stream = torch.cuda.current_stream(dev).cuda_stream
        for k, (a, b, H, W) in enumerate(runs):
            n = b - a
            plan = self.native_plan(n, H, W, dev) if native else self.plan_for(n, H, W, dev)
            g = geom_dev.data_ptr() + a * runtime.GEOM_DTYPE.itemsize
            x_in = torch.empty((n, 3, H, W), dtype=torch.float32, device=dev)
            runtime.resize_u8_to_input(x_packed.data_ptr(), g, n, H, W, mean, std, x_in.data_ptr(), stream)
            consume(plan.forward(x_in), a, b, H, W, g)
            if native and (k + 1 == len(runs) or runs[k + 1][2:] != (H, W)):
                self.trim_native_plans()
