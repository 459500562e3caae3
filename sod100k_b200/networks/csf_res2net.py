"""`networks.csf_res2net` — the reference's CSF+Res2Net module surface (config 5) on the CUDA engine.

Same class / parameter names and `state_dict()` keys as /root/reference/CSF+Res2Net/networks/{csf_res2net,gOctConv}.py
so `solver.py` (`build_model()`, `net.base.load_pretrained_model`, `load_state_dict(strict=False)`) keeps working.
Split of the forward:
  * `base` (Res2Net-50 v1b 26w4s backbone, 11 of the 19 GMAC): ordinary torch modules — cuDNN LIBRARY calls, run under
    fp16 autocast when the plan is 16-bit.  Not the product; kept on the library as SURVEY.md §7 step 9 recommends until
    the CSF head meets its bar.
  * CSF head (`fuse` -> `ms` -> `fuse1x1` -> `cls_layer` -> bilinear to the input size): parameter containers lowered by compiler_r.py to one
    fused-op program on libcsnet_b200.so (GroupNorm variant).  No torch fallback for the head.
  * Training: when autograd records, the backbone runs on torch autograd and the head on modular_r.py's autograd Functions over the
    training kernels (csnet_train_conv_* / _gn_* / _resize_*, or their _bf16 twins with `train_storage = "bf16"`), so solver.py's
    train loop runs unchanged.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn
from torch.nn import init

from .. import compiler_r, runtime, splits


PLAN_BUDGET = 2 << 30        # bytes of arena the head plans of one CSFNet may keep resident between calls


class Bottle2neck(nn.Module):
    """Res2Net bottleneck: 1x1 -> `scale` width-groups, a hierarchical chain of 3x3 convs over scale-1 of them -> 1x1,
    residual.  'stage' blocks (first of a stage) do not chain and average-pool the pass-through group."""
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, dilation_=1, downsample=None, baseWidth=26, scale=4, stype="normal"):
        super().__init__()
        width = int(math.floor(planes * (baseWidth / 64.0)))
        self.conv1 = nn.Conv2d(inplanes, width * scale, kernel_size=1, bias=False)
        self.bn1 = nn.BatchNorm2d(width * scale)
        self.nums = 1 if scale == 1 else scale - 1
        if stype == "stage":
            self.pool = nn.AvgPool2d(kernel_size=3, stride=stride, padding=1)
        self.convs = nn.ModuleList([nn.Conv2d(width, width, kernel_size=3, stride=stride, dilation=dilation_,
                                              padding=dilation_, bias=False) for _ in range(self.nums)])
        self.bns = nn.ModuleList([nn.BatchNorm2d(width) for _ in range(self.nums)])
        self.conv3 = nn.Conv2d(width * scale, planes * self.expansion, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * self.expansion)
        self.relu = nn.ReLU(inplace=True)
        self.downsample, self.stype, self.scale, self.width = downsample, stype, scale, width
        for bn in [self.bn1, self.bn3, *self.bns]:          # the reference freezes every backbone BN affine
            for q in bn.parameters():
                q.requires_grad = False

    def forward(self, x):
        spx = torch.split(self.relu(self.bn1(self.conv1(x))), self.width, 1)
        outs, sp = [], None
        for i in range(self.nums):
            sp = spx[i] if (i == 0 or self.stype == "stage") else sp + spx[i]
            sp = self.relu(self.bns[i](self.convs[i](sp)))
            outs.append(sp)
        if self.scale != 1:
            outs.append(self.pool(spx[self.nums]) if self.stype == "stage" else spx[self.nums])
        out = self.bn3(self.conv3(torch.cat(outs, 1)))
        return self.relu(out + (x if self.downsample is None else self.downsample(x)))


class Res2Net(nn.Module):
    def __init__(self, block, layers, baseWidth=26, scale=4):
        super().__init__()
        self.inplanes, self.baseWidth, self.scale = 64, baseWidth, scale
        self.conv1 = nn.Sequential(nn.Conv2d(3, 32, 3, 2, 1, bias=False), nn.BatchNorm2d(32), nn.ReLU(inplace=True),
                                   nn.Conv2d(32, 32, 3, 1, 1, bias=False), nn.BatchNorm2d(32), nn.ReLU(inplace=True),
                                   nn.Conv2d(32, 64, 3, 1, 1, bias=False))
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.layer1 = self._make_layer(block, 64, layers[0])
        self.layer2 = self._make_layer(block, 128, layers[1], stride=2)
        self.layer3 = self._make_layer(block, 256, layers[2], stride=2)
        self.layer4 = self._make_layer(block, 512, layers[3], stride=2)
        self.avgpool = nn.AvgPool2d(7, stride=1)
        for q in self.bn1.parameters():
            q.requires_grad = False
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                init.constant_(m.weight, 1)
                init.constant_(m.bias, 0)

    def load_pretrained_model(self, model):
        self.load_state_dict(model, strict=False)

    def _make_layer(self, block, planes, blocks, stride=1, dilation__=1):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion or dilation__ in (2, 4):
            downsample = nn.Sequential(nn.AvgPool2d(kernel_size=stride, stride=stride, ceil_mode=True, count_include_pad=False),
                                       nn.Conv2d(self.inplanes, planes * block.expansion, kernel_size=1, stride=1, bias=False),
                                       nn.BatchNorm2d(planes * block.expansion))
            for q in downsample[1].parameters():
                q.requires_grad = False
        layers = [block(self.inplanes, planes, stride, dilation_=dilation__, downsample=downsample, stype="stage",
                        baseWidth=self.baseWidth, scale=self.scale)]
        self.inplanes = planes * block.expansion
        layers += [block(self.inplanes, planes, dilation_=dilation__, baseWidth=self.baseWidth, scale=self.scale)
                   for _ in range(1, blocks)]
        return nn.Sequential(*layers)

    def forward(self, x):
        x = self.maxpool(self.relu(self.bn1(self.conv1(x))))
        feats = []
        for layer in (self.layer1, self.layer2, self.layer3, self.layer4):
            x = layer(x)
            feats.append(x)
        return feats


class gOctaveConv(nn.Module):
    """Parameter container: one `weights` tensor [out_total, in_total, k, k] for all (in, out) branch pairs."""

    def __init__(self, in_channels, out_channels, kernel_size, alpha_in, alpha_out, stride=1, padding=0):
        super().__init__()
        self.in_channels, self.out_channels, self.stride, self.padding = in_channels, out_channels, stride, padding
        self.weights = nn.Parameter(torch.empty(out_channels, in_channels, *kernel_size))
        self.register_parameter("bias", None)
        self.h2g_pool = nn.AvgPool2d(kernel_size=(2, 2), stride=2)
        self.alpha_in, self.alpha_out = splits.cumulative(alpha_in), splits.cumulative(alpha_out)
        self.inbranch, self.outbranch = len(alpha_in), len(alpha_out)
        init.kaiming_uniform_(self.weights, a=math.sqrt(5))


class gOctaveCBR(nn.Module):
    """gOctConv + per-branch GroupNorm(32) + PReLU (parameter container)."""

    def __init__(self, in_channels, out_channels, kernel_size=(3, 3), alpha_in=(0.5, 0.5), alpha_out=(0.5, 0.5), stride=1, padding=1):
        super().__init__()
        self.in_channels, self.out_channels, self.std_conv = in_channels, out_channels, False
        self.conv = gOctaveConv(in_channels, out_channels, kernel_size, alpha_in, alpha_out, stride, padding)
        w = splits.widths(out_channels, alpha_out)
        self.bns = nn.ModuleList([nn.GroupNorm(32, c) for c in w])
        self.prelus = nn.ModuleList([nn.PReLU(c) for c in w])
        self.outbranch, self.alpha_in, self.alpha_out = len(alpha_out), list(alpha_in), list(alpha_out)


class MSBlock(nn.Module):
    def __init__(self, in_channels, out_channels, dilations=splits.DILATIONS):
        super().__init__()
        self.dilations = list(dilations)
        each = out_channels // 5
        outs = [each] * 4 + [out_channels - 4 * each]
        self.msconv = nn.ModuleList([nn.Conv2d(in_channels, o, 3, padding=d, dilation=d, bias=False) for o, d in zip(outs, self.dilations)])
        self.bn = nn.GroupNorm(32, out_channels)
        self.prelu = nn.PReLU(out_channels)


class PallMSBlock(nn.Module):
    def __init__(self, in_channels, out_channels, alpha=(0.5, 0.5), bias=False):
        super().__init__()
        self.std_conv = False
        self.convs = nn.ModuleList([MSBlock(int(round(in_channels * a)), int(round(out_channels * a))) for a in alpha])
        self.outbranch = len(alpha)


class CSFNet(nn.Module):
    def __init__(self, num_classes=1):
        super().__init__()
        self.base = Res2Net(Bottle2neck, [3, 4, 6, 3], baseWidth=26, scale=4)
        cin, cout = 256 + 512 + 1024 + 2048, 128 + 256 + 512 + 512
        self.fuse = gOctaveCBR(cin, cout, kernel_size=(1, 1), padding=0, alpha_in=compiler_r.FUSE_IN_SPLIT,
                               alpha_out=compiler_r.FUSE_OUT_SPLIT)
        self.ms = PallMSBlock(cout, cout, alpha=compiler_r.FUSE_OUT_SPLIT)
        self.fuse1x1 = gOctaveCBR(cout, cout, kernel_size=(1, 1), padding=0, alpha_in=compiler_r.FUSE_OUT_SPLIT, alpha_out=[1])
        self.cls_layer = nn.Conv2d(cout, num_classes, kernel_size=1)
        self.precision = "fp32"
        self.train_storage = "fp32"              # training activation storage, "fp32" or "bf16" (CSFTrainer(storage=...), DESIGN §7.3)
        self._plans = OrderedDict()              # (h, w, precision, device) -> head plan, least recently used first
        self._plan_version = {}
        self.plan_budget = PLAN_BUDGET
        self._pinned_images = None               # forward_images_u8's packed host input, reused across calls

    def set_precision(self, dtype: str):
        self.precision = dtype
        return self

    def __getstate__(self):                      # device plans (ctypes handles) never travel with a copy / pickle
        d = dict(self.__dict__)
        d["_plans"], d["_plan_version"], d["_pinned_images"] = OrderedDict(), {}, None
        return d

    def __deepcopy__(self, memo):
        import copy

        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k not in ("_plans", "_plan_version", "_pinned_images"):
                new.__dict__[k] = copy.deepcopy(v, memo)
        new._plans, new._plan_version, new._pinned_images = OrderedDict(), {}, None
        return new

    def head_state(self):
        return {k: v.detach().cpu() for k, v in self.state_dict().items() if not k.startswith("base.")}

    def backbone(self, x):
        if self.precision == "fp32":
            return [f.contiguous() for f in self.base(x)]
        dt = torch.float16 if self.precision == "fp16" else torch.bfloat16
        with torch.autocast("cuda", dtype=dt):
            return [f.to(dt).contiguous() for f in self.base(x)]

    def forward(self, x):
        if not x.is_cuda:
            raise runtime.EngineError("CSFNet (CUDA engine) needs CUDA tensors; there is no CPU path")
        if torch.is_grad_enabled() and (x.requires_grad or any(q.requires_grad for q in self.parameters())):
            # training (CSF+Res2Net/solver.py:train): the backbone on torch autograd (cuDNN), the head on our training kernels (modular_r),
            # logits with a grad_fn at the input's size.  train_storage "bf16": the backbone under bf16 autocast, its bf16 features
            # through the head's bf16 kernels; "fp32" (default): fp32 throughout.  set_precision does not apply to training.
            from .. import modular_r

            if modular_r.train_dtype(self) == torch.bfloat16:
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    feats = [f.to(torch.bfloat16).contiguous() for f in self.base(x.float())]
                return modular_r.csf_head(self, feats, x.shape[2:])
            return modular_r.csf_head(self, self.base(x.float()), x.shape[2:])
        self._check_inference()
        feats = self.backbone(x.float())
        return self._run_head(feats, x.shape, x.device, self._head_version())

    def _check_inference(self):
        if self.training:
            raise NotImplementedError("CSF+Res2Net runs inference under model.eval() and torch.no_grad(), and trains with autograd "
                                      "recording (grad enabled, parameters or input requiring grad)")

    def _head_version(self) -> int:
        """Version stamp of the head's parameters and buffers.  It reads a checksum back to the host, so a pass over many runs takes
        it once."""
        from ..engine import param_version

        return param_version([t for k, t in list(self.named_parameters()) + list(self.named_buffers()) if not k.startswith("base.")])

    def _run_head(self, feats, shape, device, ver: int) -> torch.Tensor:
        """The head on backbone features of a batch of input `shape` (n, 3, h, w): fp32 logits [n, 1, h, w] on the current stream."""
        n, _, h, w = shape
        # any (h, w): the head program resizes between the backbone's ceil(h / 2) stages as the reference does.  One plan per size
        # lives in an LRU cache whose arenas `plan_budget` bounds (the plan in use stays even when it alone exceeds the budget)
        key = (h, w, self.precision, device.index or 0)
        plan = self._plans.get(key)
        # the head plan folds the head's parameters at creation: re-fold when they change (load_state_dict, weights_init,
        # `.data` writes — same version stamp as the CSNet engine), so head and backbone never run on different weights
        from ..engine import trim_plans

        if plan is None or plan.max_batch < n:
            prog = compiler_r.compile_csf_head(self.head_state(), [tuple(f.shape[1:]) for f in feats], h, w, self.precision)
            if plan is not None:
                plan.close()
            plan = self._plans[key] = runtime.Plan(prog, max_batch=n, device=key[3])
        elif self._plan_version.get(key) != ver:
            prog = compiler_r.compile_csf_head(self.head_state(), [tuple(f.shape[1:]) for f in feats], h, w, self.precision)
            if prog.signature() == plan.prog.signature():
                plan.set_blob(prog.blob, torch.cuda.current_stream(device).cuda_stream)
                plan.prog = prog
            else:
                mb = plan.max_batch
                plan.close()
                plan = self._plans[key] = runtime.Plan(prog, max_batch=mb, device=key[3])
        self._plan_version[key] = ver
        self._plans.move_to_end(key)
        trim_plans(self._plans, self.plan_budget, self._plan_version, keep=key)
        y = torch.empty((n, 1, h, w), dtype=torch.float32, device=device)
        plan.run(n, [f.data_ptr() for f in feats] + [y.data_ptr()], torch.cuda.current_stream(device).cuda_stream)
        return y

    IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)          # CSF+Res2Net/dataset/dataset.py:load_image_test

    def run_packed_images(self, x_packed: torch.Tensor, geom_dev: torch.Tensor, runs, mean, std, consume) -> None:
        """The device side of forward_images_u8 and SalImages.evaluate: for each run (a, b, H, W) of image_runs(..., key=exact_size),
        the H x W images of entries a..b-1 of the device geometry table `geom_dev` become the network input (csnet_csf_input_u8), go
        through the backbone and the head as forward runs them, and consume(logits, a, b, H, W, geometry address of entry a) takes the
        fp32 logits [b - a, 1, H, W], on the current stream.  Runs under torch.no_grad(); a net in training mode raises."""
        self._check_inference()
        dev = x_packed.device
        stream = torch.cuda.current_stream(dev).cuda_stream
        with torch.no_grad():
            ver = self._head_version()
            for a, b, H, W in runs:
                n = b - a
                g = geom_dev.data_ptr() + a * runtime.GEOM_DTYPE.itemsize
                x = torch.empty((n, 3, H, W), dtype=torch.float32, device=dev)
                runtime.csf_input_u8(x_packed.data_ptr(), g, n, H, W, mean, std, x.data_ptr(), stream)
                consume(self._run_head(self.backbone(x), x.shape, dev, ver), a, b, H, W, g)

    @staticmethod
    def _image_u8(im, i: int) -> torch.Tensor:
        """One uint8 RGB [h, w, 3] image as a tensor; a gray [h, w] one is replicated to 3 channels (cv2.IMREAD_COLOR does)."""
        if isinstance(im, np.ndarray):
            im = torch.from_numpy(np.ascontiguousarray(im))
        if not isinstance(im, torch.Tensor) or im.dtype != torch.uint8 or not (im.dim() == 2 or (im.dim() == 3 and im.shape[2] == 3)):
            raise ValueError(f"image {i}: expected a uint8 [h, w, 3] or [h, w] array or tensor, got "
                             f"{getattr(im, 'dtype', type(im).__name__)} {tuple(getattr(im, 'shape', ()))}")
        if not (1 <= im.shape[0] <= 32767 and 1 <= im.shape[1] <= 32767):
            raise ValueError(f"image {i}: h and w must lie in [1, 32767], got {tuple(im.shape[:2])}")
        return im.unsqueeze(2).expand(-1, -1, 3) if im.dim() == 2 else im

    def forward_images_u8(self, images, batch: int = None, device: int = 0, mean=IMAGENET_MEAN, std=IMAGENET_STD):
        """CSF+Res2Net/solver.py:test for a list of images of any sizes: each RGB uint8 image goes in at its own size, normalised as
        dataset.load_image_test does, and its map is the uint8 [h, w] that solver.test writes with cv2.imwrite (255 * sigmoid, rounded
        half to even).  Returns the maps in input order.  Images are grouped by exact size (padding would change the maps); no run
        takes more than `batch` images (None: all images of one size in one run).

        `images` are uint8 [h, w, 3] or gray [h, w] numpy arrays or CPU tensors (packed into one pinned buffer reused across calls and
        copied to device `device` once; the maps are views of one pinned buffer), or all CUDA tensors on one device (the maps stay on
        that device)."""
        from ..engine import exact_size, image_runs

        imgs = [self._image_u8(im, i) for i, im in enumerate(images)]
        if not imgs:
            return []
        if len({t.device for t in imgs}) > 1:
            raise ValueError("forward_images_u8 takes host images or CUDA images of one device, not a mix")
        order, runs = image_runs([t.shape[:2] for t in imgs], None, batch, key=exact_size)
        imgs = [imgs[i] for i in order]
        geom = runtime.image_geometry([t.shape[:2] for t in imgs])
        hw = (geom["h"].astype(np.int64) * geom["w"]).tolist()
        total = sum(hw)
        host = not imgs[0].is_cuda
        dev = torch.device("cuda", device) if host else imgs[0].device
        if host:
            if self._pinned_images is None or self._pinned_images.numel() < 3 * total:
                self._pinned_images = torch.empty(3 * total, dtype=torch.uint8, pin_memory=True)
            x = self._pinned_images[:3 * total]
            torch.cat([t.reshape(-1) for t in imgs], out=x)
            x = x.to(dev, non_blocking=True)
        else:
            x = torch.cat([t.reshape(-1) for t in imgs])
        g = torch.from_numpy(geom.view(np.uint8)).pin_memory().to(dev, non_blocking=True)
        y = torch.empty(total, dtype=torch.uint8, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream

        def store(logits, a, b, H, W, g_run):
            runtime.csf_maps_u8(logits.data_ptr(), b - a, H, W, g_run, y.data_ptr(), stream)

        self.run_packed_images(x, g, runs, mean, std, store)
        if host:
            y = torch.empty(total, dtype=torch.uint8, pin_memory=True).copy_(y, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
        maps = [None] * len(imgs)
        for i, o, n, t in zip(order, geom["dst_off"].tolist(), hw, imgs):
            maps[i] = y[o:o + n].view(t.shape[0], t.shape[1])
        return maps


def build_model():
    return CSFNet()


def weights_init(m):
    if isinstance(m, nn.Conv2d):
        m.weight.data.normal_(0, 0.01)
        if m.bias is not None:
            m.bias.data.zero_()
