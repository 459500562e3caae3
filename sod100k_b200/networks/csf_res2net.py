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
    fp32 training kernels (csnet_train_conv_* / _gn_* / _resize_*), so solver.py's train loop runs unchanged.
"""
from __future__ import annotations

import math
from collections import OrderedDict

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
        self._plans = OrderedDict()              # (h, w, precision, device) -> head plan, least recently used first
        self._plan_version = {}
        self.plan_budget = PLAN_BUDGET

    def set_precision(self, dtype: str):
        self.precision = dtype
        return self

    def __getstate__(self):                      # device plans (ctypes handles) never travel with a copy / pickle
        d = dict(self.__dict__)
        d["_plans"], d["_plan_version"] = OrderedDict(), {}
        return d

    def __deepcopy__(self, memo):
        import copy

        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k not in ("_plans", "_plan_version"):
                new.__dict__[k] = copy.deepcopy(v, memo)
        new._plans, new._plan_version = OrderedDict(), {}
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
            # training (CSF+Res2Net/solver.py:train): the backbone on torch autograd (cuDNN, fp32), the head on our fp32 training kernels
            # (modular_r), logits with a grad_fn at the input's size
            from .. import modular_r

            return modular_r.csf_head(self, self.base(x.float()), x.shape[2:])
        if self.training:
            raise NotImplementedError("CSF+Res2Net runs inference under model.eval() and torch.no_grad(), and trains with autograd "
                                      "recording (grad enabled, parameters or input requiring grad)")
        n, _, h, w = x.shape
        # any (h, w): the head program resizes between the backbone's ceil(h / 2) stages as the reference does.  One plan per size
        # lives in an LRU cache whose arenas `plan_budget` bounds (the plan in use stays even when it alone exceeds the budget)
        feats = self.backbone(x.float())
        key = (h, w, self.precision, x.device.index or 0)
        plan = self._plans.get(key)
        # the head plan folds the head's parameters at creation: re-fold when they change (load_state_dict, weights_init,
        # `.data` writes — same version stamp as the CSNet engine), so head and backbone never run on different weights
        from ..engine import param_version, trim_plans

        ver = param_version([t for k, t in list(self.named_parameters()) + list(self.named_buffers()) if not k.startswith("base.")])
        if plan is None or plan.max_batch < n:
            prog = compiler_r.compile_csf_head(self.head_state(), [tuple(f.shape[1:]) for f in feats], h, w, self.precision)
            if plan is not None:
                plan.close()
            plan = self._plans[key] = runtime.Plan(prog, max_batch=n, device=key[3])
        elif self._plan_version.get(key) != ver:
            prog = compiler_r.compile_csf_head(self.head_state(), [tuple(f.shape[1:]) for f in feats], h, w, self.precision)
            if prog.signature() == plan.prog.signature():
                plan.set_blob(prog.blob, torch.cuda.current_stream(x.device).cuda_stream)
                plan.prog = prog
            else:
                mb = plan.max_batch
                plan.close()
                plan = self._plans[key] = runtime.Plan(prog, max_batch=mb, device=key[3])
        self._plan_version[key] = ver
        self._plans.move_to_end(key)
        trim_plans(self._plans, self.plan_budget, self._plan_version, keep=key)
        y = torch.empty((n, 1, h, w), dtype=torch.float32, device=x.device)
        plan.run(n, [f.data_ptr() for f in feats] + [y.data_ptr()], torch.cuda.current_stream(x.device).cuda_stream)
        return y


def build_model():
    return CSFNet()


def weights_init(m):
    if isinstance(m, nn.Conv2d):
        m.weight.data.normal_(0, 0.01)
        if m.bias is not None:
            m.bias.data.zero_()
