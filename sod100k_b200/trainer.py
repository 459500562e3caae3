"""One reference training step (CSNet_training/train.py:203-216) on the engine's kernels:
train-mode forward -> mean BCE-with-logits (+ WEIGHT * get_flops()) -> backward -> [DP: one all-reduce of the single
flat gradient bucket] -> Adam in the reference's two weight-decay groups (train.py:97-123).

Data parallelism (SURVEY.md §8e): one process per GPU; the gradients travel in the all-reduce(sum)/world of ONE flat fp32
bucket holding every gradient (140 894 floats for csnet-L-x2) — every `p.grad` is a view into that bucket, so there is no
flatten / unflatten copy.  BatchNorm statistics are each rank's own unless the model was converted with
`nn.SyncBatchNorm.convert_sync_batchnorm(model, group)`: then every train-mode BatchNorm normalises by the statistics of the
group's whole batch, with one small float64 all-reduce per BatchNorm call in each direction (train_ops.SyncBnPreluFn, DESIGN
§5.1), so a G-GPU step at global batch B computes the step one GPU computes at batch B.  The dynamic-weight-decay term stays per
rank (each rank's own activations); the bucket's mean averages it.
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Tuple

import torch

from . import train_ops as T


def reference_param_groups(model) -> Tuple[List[torch.nn.Parameter], List[torch.nn.Parameter]]:
    """(normal, zero-weight-decay) exactly as train.py:101-105 picks them — including its repeated
    'conv3x3_1.bns' test (conv3x3_2's BN gammas stay in the decayed group)."""
    normal, picked = [], []
    for name, p in model.named_parameters():
        if not p.requires_grad:                  # frozen parameters take no optimizer step (no zero grads, no weight decay)
            continue
        if "stage" in name and ("conv1x1.bns" in name or "conv3x3_1.bns" in name or "conv3x3_1.bns" in name) and "weight" in name:
            picked.append(p)
        else:
            normal.append(p)
    return normal, picked


class FlatGrads:
    """All gradients of `params` as views of one contiguous fp32 bucket."""

    def __init__(self, params: Iterable[torch.nn.Parameter]):
        self.params = [p for p in params if p.requires_grad]
        total = sum(p.numel() for p in self.params)
        self.bucket = torch.zeros(total, dtype=torch.float32, device=self.params[0].device)
        off = 0
        for p in self.params:
            p.grad = self.bucket[off:off + p.numel()].view_as(p)
            off += p.numel()

    def zero(self):
        self.bucket.zero_()

    def intact(self) -> bool:
        """autograd must have accumulated in place (the views still alias the bucket)."""
        base = self.bucket.data_ptr()
        off = 0
        for p in self.params:
            if p.grad is None or p.grad.data_ptr() != base + 4 * off:
                return False
            off += p.numel()
        return True

    def all_reduce_mean(self, group=None):
        import torch.distributed as dist

        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            dist.all_reduce(self.bucket, op=dist.ReduceOp.SUM, group=group)
            self.bucket.div_(dist.get_world_size(group))


class Trainer:
    def __init__(self, model, lr: float = 1e-4, weight_decay: float = 5e-3, betas=(0.9, 0.99), eps: float = 1e-8,
                 flops_weight: Optional[float] = None, flops_expand: float = 1.0, process_group=None, recompute: bool = False,
                 storage: str = "fp32"):
        if storage not in T.STORAGES:
            raise ValueError(f"storage must be one of {sorted(T.STORAGES)}, got {storage!r}")
        self.model = model
        model.recompute = bool(recompute)        # modular.csnet_forward: checkpoint every ILBlock (memory for one extra forward)
        model.train_storage = storage            # modular.csnet_forward: activation storage, "fp32" or "bf16" (DESIGN.md §6)
        self.flops_weight = flops_weight
        self.group = process_group
        if flops_weight is not None:
            model.flops_hook(expandflop=flops_expand)
        self.flat = FlatGrads(model.parameters())
        normal, picked = reference_param_groups(model)
        self.opt = T.FusedAdam([(normal, weight_decay), (picked, 0.0)], lr=lr, betas=betas, eps=eps)

    def step_host(self, x_host: torch.Tensor, target_host: torch.Tensor) -> torch.Tensor:
        """`step` fed from (pinned) host tensors: the batch is copied into one of two device staging slots on a copy stream, so —
        as nothing in the step syncs with the host — the copy of call k+1 runs under the kernels of call k (what a DataLoader with
        pin_memory and non_blocking copies gives `train.py:197-203`).  Returns the loss as a device tensor; read it a step late
        (or not every step) to keep the overlap."""
        dev = next(self.model.parameters()).device
        if not hasattr(self, "_feed"):
            self._feed = {"stream": torch.cuda.Stream(dev), "slots": [None, None], "free": [None, None], "k": 0}
        f = self._feed
        k = f["k"] = f["k"] ^ 1
        main = torch.cuda.current_stream(dev)
        with torch.cuda.stream(f["stream"]):
            if f["free"][k] is not None:
                f["stream"].wait_event(f["free"][k])          # the step that last read this slot has finished
            slot = f["slots"][k]
            if slot is None or slot[0].shape != x_host.shape or slot[1].shape != target_host.shape:
                slot = f["slots"][k] = (torch.empty(x_host.shape, dtype=torch.float32, device=dev),
                                        torch.empty(target_host.shape, dtype=torch.float32, device=dev))
            slot[0].copy_(x_host, non_blocking=True)
            slot[1].copy_(target_host, non_blocking=True)
            ready = torch.cuda.Event()
            ready.record(f["stream"])
        main.wait_event(ready)
        loss = self.step(slot[0], slot[1])
        f["free"][k] = torch.cuda.Event()
        f["free"][k].record(main)
        return loss

    def step(self, x: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        """Returns the BCE loss (without the regulariser), like `losses.update(loss.item())` at train.py:211 —
        as a device tensor: no host sync inside the step."""
        m = self.model
        m.train()
        self.flat.zero()
        if self.flops_weight is not None:
            m.clear_flops()
            m.set_batchsize(x.shape[0])
        out = m(x)
        loss = T.BceFn.apply(out, target)
        total = loss if self.flops_weight is None else loss + self.flops_weight * m.get_flops()
        total.backward()
        if not self.flat.intact():
            raise T.runtime.EngineError("gradient views were replaced; the flat bucket is stale")
        self.flat.all_reduce_mean(self.group)
        self.opt.step()
        return loss.detach()


class CSFSchedule:
    """solver.train's bookkeeping (CSF+Res2Net/solver.py:81-127): `aveGrad` counts micro-steps across epochs and every iter_size-th
    one takes an Adam step; after epoch e in lr_decay_epochs, lr is multiplied by 0.1 and a new Adam (zero moments, step 0) is built.
    The epoch-start net.zero_grad() discards a partial accumulation but keeps the count, so an epoch's first Adam step can sum fewer
    than iter_size micro-steps."""

    def __init__(self, iter_size: int, lr: float, lr_decay_epochs=(15,)):
        if int(iter_size) < 1:
            raise ValueError(f"iter_size must be >= 1, got {iter_size}")
        self.iter_size, self.lr, self.decay = int(iter_size), float(lr), frozenset(int(e) for e in lr_decay_epochs)
        self.count = 0

    def micro_step(self) -> bool:
        """Count one micro-step; True when it ends with an Adam step."""
        self.count += 1
        if self.count % self.iter_size == 0:
            self.count = 0
            return True
        return False

    def epoch_end(self, epoch: int) -> bool:
        """True when epoch `epoch` decays lr (and the optimiser is rebuilt)."""
        if epoch in self.decay:
            self.lr *= 0.1
            return True
        return False


class CSFTrainer:
    """CSF+Res2Net/solver.py:train's step on the device: forward on the module's training path in eval mode (frozen BatchNorm, as
    solver.py:49 keeps the net), BCE summed over the batch / (iter_size * batch_size) (BceSumFn, no host sync), backward into one flat
    gradient bucket (FlatGrads), and every iter_size-th micro-step one FusedAdam launch (torch.optim.Adam with L2 weight decay, betas
    (0.9, 0.999), eps 1e-8) over the trainable parameters, then a zeroed bucket.  `storage` sets net.train_storage: "fp32" (default)
    or "bf16" (bf16 activations, the backbone under autocast, the head's convolutions on tensor cores; DESIGN.md §7.3).  set_precision
    applies to inference only.

        trainer = CSFTrainer(net, iter_size=10)
        for epoch in range(epochs):
            trainer.epoch_begin()
            rng = random.Random(base_seed)                    # the reference's per-epoch worker seed
            for i in torch.randperm(len(ds)).tolist():
                loss = trainer.step(*ds.csf_train_batch([i], rng))
            trainer.epoch_end(epoch)

    Gradients live in the bucket: a net.zero_grad() (or anything else that replaces p.grad) makes the next step raise EngineError."""

    def __init__(self, net, lr: float = 5e-5, weight_decay: float = 5e-4, iter_size: int = 10, lr_decay_epochs=(15,),
                 batch_size: int = 1, storage: str = "fp32"):
        if int(batch_size) < 1:
            raise ValueError(f"batch_size must be >= 1, got {batch_size}")
        if storage not in T.STORAGES:
            raise ValueError(f"storage must be one of {sorted(T.STORAGES)}, got {storage!r}")
        self.net = net
        net.train_storage = storage
        self.schedule = CSFSchedule(iter_size, lr, lr_decay_epochs)
        self.divisor = self.schedule.iter_size * int(batch_size)
        self.weight_decay = float(weight_decay)
        self.flat = FlatGrads(net.parameters())
        self.opt = self._adam()

    def _adam(self) -> T.FusedAdam:
        return T.FusedAdam([(self.flat.params, self.weight_decay)], lr=self.schedule.lr, betas=(0.9, 0.999), eps=1e-8)

    def _check_bucket(self):
        if not self.flat.intact():
            raise T.runtime.EngineError("gradient views were replaced (net.zero_grad()?); the flat bucket is stale — use "
                                        "CSFTrainer.epoch_begin() to discard gradients")

    def epoch_begin(self):
        """The epoch-start net.zero_grad(): discards a partial accumulation, keeps the micro-step count."""
        self._check_bucket()
        self.flat.zero()

    def step(self, x: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        """One micro-step on CUDA fp32 x [N,3,H,W] and target [N,1,H,W]; returns its loss (sum-BCE / divisor) as a device tensor."""
        self._check_bucket()
        if self.net.training:                          # eval() walks every sub-module: about 1 ms of host time a step
            self.net.eval()
        with torch.enable_grad():
            out = self.net(x)
            loss = T.BceSumFn.apply(out, target, self.divisor)
            loss.backward()
        self._check_bucket()
        if self.schedule.micro_step():
            self.opt.step()
            self.flat.zero()
        return loss.detach()

    def epoch_end(self, epoch: int):
        """Learning-rate decay after epoch `epoch` in lr_decay_epochs, with fresh Adam state."""
        if self.schedule.epoch_end(epoch):
            self.opt = self._adam()
