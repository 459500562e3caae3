"""Error bounds of the bf16-storage entry points (`csnet_train_*_bf16`, include/csnet_b200.h), on top of tests/trainref.py.

A bf16-storage kernel computes exactly what its fp32 twin computes — the same fp32 accumulation, in the same order, on the
values it read (bf16 inputs widen to fp32 exactly) — and then rounds each output it stores in bf16 to nearest even.  So for
such an output, with trainref's float64 reference r and fp32 bound b evaluated on the kernel's own bf16 inputs:

    |got - r| <= |fp32 value - r| + |rn_bf16(fp32 value) - fp32 value| <= b + 2^-8 (|r| + b) + 2^-134

2^-8 is the unit roundoff of bf16's 8-bit significand and 2^-134 half its smallest subnormal.  Outputs stored in fp32
(weight gradients, BatchNorm statistics and parameter gradients, the per-image channel means, an fp32 destination) keep b.
"""
from __future__ import annotations

import torch

U_BF16 = 2.0 ** -8
TINY_BF16 = 2.0 ** -134

# the outputs of each kernel-test case kind that the bf16 entry points store in bf16 (with bf16 activations on both sides)
BF16_OUTPUTS = {
    "mix": ("dst", "dsrc"),            # dsrc0, dsrc1, ...: prefixes
    "dw": ("y", "dxT", "bwd_dx"),
    "bn": ("y", "dz"),                 # dz0, dz1
    "pool": ("dst", "dsrc"),
}
# the activation inputs of each case kind (rounded to bf16 for the bf16 cases)
BF16_INPUTS = {"mix": ("srcs", "ddst"), "dw": ("x", "dy"), "bn": ("z", "dy"), "pool": ("src", "dpool")}


def widen(ref: torch.Tensor, bound: torch.Tensor) -> torch.Tensor:
    """The bound of an output stored in bf16 (round to nearest even) whose fp32 value is within `bound` of `ref`."""
    return bound * (1.0 + U_BF16) + U_BF16 * ref.abs() + TINY_BF16


def round_bf16(t: torch.Tensor) -> torch.Tensor:
    """fp32 values rounded to the nearest bf16 (ties to even), returned as fp32."""
    return t.float().to(torch.bfloat16).float()


def truncate_bf16(t: torch.Tensor) -> torch.Tensor:
    """fp32 values with their low 16 bits cleared: bf16 by truncation, the rounding a kernel must not use."""
    return (t.float().contiguous().view(torch.int32) & -65536).view(torch.float32)


def bf16_inputs(kind: str, inp: dict, sides=("srcs", "ddst")) -> dict:
    """A kernel-test case's inputs with its activations rounded to bf16 (`sides` picks a mix's bf16 operands: sources,
    destination gradient or both)."""
    out = dict(inp)
    names = BF16_INPUTS.get(kind, ())
    for name in names:
        if kind == "mix" and name not in sides:
            continue
        v = inp[name]
        out[name] = [round_bf16(t) for t in v] if isinstance(v, list) else round_bf16(v)
    return out


def stored_bf16(kind: str, name: str, bf16_dst=True, bf16_src=True) -> bool:
    """Whether output `name` of a case of `kind` is stored in bf16; for a mix, dst follows the destination's dtype and the
    data gradients the sources'."""
    if kind == "mix":
        return bf16_dst if name == "dst" else (bf16_src if name.startswith("dsrc") else False)
    return any(name.startswith(p) for p in BF16_OUTPUTS.get(kind, ()))


def widen_refs(kind: str, refs: dict, bf16_dst=True, bf16_src=True) -> dict:
    """trainref's {name: (ref, bound)} with the bounds of the bf16-stored outputs widened."""
    out = {}
    for name, rb in refs.items():
        if name != "idx" and stored_bf16(kind, name, bf16_dst, bf16_src):
            out[name] = (rb[0], widen(rb[0], rb[1]))
        else:
            out[name] = rb
    return out
