"""CSF+Res2Net bf16 training without a GPU: the tensor-core GEMM bound of tests/trainref_r_bf16.py holds for an emulated fp32
accumulation of bf16 products and keeps its power (a dropped k16 step and truncated weights are flagged), and the storage option is
validated."""
import pytest
import torch

from sod100k_b200 import modular_r
from sod100k_b200.networks import csf_res2net
from sod100k_b200.trainer import CSFTrainer
from tests import trainref_r_bf16 as B


def _q(got, ref_bound):
    ref, bound = ref_bound
    return float(((got.double() - ref).abs() / bound).max())


def _k16_sum(a: torch.Tensor, b: torch.Tensor, splits: int) -> torch.Tensor:
    """sum_k a[:, k] b[k, :] as the kernel orders it: fp32 partial sums of 16 products added to an fp32 accumulator per k16 step,
    S split partials merged in split order (a tensor core's rounding inside a k16 step is at least as fine as fp32's)."""
    K = a.shape[1]
    bounds = [(s * K) // splits for s in range(splits + 1)]
    out = None
    for s in range(splits):
        acc = torch.zeros(a.shape[0], b.shape[1], dtype=torch.float32)
        for k0 in range(bounds[s], bounds[s + 1], 16):
            k1 = min(k0 + 16, bounds[s + 1])
            acc = acc + (a[:, k0:k1] @ b[k0:k1])
        out = acc if out is None else out + acc
    return out


@pytest.mark.parametrize("K,splits", [(16, 1), (300, 1), (1152, 3), (3840, 8)])
def test_gemm_bound_covers_an_fp32_k16_accumulation(K, splits):
    g = torch.Generator().manual_seed(K)
    a = B.round_bf16(torch.randn(24, K, generator=g))
    b = B.round_bf16(torch.randn(K, 40, generator=g) * (1 + 100 * (torch.rand(K, 1, generator=g) < 0.01)))
    got = _k16_sum(a, b, splits)
    r = a.double() @ b.double()
    m = a.double().abs() @ b.double().abs()
    assert _q(got, (r, B.gemm_bound(m, K, splits))) <= 1.0
    assert _q(B.round_bf16(got), B.store(r, B.gemm_bound(m, K, splits), True)) <= 1.0


@pytest.mark.parametrize("k,dil,cin,cout,bf16_out", [(1, 1, 300, 40, False), (3, 2, 64, 27, False), (3, 1, 40, 25, True), (1, 1, 1792, 128, True)])
def test_conv_defects_exceed_the_bound(k, dil, cin, cout, bf16_out):
    """An fp32 CPU convolution of the bf16 operands passes the bound; a dropped k16 step always, and (fp32 destination) weights
    truncated instead of rounded, fail it."""
    g = torch.Generator().manual_seed(cin + k)
    x = B.round_bf16(torch.randn(1, cin, 9, 11, generator=g))
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    y = torch.nn.functional.conv2d(x, B.round_bf16(w), padding=dil if k == 3 else 0, dilation=dil)
    if bf16_out:
        y = B.round_bf16(y)
    seg = [(x, w, dil)]
    assert _q(y, B.conv_fwd(seg, splits=1, bf16_out=bf16_out)) <= 1.0
    assert _q(y, B.conv_fwd(seg, splits=1, bf16_out=bf16_out, defect="drop_k16")) > 1.0
    if not bf16_out:
        assert _q(y, B.conv_fwd(seg, splits=1, bf16_out=False, defect="truncated_w")) > 1.0
    dy = B.round_bf16(torch.randn(1, cout, 9, 11, generator=g))
    dx = torch.nn.functional.conv_transpose2d(dy, B.round_bf16(w), padding=dil if k == 3 else 0, dilation=dil)
    assert _q(dx, B.conv_dgrad([(dy, w, dil)], bf16_out=False)) <= 1.0
    assert _q(dx, B.conv_dgrad([(dy, w, dil)], bf16_out=False, defect="drop_k16")) > 1.0
    assert _q(dx, B.conv_dgrad([(dy, w, dil)], bf16_out=False, defect="truncated_w")) > 1.0
    dw = torch.nn.grad.conv2d_weight(x, w.shape, dy, padding=dil if k == 3 else 0, dilation=dil)
    assert _q(dw, B.conv_wgrad(x, dy, tuple(w.shape), dil)) <= 1.0
    assert _q(dw, B.conv_wgrad(x, dy, tuple(w.shape), dil, defect="drop_k16")) > 1.0


def test_storage_option_is_validated():
    net = csf_res2net.build_model()
    assert net.train_storage == "fp32" and modular_r.train_dtype(net) == torch.float32
    net.train_storage = "bf16"
    assert modular_r.train_dtype(net) == torch.bfloat16
    for bad in ("fp16", "BF16", None):
        net.train_storage = bad
        with pytest.raises(ValueError):
            modular_r.train_dtype(net)
    with pytest.raises(ValueError):
        CSFTrainer(net, storage="fp16")
    tr = CSFTrainer(net, storage="bf16")
    assert net.train_storage == "bf16" and tr.net is net
    CSFTrainer(net)
    assert net.train_storage == "fp32"
    net.set_precision("bf16")                            # inference precision: the training storage is untouched
    assert net.train_storage == "fp32"
