"""nn.SyncBatchNorm.convert_sync_batchnorm on CSNet without a GPU: which BatchNorm modules synchronize, and a converted model
slims, counts FLOPs and takes updateWeight exactly like an unconverted one.  Also checks that tests/syncbnref.py flags its
defects on exact inputs (the GPU test flags them against the kernels)."""
import pytest
import torch
import torch.nn as nn

from sod100k_b200 import slim, train_ops as T
from sod100k_b200.model import csnet
from sod100k_b200.model.utils import simplesum_octconv
from tests import fixtures
from tests import syncbnref as S
from tests.test_slim import _cfg_lists

TAG = "csnet-L-x2"


def _pair():
    cfg, sd = fixtures.checkpoint(TAG)
    plain = csnet.CSNet(cfg)
    plain.load_state_dict(sd)
    conv = csnet.CSNet(cfg)
    conv.load_state_dict(sd)
    return cfg, plain, nn.SyncBatchNorm.convert_sync_batchnorm(conv)


def test_conversion_keeps_the_state_dict():
    _, plain, conv = _pair()
    assert sum(isinstance(m, nn.SyncBatchNorm) for m in conv.modules()) == 106
    assert list(conv.state_dict()) == list(plain.state_dict())


def test_sync_only_with_an_initialised_group():
    bn, sbn = nn.BatchNorm2d(4), nn.SyncBatchNorm(4)
    assert not torch.distributed.is_initialized()
    assert T.sync_group(bn) is None and T.sync_group(sbn) is None          # no process group: the statistics of this process
    sbn.eval()
    assert T.sync_group(sbn) is None


@pytest.mark.parametrize("thres", [1e-3, 1e-2])
def test_converted_model_slims_the_same(thres):
    cfg, plain, conv = _pair()
    p_cfg, p_masks = slim.finetune_config(plain, cfg, thres)
    c_cfg, c_masks = slim.finetune_config(conv, cfg, thres)
    assert _cfg_lists(c_cfg) == _cfg_lists(p_cfg)
    p_sd = slim.build_model_with_weight(p_cfg, plain, p_masks).state_dict()
    c_sd = slim.build_model_with_weight(c_cfg, conv, c_masks).state_dict()
    assert list(c_sd) == list(p_sd) and all(torch.equal(c_sd[k], p_sd[k]) for k in p_sd)


def test_converted_model_update_weight_and_flops():
    _, plain, conv = _pair()
    for m in (plain, conv):
        for p in m.parameters():
            p.grad = torch.zeros_like(p)
        m.updateWeight(0.01)
    assert all(torch.equal(a.grad, b.grad) for a, b in zip(plain.parameters(), conv.parameters()))
    assert any(bool(p.grad.abs().sum() > 0) for p in conv.parameters())
    assert simplesum_octconv.simplesum(conv, (3, 224, 224)) == simplesum_octconv.simplesum(plain, (3, 224, 224))


def test_reference_defects_are_flagged():
    g = torch.Generator().manual_seed(5)
    shards = [2.0 * torch.randn((n, 3, 5, 7), generator=g, dtype=torch.float64) + 0.5 * r for r, n in enumerate((1, 3, 2))]
    rows = torch.stack([torch.stack([S.partial(z)[k][0] for k in ("count", "mean", "M2")], -1) for z in shards])
    ref, bad = S.merge(rows), S.merge(rows, defect="no_chan")
    assert float(((bad["var"][0] - ref["var"][0]).abs() / ref["var"][1]).max()) > 1.0
    assert float(((ref["mean"][0] - torch.cat(shards).mean((0, 2, 3))).abs() / ref["mean"][1]).max()) <= 1.0
    assert float(((ref["var"][0] - torch.cat(shards).var((0, 2, 3), unbiased=False)).abs() / ref["var"][1]).max()) <= 1.0
    z, dy = shards[1], torch.randn(shards[1].shape, generator=g, dtype=torch.float64)
    C = z.shape[1]
    a = (ref["mean"][0].float(), ref["var"][0].float(), torch.ones(C), torch.zeros(C), torch.full((C,), 0.25), 1e-5)
    s = [S.bwd_reduce(x, torch.randn(x.shape, generator=g, dtype=torch.float64), *a) for x in shards]
    rows2 = torch.stack([torch.stack([e["S1"][0], e["S2"][0]], -1) for e in s])
    good, bad = S.bwd_apply(z, dy, *a, rows2, ref["count"][0]), S.bwd_apply(z, dy, *a, rows2, ref["count"][0], defect="local_count")
    assert float(((bad["dz"][0] - good["dz"][0]).abs() / good["dz"][1]).max()) > 1.0
