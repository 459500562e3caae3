"""bf16 activation storage without a GPU: the widened bounds of tests/trainref_bf16.py keep their power, and the storage
option is validated.

  * On the kernel cases' inputs rounded to bf16, the correct result rounded to bf16 passes the widened bound and every
    trainref defect (tests/test_trainref_cpu.py's DEFECT_CASES) is still flagged under it.
  * Truncation in place of round-to-nearest-even at a bf16 output is flagged.
  * Trainer(storage=...) takes "fp32" (the default) and "bf16" and nothing else."""
import pytest
import torch

from tests import trainref as R
from tests import trainref_bf16 as RB
from tests.test_gpu_train_kernels_vs_float64 import BY_ID, make_inputs, reference
from tests.test_trainref_cpu import DEFECT_CASES

BF16_KINDS = ("mix", "dw", "bn", "pool")


def test_widen_is_the_rounding_bound():
    g = torch.Generator().manual_seed(5)
    e = torch.randint(-140, 120, (100000,), generator=g).double()
    v = (torch.randn(100000, generator=g, dtype=torch.float64) * torch.pow(2.0, e)).float()       # fp32 values, subnormals included
    v[:8] = torch.tensor([0.0, 1e-45, -3e-41, 2.0 ** -133, 2.0 ** -126, 1.0, 1.00390625, 3.3e38], dtype=torch.float32)
    b = v.double().abs() * 2.0 ** -20 + 2.0 ** -140
    for r in (v.double() - b, v.double() + b):                # the fp32 value lies within b of r, on either side
        assert R.check(RB.round_bf16(v), r, RB.widen(r, b))[0] <= 1.0


def test_round_and_truncate_differ_as_expected():
    x = torch.tensor([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -9, -(1.0 + 3 * 2.0 ** -9), 1.0 + 2.0 ** -9], dtype=torch.float32)
    assert RB.round_bf16(x).tolist() == [1.0, 1.0 + 2.0 ** -7, -(1.0 + 2.0 ** -7), 1.0]       # ties to even
    assert RB.truncate_bf16(x).tolist() == [1.0, 1.0, -1.0, 1.0]


BF16_DEFECTS = [(d, c, o) for d, c, o in DEFECT_CASES if BY_ID[c].kind in BF16_KINDS]


@pytest.mark.parametrize("defect,case_id,outputs", BF16_DEFECTS, ids=[f"{d}-{c}" for d, c, _ in BF16_DEFECTS])
def test_each_defect_is_flagged_on_bf16_inputs(defect, case_id, outputs):
    case = BY_ID[case_id]
    inp = RB.bf16_inputs(case.kind, make_inputs(case))
    good = RB.widen_refs(case.kind, reference(case, inp))
    bad = reference(case, inp, defect=defect)
    for name in outputs:
        if name == "idx":
            assert R.check_idx(bad["idx"][0], *good["idx"]) > 0
            assert R.check_idx(good["idx"][0], *good["idx"]) == 0
            continue
        ref, bound = good[name]
        store = RB.round_bf16 if RB.stored_bf16(case.kind, name) else (lambda t: t.float())
        # the correct result as the kernel stores it passes; the defective one does not
        assert R.check(store(ref), ref, bound)[0] <= 1.0, name
        q, _ = R.check(store(bad[name][0]), ref, bound)
        print(f"DEFECT_Q_BF16 {defect} {case_id}/{name} {q:.3g}")
        assert q > 1.0, (defect, case_id, name, q)


TRUNC_CASES = [("c1_narrow", ["dst", "dsrc0"]), ("k3_ipb_14", ["dst", "dsrc0"]), ("dw_h5", ["y", "dxT", "bwd_dx"]),
               ("bn_s1", ["y", "dz0", "dz1"]), ("pool2_avg_real", ["dst"]), ("c1_with_resample", ["dsrc1"])]


@pytest.mark.parametrize("case_id,outputs", TRUNC_CASES, ids=[c for c, _ in TRUNC_CASES])
def test_truncation_is_flagged(case_id, outputs):
    case = BY_ID[case_id]
    inp = RB.bf16_inputs(case.kind, make_inputs(case))
    good = RB.widen_refs(case.kind, reference(case, inp))
    for name in outputs:
        ref, bound = good[name]
        assert RB.stored_bf16(case.kind, name)
        assert R.check(RB.round_bf16(ref), ref, bound)[0] <= 1.0, name
        q, _ = R.check(RB.truncate_bf16(ref.float()), ref, bound)
        print(f"TRUNC_Q_BF16 {case_id}/{name} {q:.3g}")
        assert q > 1.0, (case_id, name, q)


def _model():
    from sod100k_b200.model import csnet
    from tests import fixtures

    cfg, sd = fixtures.checkpoint("csnet-L-x2")
    m = csnet.CSNet(cfg)
    m.load_state_dict(sd)
    return m


@pytest.mark.parametrize("storage", ["fp16", "float32", "BF16", "", None])
def test_trainer_rejects_other_storage(storage):
    from sod100k_b200.trainer import Trainer

    m = _model()
    with pytest.raises(ValueError):
        Trainer(m, storage=storage)
    assert not hasattr(m, "train_storage")


@pytest.mark.parametrize("storage", ["fp32", "bf16"])
def test_trainer_sets_train_storage(storage):
    from sod100k_b200.trainer import Trainer

    m = _model()
    Trainer(m, storage=storage)
    assert m.train_storage == storage
    m2 = _model()
    Trainer(m2)
    assert m2.train_storage == "fp32"
