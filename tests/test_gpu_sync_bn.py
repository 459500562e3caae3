"""Synchronized BatchNorm (nn.SyncBatchNorm.convert_sync_batchnorm) in the fused training path.

1. Kernels against float64 (tests/syncbnref.py): csnet_train_bn_sync_partial / _merge / _bwd_reduce / _bwd_apply on G = 1, 2, 3
   and 8 synthetic shards of unequal batch (N = 1 shards, H W % 4 != 0, a channel at mean 1e4 std, a constant channel, and one
   case on the segmented, vectorised grid), fp32 and bf16.  The collective is emulated by adding the ranks' zeroed row buffers:
   a second run and a run that computes and adds the ranks in another order give the same bits, and the injected defects of
   syncbnref exceed their bounds.  Each entry point launches one kernel per dtype, so these cases run all seven kernels of
   csrc/bn_sync.cu.
2. World size 1 is today's code: a converted model without a process group, or in a one-rank group, trains bit-identically to
   an unconverted one (flops_weight on).
3. Two ranks equal one GPU over the whole batch: two spawned processes share the GPU over a gloo group (which takes CUDA tensors
   for all_reduce); csnet-L-x2 at 64 x 64, global batch 2 + 2, three Trainer steps against one process over the 4 images.
4. Negative controls in the same harness: an unconverted 2-rank run and a run that synchronizes only the forward fail (3)'s
   gradient gate.
5. After SyncBN training, the converted model's eval forward and its slimming equal those of an unconverted model with the same
   state_dict.
"""
import ctypes as C
import os
import socket
import traceback

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from sod100k_b200 import ir
from tests import syncbnref as S
from tests import trainref as R

pytestmark = pytest.mark.gpu

EPS = 1e-5

# (id, images per rank, H, W)
CASES = [("g1", [3], 7, 9), ("g2", [2, 1], 7, 9), ("g3", [1, 3, 2], 5, 13), ("g8", [1, 2, 1, 3, 1, 1, 2, 1], 6, 7),
         ("g2_segmented", [1, 2], 128, 128)]
NC = 5


# ---- (1) kernels ---------------------------------------------------------------------------------------------------------------
def _inputs(case):
    cid, shards, H, W = case
    g = torch.Generator().manual_seed(sum(map(ord, cid)))
    out = []
    for r, n in enumerate(shards):
        z = 2.0 * torch.randn((n, NC, H, W), generator=g, dtype=torch.float64) + 0.3 + 0.5 * r      # shards differ in mean
        z[:, 1] = 0.7                                                                                # a constant channel
        z[:, 2] = 0.5 * torch.randn((n, H, W), generator=g, dtype=torch.float64) + 1e4 + 0.5 * r     # mean 1e4 std
        dy = torch.randn((n, NC, H, W), generator=g, dtype=torch.float64) + 0.2
        out.append((z, dy))
    par = dict(gamma=(torch.rand(NC, generator=g) + 0.5).float(), beta=torch.randn(NC, generator=g).float(),
               slope=torch.tensor([-0.5, 1.5, 0.25, 0.0, 0.1]).float())
    return out, par


def _lib():
    from sod100k_b200 import train_ops as T

    return T.lib()


def _p(t):
    return C.c_void_p(t.data_ptr())


def _ck(rc):
    assert rc == 0, _lib().csnet_train_last_error().decode()


def run_sync(shards, par, dt, order):
    """The kernels over all ranks as the training step runs them, each rank into its own zeroed row buffer; the buffers are
    added in `order` (the collective).  Returns every output, on the CPU."""
    lib, st = _lib(), torch.cuda.current_stream().cuda_stream
    code = ir.BF16 if dt == torch.bfloat16 else ir.F32
    G = len(shards)
    zs = [z.to(dt).cuda() for z, _ in shards]
    dys = [dy.to(dt).cuda() for _, dy in shards]
    g, b, a = (par[k].cuda() for k in ("gamma", "beta", "slope"))
    out = {"rows": [None] * G, "red": [None] * G, "dz": [None] * G}
    bufs = [None] * G
    for r in order:
        n, _, H, W = zs[r].shape
        bufs[r] = torch.zeros((G, NC, 3), dtype=torch.float64, device="cuda")
        _ck(lib.csnet_train_bn_sync_partial(_p(zs[r]), code, n, NC, H * W, r, _p(bufs[r]), st))
        out["rows"][r] = bufs[r][r].cpu()
    rows = torch.zeros_like(bufs[0])
    for r in order:
        rows = rows + bufs[r]
    mean, var = torch.empty(NC, device="cuda"), torch.empty(NC, device="cuda")
    count = torch.empty(1, dtype=torch.float64, device="cuda")
    _ck(lib.csnet_train_bn_sync_merge(_p(rows), G, NC, _p(mean), _p(var), _p(count), st))
    out.update(gathered=rows.cpu(), mean=mean.cpu(), var=var.cpu(), count=count.cpu())
    bufs2 = [None] * G
    for r in order:
        n, _, H, W = zs[r].shape
        bufs2[r] = torch.zeros((G, NC, 2), dtype=torch.float64, device="cuda")
        dg, db, ds = (torch.empty(NC, device="cuda") for _ in range(3))
        _ck(lib.csnet_train_bn_sync_bwd_reduce(_p(zs[r]), _p(dys[r]), code, n, NC, H * W, _p(mean), _p(var), _p(g), _p(b), _p(a),
                                               C.c_float(EPS), _p(dg), _p(db), _p(ds), r, _p(bufs2[r]), st))
        out["red"][r] = dict(dgamma=dg.cpu(), dbeta=db.cpu(), dslope=ds.cpu(), S1=bufs2[r][r, :, 0].cpu(), S2=bufs2[r][r, :, 1].cpu())
    rows2 = torch.zeros_like(bufs2[0])
    for r in order:
        rows2 = rows2 + bufs2[r]
    out["gathered2"] = rows2.cpu()
    for r in order:
        n, _, H, W = zs[r].shape
        dz = torch.empty_like(zs[r])
        _ck(lib.csnet_train_bn_sync_bwd_apply(_p(zs[r]), _p(dys[r]), _p(dz), code, n, NC, H * W, _p(mean), _p(var), _p(g), _p(b), _p(a),
                                              C.c_float(EPS), _p(rows2), G, _p(count), st))
        out["dz"][r] = dz.float().cpu()
    torch.cuda.synchronize()
    out["inputs"] = [(z.cpu(), dy.cpu()) for z, dy in zip(zs, dys)]
    return out


def _flat(o):
    ts = []
    for v in o.values():
        if isinstance(v, torch.Tensor):
            ts.append(v)
        elif isinstance(v, list):
            for e in v:
                ts += list(e.values()) if isinstance(e, dict) else (list(e) if isinstance(e, tuple) else [e])
    return ts


def _within(name, got, rb):
    q, where = R.check(got, *rb)
    assert q <= 1.0, f"{name}: {where}"
    return q


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_sync_kernels_match_float64(case, dt):
    shards, par = _inputs(case)
    G = len(shards)
    got = run_sync(shards, par, dt, list(range(G)))
    again = run_sync(shards, par, dt, list(range(G)))
    perm = run_sync(shards, par, dt, [(r + 1) % G for r in range(G)])
    perm2 = run_sync(shards, par, dt, list(reversed(range(G))))
    for other in (again, perm, perm2):
        assert all(torch.equal(x, y) for x, y in zip(_flat(got), _flat(other)))
    for r in range(G):
        z, dy = got["inputs"][r]
        ref = S.partial(z)
        for k, col in (("count", 0), ("mean", 1), ("M2", 2)):
            _within(f"partial[{r}].{k}", got["rows"][r][:, col], ref[k])
    ref = S.merge(got["gathered"])
    for k in ("mean", "var", "count"):
        _within(f"merge.{k}", got[k], ref[k])
    if G > 1:
        assert R.check(got["var"], *S.merge(got["gathered"], defect="no_chan")["var"])[0] > 1.0
    a = (got["mean"], got["var"], par["gamma"], par["beta"], par["slope"], EPS)
    for r in range(G):
        z, dy = got["inputs"][r]
        ref = S.bwd_reduce(z, dy, *a)
        for k in ("dgamma", "dbeta", "dslope", "S1", "S2"):
            _within(f"bwd_reduce[{r}].{k}", got["red"][r][k], ref[k])
        bf = dt == torch.bfloat16
        _within(f"bwd_apply[{r}].dz", got["dz"][r], S.bwd_apply(z, dy, *a, got["gathered2"], got["count"], bf16=bf)["dz"])
        if G > 1:
            bad = S.bwd_apply(z, dy, *a, got["gathered2"], got["count"], bf16=bf, defect="local_count")["dz"]
            assert R.check(got["dz"][r], *bad)[0] > 1.0


# ---- shared: the model and the batch ---------------------------------------------------------------------------------------------
TAG, HW, PER, STEPS = "csnet-L-x2", 64, 2, 3


def _batch(world=2):
    from sod100k_b200 import synth

    return (torch.from_numpy(synth.randn_images(PER * world, HW, HW, 11)), torch.from_numpy(synth.random_masks(PER * world, HW, HW, 12)))


def _model(convert):
    from sod100k_b200 import checkpoints

    m, _, _ = checkpoints.build_from_npz(TAG)
    if convert:
        m = nn.SyncBatchNorm.convert_sync_batchnorm(m)
    return m.cuda()


def _bn_buffers(m):
    return [t.detach().clone() for n, t in m.named_buffers() if n.endswith(("running_mean", "running_var", "num_batches_tracked"))]


def _train(convert, x, t, storage="fp32", recompute=False, flops_weight=None, steps=STEPS):
    from sod100k_b200.trainer import Trainer

    m = _model(convert)
    tr = Trainer(m, lr=1e-4, flops_weight=flops_weight, storage=storage, recompute=recompute)
    losses, bucket = [], None
    for s in range(steps):
        losses.append(float(tr.step(x, t)))
        if s == 0:
            bucket, buffers1 = tr.flat.bucket.detach().clone(), [b.cpu() for b in _bn_buffers(m)]
    return dict(losses=losses, bucket=bucket.cpu(), buffers1=buffers1, params=[p.detach().cpu().clone() for p in m.parameters()],
                buffers=[b.cpu() for b in _bn_buffers(m)], state_dict={k: v.detach().cpu().clone() for k, v in m.state_dict().items()})


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


# ---- (2) world size 1 ------------------------------------------------------------------------------------------------------------
def test_world_size_one_is_unchanged():
    x, t = (v[:PER].cuda() for v in _batch())
    plain = _train(False, x, t, flops_weight=3.0)
    conv = _train(True, x, t, flops_weight=3.0)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{_free_port()}", rank=0, world_size=1)
    try:
        one = _train(True, x, t, flops_weight=3.0)
    finally:
        dist.destroy_process_group()
    for other in (conv, one):
        assert all(torch.equal(a, b) for a, b in zip(plain["params"] + plain["buffers"], other["params"] + other["buffers"]))


# ---- (3, 4) two ranks on one GPU over gloo -------------------------------------------------------------------------------------
def _forward_only_backward(ctx, dy, _dm, _dv, _dc, _dg):
    """SyncBnPreluFn.backward with this rank's sums and count: synchronizes the forward only (negative control)."""
    from sod100k_b200 import train_ops as T

    z, mean, var, count, g, b, a = ctx.saved_tensors
    dy = dy.contiguous().float()
    n, c, h, w = z.shape
    dz = torch.empty_like(z)
    dgamma, dbeta, dslope = (torch.empty(c, device=z.device) for _ in range(3))
    T._ck(T.lib().csnet_train_bn_prelu_bwd(z.data_ptr(), dy.data_ptr(), dz.data_ptr(), n, c, h * w, mean.data_ptr(), var.data_ptr(),
                                           g.data_ptr(), b.data_ptr(), a.data_ptr(), T.BN_EPS, dgamma.data_ptr(), dbeta.data_ptr(),
                                           dslope.data_ptr(), 0, T._stream(z)), "csnet_train_bn_prelu_bwd")
    return dz, dgamma, dbeta, dslope, None, None, None


def _worker(rank, world, port, out_dir):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        from sod100k_b200 import train_ops as T

        x, t = _batch(world)
        x, t = x[rank * PER:(rank + 1) * PER].cuda(), t[rank * PER:(rank + 1) * PER].cuda()
        res = {"sync": _train(True, x, t), "sync_recompute": _train(True, x, t, recompute=True),
               "sync_bf16": _train(True, x, t, storage="bf16"), "local": _train(False, x, t, steps=1)}
        saved = T.SyncBnPreluFn.backward
        T.SyncBnPreluFn.backward = staticmethod(_forward_only_backward)
        try:
            res["forward_only"] = _train(True, x, t, steps=1)
        finally:
            T.SyncBnPreluFn.backward = saved
        torch.save(res, os.path.join(out_dir, f"rank{rank}.pt"))
        dist.destroy_process_group()
    except BaseException:
        with open(os.path.join(out_dir, f"rank{rank}.err"), "w") as f:
            f.write(traceback.format_exc())
        raise


@pytest.fixture(scope="module")
def two_ranks(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("sync_bn"))
    ctx = mp.get_context("spawn")
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=900)
    for p in procs:
        if p.is_alive():
            p.terminate()
            p.join()
    errs = [open(os.path.join(out, f)).read() for f in sorted(os.listdir(out)) if f.endswith(".err")]
    assert not errs, "\n".join(errs)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    ranks = [torch.load(os.path.join(out, f"rank{r}.pt")) for r in range(2)]
    x, t = (v.cuda() for v in _batch(2))
    perm = torch.tensor([2, 3, 0, 1], device="cuda")
    single = {"fp32": _train(False, x, t), "bf16": _train(False, x, t, storage="bf16"),
              "fp32_reordered": _train(False, x[perm], t[perm])}         # the same step, the batch summed in another order
    return ranks, single


def _split(bucket, params):
    out, off = [], 0
    for p in params:
        out.append(bucket[off:off + p.numel()])
        off += p.numel()
    return out


def _grad_err(run, ref):
    """(max over parameter tensors of max |g - g_ref| / max |g_ref|, that tensor's size, the relative L2 error of the whole
    bucket) of the first step's all-reduced bucket."""
    worst = (0.0, 0)
    for g, gr in zip(_split(run["bucket"], ref["params"]), _split(ref["bucket"], ref["params"])):
        s = float(gr.abs().max())
        if s > 0:
            worst = max(worst, (float((g - gr).abs().max()) / s, g.numel()))
    return worst + (float((run["bucket"] - ref["bucket"]).norm() / ref["bucket"].norm()),)


def _stat_err(bufs, ref_bufs):
    """max over the running means / variances of max |b - b_ref| / max |b_ref|"""
    return max(float((a - b).abs().max()) / float(b.abs().max()) for a, b in zip(bufs, ref_bufs) if a.is_floating_point())


def test_two_ranks_equal_one_gpu_over_the_whole_batch(two_ranks):
    """The first step starts from the same parameters on both sides and is held to the tight gates.  Its gradients are
    compared per tensor, where a max-pool arg-max or a PReLU sign at a near-tie (reached through a 1-ulp difference: a
    batch of 2 and a batch of 4 tile the convolutions differently) gives one small tensor a different, equally valid
    sub-gradient (tests/test_gpu_train.py), and over the whole bucket.  Adam's first steps move a weight by about lr *
    sign(g), so such a difference moves some weights by 2 lr and the later steps drift apart by more than rounding; they
    keep looser gates."""
    ranks, single = two_ranks
    ref = single["fp32"]
    mean_losses = [(a + b) / 2 for a, b in zip(ranks[0]["sync"]["losses"], ranks[1]["sync"]["losses"])]
    rel = [abs(a - b) / abs(b) for a, b in zip(mean_losses, ref["losses"])]
    grad, stat1, stat3 = _grad_err(ranks[0]["sync"], ref), _stat_err(ranks[0]["sync"]["buffers1"], ref["buffers1"]), \
        _stat_err(ranks[0]["sync"]["buffers"], ref["buffers"])
    print(f"2 ranks vs one GPU: loss rel diff per step {rel}, first-step gradient (worst tensor, its size, bucket L2) {grad}, "
          f"running statistics after 1 / {STEPS} steps {stat1:.3g} / {stat3:.3g}; batch reordered on one GPU: loss "
          f"{[abs(a - b) / abs(b) for a, b in zip(single['fp32_reordered']['losses'], ref['losses'])]}, gradient "
          f"{_grad_err(single['fp32_reordered'], ref)}, statistics {_stat_err(single['fp32_reordered']['buffers'], ref['buffers']):.3g}")
    assert rel[0] <= 1e-5 and max(rel) <= 1e-4, rel
    assert grad[2] <= 1e-3 and grad[0] <= 5e-3, grad
    assert stat1 <= 1e-5 and stat3 <= 3e-3, (stat1, stat3)
    assert all(torch.equal(a, b) for a, b in zip(ranks[0]["sync"]["buffers1"], ranks[1]["sync"]["buffers1"]))
    assert torch.equal(ranks[0]["sync"]["bucket"], ranks[1]["sync"]["bucket"])
    for key in ("sync", "sync_recompute", "sync_bf16"):
        assert all(torch.equal(a, b) for a, b in zip(ranks[0][key]["params"] + ranks[0][key]["buffers"],
                                                     ranks[1][key]["params"] + ranks[1][key]["buffers"])), key
    assert all(torch.equal(a, b) for a, b in zip(ranks[0]["sync"]["params"] + ranks[0]["sync"]["buffers"],
                                                 ranks[0]["sync_recompute"]["params"] + ranks[0]["sync_recompute"]["buffers"]))
    # bf16: two bf16 evaluations of the same step that round differently differ by up to twice what bf16 storage moves the
    # step's loss from fp32; the first step (same parameters) is held to that, or to 1e-3 where bf16 moves it less
    floor = abs(single["bf16"]["losses"][0] - ref["losses"][0]) / abs(ref["losses"][0])
    bf = [abs((a + b) / 2 - c) / abs(c) for a, b, c in zip(ranks[0]["sync_bf16"]["losses"], ranks[1]["sync_bf16"]["losses"],
                                                             single["bf16"]["losses"])]
    print(f"bf16: 2 ranks vs one GPU loss rel diff per step {bf}; one GPU bf16 vs fp32 on the first step {floor:.3g}")
    assert bf[0] <= max(1e-3, 2 * floor), (bf, floor)


def test_local_statistics_fail_the_gradient_gate(two_ranks):
    ranks, single = two_ranks
    for key in ("local", "forward_only"):
        err = _grad_err(ranks[0][key], single["fp32"])
        print(key, "first-step gradient (worst tensor, its size, bucket L2)", err)
        assert err[0] > 5e-3 and err[2] > 1e-3, key


# ---- (5) inference and slimming after SyncBN training --------------------------------------------------------------------------
def test_inference_and_slimming_after_sync_training(two_ranks):
    from sod100k_b200 import slim, synth
    from tests import fixtures
    from tests.test_slim import _cfg_lists

    sd = two_ranks[0][0]["sync"]["state_dict"]
    conv, plain = _model(True), _model(False)
    conv.load_state_dict(sd)
    plain.load_state_dict(sd)
    conv.eval(), plain.eval()
    x = torch.from_numpy(synth.randn_images(2, 96, 64, 21)).cuda()
    with torch.no_grad():
        assert torch.equal(conv(x), plain(x))
    cfg, _ = fixtures.checkpoint(TAG)
    for thres in (1e-3, 1e-2):
        c_cfg, c_masks = slim.finetune_config(conv, cfg, thres)
        p_cfg, p_masks = slim.finetune_config(plain, cfg, thres)
        assert _cfg_lists(c_cfg) == _cfg_lists(p_cfg)
        c_sd = slim.build_model_with_weight(c_cfg, conv, c_masks).state_dict()
        p_sd = slim.build_model_with_weight(p_cfg, plain, p_masks).state_dict()
        assert list(c_sd) == list(p_sd) and all(torch.equal(c_sd[k], p_sd[k]) for k in p_sd)
