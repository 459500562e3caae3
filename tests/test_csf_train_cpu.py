"""CSF+Res2Net training checks that need no GPU: the resize adjoint's tap inversion against the transpose of the forward tap
matrix, and the oracle's float64-capable autograd against the reference's golden training step."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import csf_res2net_oracle as R
from sod100k_b200 import synth
from tests import fixtures
from tests.trainref_r import tap_matrix

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
SIZES = [(11, 22), (22, 88), (88, 352), (3, 24), (5, 130), (75, 19), (100, 25), (10, 7), (13, 9), (1, 4), (9, 9), (6, 1), (7, 1),
         (1, 1), (13, 40), (17, 41), (2, 3), (400, 13)]


@pytest.fixture(scope="module")
def adj_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu") / "libresize_adj_emu.so")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17", "-o", out,
                    os.path.join(EMU, "resize_adj_emu.cpp")], check=True)
    lib = C.CDLL(out)
    lib.csnet_emu_resize_adjoint.argtypes = [C.c_int, C.c_int, C.c_void_p]
    return lib


@pytest.mark.parametrize("n_in,n_out", SIZES)
def test_adjoint_taps_are_the_transposed_forward_taps(adj_lib, n_in, n_out):
    adj = np.zeros((n_in, n_out))
    adj_lib.csnet_emu_resize_adjoint(n_in, n_out, adj.ctypes.data)
    A = tap_matrix(n_in, n_out)
    assert np.array_equal(adj, A.T)
    # and the matrix is F.interpolate's (to fp32 tap rounding)
    eye = torch.eye(n_in, dtype=torch.float64).view(n_in, 1, n_in, 1)
    ref = F.interpolate(eye, size=(n_out, 1), mode="bilinear", align_corners=False).view(n_in, n_out)
    assert np.abs(ref.numpy() - adj).max() <= 4 * 2.0 ** -24 * (n_in + 2)


def test_oracle_autograd_matches_reference_training_golden():
    z = np.load(os.path.join(fixtures.GOLDEN, "csf_train.npz"))
    meta = json.loads(str(z["__meta__"]))
    from sod100k_b200.networks import csf_res2net

    m = csf_res2net.build_model()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    sd = {k: torch.from_numpy(v) for k, v in synth.synth_state_r(shapes, meta["seed"]).items()}
    names = meta["grad_names"]
    params = [sd[k].requires_grad_(True) for k in names]
    opt = torch.optim.Adam(params, lr=meta["lr"], weight_decay=meta["wd"])
    for step, (h, w, seed) in enumerate(meta["steps"]):
        x = torch.from_numpy(synth.randn_images(1, h, w, seed))
        y = torch.from_numpy((np.random.default_rng(seed).random((1, 1, h, w)) > 0.5).astype(np.float32))
        loss = F.binary_cross_entropy_with_logits(R.csfnet_forward(sd, x), y, reduction="sum") / meta["iter_size"]
        assert abs(loss.item() - float(z["loss"][step])) <= 1e-4 * abs(float(z["loss"][step]))
        loss.backward()
    for k, p in zip(names, params):
        got = p.grad.reshape(-1)[torch.from_numpy(z[f"gidx/{k}"])].double().numpy()
        assert np.abs(got - z[f"gsample/{k}"]).max() <= 1e-3 * float(z[f"gscale/{k}"]) + 1e-30, k
        assert abs(p.grad.double().norm().item() - float(z[f"gnorm/{k}"])) <= 1e-3 * float(z[f"gnorm/{k}"]) + 1e-30, k
    opt.step()
    for k, p in zip(names, params):
        got = p.detach().reshape(-1)[torch.from_numpy(z[f"gidx/{k}"])].double().numpy()
        assert np.abs(got - z[f"psample/{k}"]).max() <= 1e-3 * float(z[f"pscale/{k}"]), k
