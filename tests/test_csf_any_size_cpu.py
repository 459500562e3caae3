"""CSF+Res2Net at input sizes that are not multiples of 32, CPU side: the oracle against the reference's goldens at those sizes, the
head program with its RESIZE ops (host emulation of the kernels' per-pixel code) against the oracle, the RESIZE body against
float64 F.interpolate, and the programs at multiples of 32 unchanged."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import csf_res2net_oracle as R
from sod100k_b200 import compiler_r, ir, synth
from tests import fixtures
from tests.emu import resize as emu_resize
from tests.resize_ref import resize64


def _golden():
    z = np.load(os.path.join(fixtures.GOLDEN, "csf_res2net_sizes.npz"))
    return z, json.loads(str(z["__meta__"]))


def _state(meta):
    sd = synth.synth_state_r({k: tuple(v) for k, v in meta["shapes"].items()}, meta["seed"])
    return {k: torch.from_numpy(v) for k, v in sd.items()}


def _tap_record(t, seed, n):
    flat = t.reshape(-1)
    idx = np.random.default_rng(seed).integers(0, flat.size, n)
    return np.concatenate([[flat.mean(), flat.std(), np.abs(flat).max()], flat[idx]])


def test_oracle_matches_reference_goldens_at_any_size():
    z, meta = _golden()
    sd = _state(meta)
    for tag, (h, w, seed) in meta["cases"].items():
        taps = {}
        with torch.no_grad():
            y = R.csfnet_forward(sd, torch.from_numpy(synth.randn_images(1, h, w, seed)), taps).numpy()
        assert [tuple(f.shape[2:]) for f in taps["feats"]] == compiler_r.res2net_feat_dims(h, w), tag
        if tag in meta["sampled"]:
            got, ref = y.reshape(-1)[z[f"{tag}/logits_idx"]], z[f"{tag}/logits_sample"]
        else:
            got, ref = y, z[f"{tag}/logits"]
        assert got.shape == ref.shape and np.abs(got - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max()), tag
        named = {f"fuse/{j}": t for j, t in enumerate(taps["fuse"])}
        named.update({f"ms/{j}": t for j, t in enumerate(taps["ms"])})
        named["fuse1x1/0"] = taps["fuse1x1"]
        for k, t in named.items():
            ref = z[f"{tag}/tap/{k}"]
            got = _tap_record(t.numpy(), seed, meta["n_sample"])
            assert np.abs(got - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max()), (tag, k)


@pytest.mark.parametrize("tag", ["75x100", "24x130"])
def test_emulated_inexact_head_program_matches_oracle(tag):
    z, meta = _golden()
    sd = _state(meta)
    h, w, seed = meta["cases"][tag]
    x = torch.from_numpy(synth.randn_images(1, h, w, seed))
    taps = {}
    with torch.no_grad():
        ref = R.csfnet_forward(sd, x, taps).numpy()
    feats = [np.ascontiguousarray(f.numpy()) for f in taps["feats"]]
    prog = compiler_r.compile_csf_head(sd, [f.shape[1:] for f in feats], h, w, "fp32", reuse_arena=False)
    kinds = [o.kind for o in prog.ops]
    assert kinds.count(ir.OP_RESIZE) == 6 + 6 + 3 + 1          # fuse down + up paths, fuse1x1 up paths, the final resize
    y = np.zeros((1, 1, h, w), np.float32)
    names = ["fuse/0", "fuse/1", "fuse/2", "fuse/3", "ms/1", "fuse1x1/0"]
    got = emu_resize.run_ext(prog, feats + [y], 1, taps=names)
    for name in names:
        kind, j = name.split("/")
        r = (taps["fuse1x1"] if kind == "fuse1x1" else taps[kind][int(j)]).numpy()
        assert np.abs(got[name] - r).max() <= 2e-4 * max(1.0, np.abs(r).max()), name
    assert np.abs(y - ref).max() <= 2e-4 * max(1.0, np.abs(ref).max())
    z_ref = z[f"{tag}/logits"]
    assert np.abs(y - z_ref).max() <= 2e-4 * max(1.0, np.abs(z_ref).max())


def _resize_prog(Cs, Hs, Ws, Cd, Hd, Wd, c0, cout0, C, accumulate, sdt=ir.F32, ddt=ir.F32):
    b = ir.Builder()
    s = b.tensor(Cs, Hs, Ws, sdt, external=0, name="src")
    d = b.tensor(Cd, Hd, Wd, ddt, external=1, name="dst")
    b.op(ir.OP_RESIZE, d, [ir.Path(s, C, C, c0=c0, cout0=cout0, ksize=0)], name="resize").ext_off = [int(accumulate)]
    return b.finish(reuse=False)


# (Hs, Ws) -> (Hd, Wd): up, down, equal, one-pixel sources and destinations, mixed ratios per axis
GEOMS = [((5, 7), (13, 17)), ((13, 17), (4, 5)), ((6, 9), (6, 9)), ((1, 1), (5, 3)), ((7, 9), (1, 1)), ((1, 9), (4, 2)),
         ((10, 13), (75, 100)), ((19, 25), (10, 13))]


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("geom", GEOMS, ids=[f"{a[0]}x{a[1]}to{b[0]}x{b[1]}" for a, b in GEOMS])
def test_resize_body_matches_float64_interpolate(geom, accumulate):
    (Hs, Ws), (Hd, Wd) = geom
    rng = np.random.default_rng(Hs * 1000 + Wd)
    N, Cs, Cd, c0, cout0, C = 2, 5, 6, 1, 2, 3
    prog = _resize_prog(Cs, Hs, Ws, Cd, Hd, Wd, c0, cout0, C, accumulate)
    src = rng.standard_normal((N, Cs, Hs, Ws)).astype(np.float32)
    dst = rng.standard_normal((N, Cd, Hd, Wd)).astype(np.float32)
    old = dst.copy()
    emu_resize.run_ext(prog, [src, dst], N)
    ref, bound = resize64(src[:, c0:c0 + C].astype(np.float64), Hd, Wd, old[:, cout0:cout0 + C] if accumulate else None)
    err = np.abs(dst[:, cout0:cout0 + C] - ref.numpy())
    assert (err <= bound.numpy()).all(), float((err / bound.numpy()).max())
    keep = np.ones(Cd, bool)
    keep[cout0:cout0 + C] = False
    assert np.array_equal(dst[:, keep], old[:, keep])                  # channels outside the slice are untouched


# signature() of the head programs at multiples of 32, recorded from the compiler before RESIZE ops existed
EXACT_SIGNATURES = {
    (64, 96, "fp32"): "40ff890ba2382a1d8a20545e2055cbd92df5f52fca36a8b0b65a14a3e30c50ee",
    (64, 96, "fp16"): "79d412224aa5eb8d3ede211af442584e056c534360b5574c2b309b8f6633ab87",
    (96, 96, "fp32"): "67e3d022c87c8e61d3d7796146e2c8fde3a1606b1c0e70beaa317119978899ff",
    (96, 96, "fp16"): "adf632f340402e3958dc0e8cfe9d5542b3bc04c45a07d853b9be1f015adaf724",
    (352, 352, "fp32"): "8dcf181aa4462a617f19b8df66e63296c474a842fa014a246a5c01a232cedbdb",
    (352, 352, "fp16"): "a95a10ffc53ad8a27674e65a41cc2a6174b9a0a402ff0fe294d2f022c46139dc",
}


def _dims(H, W):
    return [(c, h, w) for c, (h, w) in zip((256, 512, 1024, 2048), compiler_r.res2net_feat_dims(H, W))]


@pytest.mark.parametrize("H,W,dtype", sorted(EXACT_SIGNATURES))
def test_programs_at_multiples_of_32_are_unchanged(H, W, dtype):
    _, meta = _golden()
    sd = _state(meta)
    prog = compiler_r.compile_csf_head(sd, _dims(H, W), H, W, dtype)
    assert prog.signature().hex() == EXACT_SIGNATURES[(H, W, dtype)]
    assert all(o.kind != ir.OP_RESIZE for o in prog.ops)


def test_ceil_chain_and_mismatched_feature_dims_raise():
    assert compiler_r.res2net_feat_dims(75, 100) == [(19, 25), (10, 13), (5, 7), (3, 4)]
    assert compiler_r.res2net_feat_dims(24, 130) == [(6, 33), (3, 17), (2, 9), (1, 5)]
    _, meta = _golden()
    sd = _state(meta)
    good = _dims(75, 100)
    compiler_r.compile_csf_head(sd, good, 75, 100, "fp32")
    for bad in ([(256, 19, 25), (512, 9, 13), (1024, 5, 7), (2048, 3, 4)],          # floor instead of ceil at stage 1
                [(256, 18, 25), (512, 9, 13), (1024, 5, 7), (2048, 3, 4)],          # the whole chain of a 72x100 input
                [(256, 16, 24), (512, 8, 12), (1024, 4, 6), (2048, 2, 3)]):         # exact halving, wrong input size
        with pytest.raises(ValueError):
            compiler_r.compile_csf_head(sd, bad, 75, 100, "fp32")
    with pytest.raises(ValueError):
        compiler_r.compile_csf_head(sd, _dims(64, 96), 64, 128, "fp32")
