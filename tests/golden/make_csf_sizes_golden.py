"""Generate tests/golden/csf_res2net_sizes.npz: the UNMODIFIED reference CSF+Res2Net at input sizes that are not multiples of 32.

    python tests/golden/make_csf_sizes_golden.py

Needs the reference checkout (absent on the GPU box — the fixture is what travels); it is imported as-is, the way
make_golden.py's main_r does.  Weights are the seeded synthetic ones of sod100k_b200/synth.py (synth_state_r, seed 21), inputs
synth.randn_images.  The sizes reach: both stage ratios inexact (75x100, 97x131), one axis exact and the other not (96x100),
multiples of 16 that are not multiples of 32 (80x112), a 1-pixel stage-4 axis (24x130) and ECSSD-like 300x400 / 400x300.
Stored per case: the logits (sampled for the two large cases) and, for every head output (fuse.j, ms.j, fuse1x1), its mean,
std, max |.| and N_SAMPLE sampled elements.
"""
from __future__ import annotations

import contextlib
import io
import json
import os
import sys

import numpy as np

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("CSF_REFERENCE", os.path.join(os.path.dirname(ROOT), "reference", "CSF+Res2Net"))
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)

import torch  # noqa: E402

from sod100k_b200 import synth  # noqa: E402

SEED = 21
N_SAMPLE = 64
N_LOGIT_SAMPLE = 4096
CASES = {"75x100": (75, 100, 1401), "97x131": (97, 131, 1402), "96x100": (96, 100, 1403), "80x112": (80, 112, 1404),
         "24x130": (24, 130, 1405), "300x400": (300, 400, 1406), "400x300": (400, 300, 1407)}
SAMPLED = ("300x400", "400x300")


def sample_idx(numel, seed):
    return np.random.default_rng(seed).integers(0, numel, N_SAMPLE)


def tap_record(t: np.ndarray, seed: int) -> np.ndarray:
    flat = t.reshape(-1)
    return np.concatenate([[flat.mean(), flat.std(), np.abs(flat).max()], flat[sample_idx(flat.size, seed)]]).astype(np.float32)


def main():
    from networks.csf_res2net import build_model  # the reference

    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        net = build_model().eval()
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    net.load_state_dict({k: torch.from_numpy(v) for k, v in synth.synth_state_r(shapes, SEED).items()})
    taps = {}

    def hook(name):
        def fn(mod, inp, out):
            for j, t in enumerate(out):
                taps[f"{name}/{j}"] = t.detach().numpy()
        return fn

    hooks = [getattr(net, m).register_forward_hook(hook(m)) for m in ("fuse", "ms", "fuse1x1")]
    out = {}
    for tag, (h, w, seed) in CASES.items():
        taps.clear()
        with torch.no_grad():
            y = net(torch.from_numpy(synth.randn_images(1, h, w, seed))).numpy()
        if tag in SAMPLED:
            idx = np.random.default_rng(seed).integers(0, y.size, N_LOGIT_SAMPLE)
            out[f"{tag}/logits_idx"] = idx.astype(np.int64)
            out[f"{tag}/logits_sample"] = y.reshape(-1)[idx]
        else:
            out[f"{tag}/logits"] = y
        for k, t in taps.items():
            out[f"{tag}/tap/{k}"] = tap_record(t, seed)
        out[f"{tag}/feat_dims"] = np.array([t.shape[2:] for k, t in sorted(taps.items()) if k.startswith("fuse/")], np.int64)
    for hk in hooks:
        hk.remove()
    meta = dict(seed=SEED, shapes={k: list(v) for k, v in shapes.items()}, cases={k: list(v) for k, v in CASES.items()},
                sampled=list(SAMPLED), n_sample=N_SAMPLE, torch=torch.__version__)
    np.savez_compressed(os.path.join(HERE, "csf_res2net_sizes.npz"), __meta__=np.array(json.dumps(meta)), **out)
    print("wrote csf_res2net_sizes.npz", {tag: out[f"{tag}/feat_dims"].tolist() for tag in CASES})


if __name__ == "__main__":
    main()
