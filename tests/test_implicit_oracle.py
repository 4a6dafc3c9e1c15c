"""CPU checks of the implicit diffusion (diffusion_method='implicit_dense'): the fp64 sparse-direct oracle
(oracle/dn_oracle_implicit.implicit_diffusion) against what the live reference computed (tests/golden/implicit_small.npz,
from oracle/make_golden_implicit.py), and checkpoint loading into implicit nets.  No GPU here."""
import glob
import json
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from conftest import GOLDEN, ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle_implicit as OI  # noqa: E402
import ref_import  # noqa: E402

import diffusion_net_b200 as dn  # noqa: E402

MESHES = ["torus", "patch"]


def _mesh(fx, tag):
    f = lambda k: fx["{}:{}".format(tag, k)]
    V = f("mass").shape[0]
    L = sp.csr_matrix((f("L_vals").astype(np.float64), (f("L_rows"), f("L_cols"))), shape=(V, V))
    return f, L


@pytest.mark.parametrize("tag", MESHES)
def test_oracle_matches_reference_implicit_diffusion(tag):
    f, L = _mesh(load_golden("implicit_small"), tag)
    y, gx, gt = OI.implicit_diffusion(f("x"), f("mass"), L, f("time_raw"), grad_out=f("g"))
    for mine, key in ((y, "y64"), (gx, "gx64"), (gt, "gt64")):
        gold = f(key)
        assert np.abs(mine - gold).max() <= 1e-10 * np.abs(gold).max(), key
    # the clamp of layers.py:48-49: the negative and the 1e-8 entries both end at 1e-8
    assert np.array_equal(f("time_clamped32"), np.maximum(f("time_raw"), np.float32(1e-8)))
    assert np.all(np.diff(f("time_raw")[1:]) > 0) and f("time_raw")[0] < 0 and f("time_raw")[-1] == np.float32(0.5)


def _net_from_manifest_keys(keys, **kw):
    C_in, C_out, C_width = keys["first_lin.weight"][1], keys["last_lin.weight"][0], keys["first_lin.weight"][0]
    n_block = len([k for k in keys if k.endswith("diffusion.diffusion_time")])
    return dn.DiffusionNet(C_in=C_in, C_out=C_out, C_width=C_width, N_block=n_block, **kw)


def test_shipped_state_dicts_strict_load_into_implicit_nets():
    man = json.load(open(os.path.join(GOLDEN, "statedict_manifest.json")))
    pre = "feature_extractor."
    for name, keys in man.items():
        if all(k.startswith(pre) for k in keys):
            keys = {k[len(pre):]: v for k, v in keys.items()}
        net = _net_from_manifest_keys(keys, diffusion_method="implicit_dense")
        g = torch.Generator().manual_seed(0)
        sd = {k: torch.randn(v, generator=g) for k, v in keys.items()}
        net.load_state_dict(sd, strict=True)
        assert all(b.diffusion.method == "implicit_dense" for b in net.blocks), name


@pytest.mark.skipif(not ref_import.reference_available() or
                    not glob.glob("/root/reference/experiments/*/pretrained_models/*.pth"),
                    reason="the reference's pretrained checkpoints are not present")
def test_live_checkpoints_strict_load_into_implicit_nets():
    for path in sorted(glob.glob("/root/reference/experiments/*/pretrained_models/*.pth")):
        sd = torch.load(path, map_location="cpu", weights_only=False)
        pre = "feature_extractor."
        if all(k.startswith(pre) for k in sd):
            sd = {k[len(pre):]: v for k, v in sd.items()}
        net = _net_from_manifest_keys({k: list(v.shape) for k, v in sd.items()}, diffusion_method="implicit_dense")
        net.load_state_dict(sd, strict=True)
