"""CPU checks of the functional-map oracle (oracle/dn_oracle_fmaps.py) against what the live reference computed
(tests/golden/fmaps_small.*.npz, from oracle/make_golden_fmaps.py), and of the model's state_dict layout.  No GPU here."""
import os
import sys

import numpy as np
import torch

from conftest import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle_fmaps as OF  # noqa: E402

import diffusion_net_b200 as dn  # noqa: E402

N = 30
LAMBDA = 1e-3


def _spectral(fx, tag, feat):
    return OF.spectral(feat, fx[tag + ":evecs"], fx[tag + ":mass"], N)


def test_oracle_matches_reference_correspondence():
    fx = load_golden("fmaps_small")
    A = _spectral(fx, "x", fx["feat1_64"])
    B = _spectral(fx, "y", fx["feat2_64"])
    C = OF.solve(A, B, fx["x:evals"][:N], fx["y:evals"][:N], LAMBDA)
    gold = fx["C64"]
    assert np.abs(C - gold).max() <= 1e-10 * np.abs(gold).max()
    # the same through the reference's own signature (evecs_trans = evecs.t()[:n] @ diag(mass))
    et = lambda tag: fx[tag + ":evecs"].astype(np.float64)[:, :N].T * fx[tag + ":mass"].astype(np.float64)[None, :]
    C2 = OF.compute_correspondence(fx["feat1_64"], fx["feat2_64"], fx["x:evals"][:N], fx["y:evals"][:N], et("x"),
                                   et("y"), LAMBDA)
    assert np.abs(C2 - gold).max() <= 1e-10 * np.abs(gold).max()


def test_composed_fp64_model_matches_reference():
    """dn_oracle_fmaps.model_torch (the GPU tests' gradient gold) reproduces the reference's fp64 run: C, both feature
    sets and every recorded parameter gradient of mean((C_pred - C_gt)^2)."""
    fx = load_golden("fmaps_small")
    C, f1, f2, prm = OF.fixture_model_gold(fx, n=N, lam=LAMBDA)
    for mine, key in ((C, "C64"), (f1, "feat1_64"), (f2, "feat2_64")):
        gold = fx[key]
        assert np.abs(mine.detach().numpy() - gold).max() <= 1e-10 * np.abs(gold).max(), key
    torch.mean(torch.square(C - torch.from_numpy(fx["C_gt"]))).backward()
    keys = [k[5:] for k in fx if k.startswith("grad:")]
    assert len(keys) == 3 + 4 * 4          # first_lin, last_lin.bias; per block the time and three biases
    for k in keys:
        gold = fx["grad:" + k]
        assert np.abs(prm[k].grad.numpy() - gold).max() <= 1e-10 * np.abs(gold).max(), k
    assert set(k[10:] for k in fx if k.startswith("gradfloor:")) == set(prm)


def _torch_solve(A, B, ex, ey, lam):
    """float64 torch restatement of fmaps_model.py:26-38 (explicit inverse per row, as the reference)."""
    D = (ex[None, :] - ey[:, None]) ** 2
    AAt, BAt = A @ A.T, B @ A.T
    return torch.stack([torch.linalg.inv(AAt + lam * torch.diag(D[i])) @ BAt[i] for i in range(A.shape[0])])


def test_oracle_adjoint_matches_autograd():
    rs = np.random.RandomState(0)
    n, d = 12, 20
    A, B = rs.randn(n, d), rs.randn(n, d)
    ex, ey = np.sort(rs.rand(n)) * 10, np.sort(rs.rand(n)) * 10
    g = rs.randn(n, n)
    dA, dB = OF.solve_adjoint(A, B, ex, ey, 0.1, g)
    At, Bt = torch.tensor(A, requires_grad=True), torch.tensor(B, requires_grad=True)
    (_torch_solve(At, Bt, torch.tensor(ex), torch.tensor(ey), 0.1) * torch.tensor(g)).sum().backward()
    assert np.abs(dA - At.grad.numpy()).max() <= 1e-10 * np.abs(dA).max()
    assert np.abs(dB - Bt.grad.numpy()).max() <= 1e-10 * np.abs(dB).max()


def test_oracle_nearest_neighbor_matches_reference_kd_tree():
    fx = load_golden("fmaps_small")
    idx, d1, d2 = OF.nearest_neighbor(fx["y:evecs"][:, :N], fx["map_target"])
    assert np.array_equal(idx, fx["map"])
    assert np.array_equal(d1, fx["map_d1"]) and np.array_equal(d2, fx["map_d2"])
    assert (d2 > d1).all()


def test_model_state_dict_strict_loads_checkpoint():
    fx = load_golden("fmaps_small")
    sd = {k[2:]: torch.from_numpy(v.astype(np.float32)) for k, v in fx.items() if k.startswith("p:")}
    assert all(k.startswith("feature_extractor.") for k in sd)
    m = dn.FunctionalMapCorrespondenceWithDiffusionNetFeatures(n_feat=128, n_fmap=50, input_features="xyz")
    m.load_state_dict(sd, strict=True)
    assert m.n_fmap == 30     # the reference's quirk: the argument is ignored
    assert set(m.state_dict()) == set(sd)
    assert dn.FunctionalMapCorrespondenceWithDiffusionNetFeatures(input_features="hks").feature_extractor.C_in == 16
