"""fp64 numpy/scipy restatement of the functional-map head (TEST INFRASTRUCTURE ONLY; never imported by the package).

Citations are to /root/reference/experiments/functional_correspondence/:
  * ``solve`` / ``compute_correspondence``: fmaps_model.py:11-40 (the per-row inverse as a per-row ``cho_factor`` /
    ``cho_solve`` of S_i = A A^T + lambda diag(D[i, :]), D[i][j] = (evals_x[j] - evals_y[i])^2);
  * ``solve_adjoint``: its reverse mode, w_i = S_i^-1 g_i, dB = W A, dA = W^T B - sum_i (w_i c_i^T + c_i w_i^T) A;
  * ``nearest_neighbor``: brute-force fp64 1-NN, what functional_correspondence.py:194-196 computes with
    ``find_knn(..., k=1, method='cpu_kd')``, plus each query's best and second-best distance.
"""
from __future__ import annotations

import numpy as np
from scipy.linalg import cho_factor, cho_solve


def solve(A, B, evals_x, evals_y, lam, with_factors=False):
    """C (n, n), row i = S_i^-1 A b_i (fmaps_model.py:26-38); A, B (n, d) are F_hat, G_hat."""
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    ex, ey = np.asarray(evals_x, np.float64), np.asarray(evals_y, np.float64)
    n = A.shape[0]
    AAt, BAt = A @ A.T, B @ A.T                                                # :31-33
    D = (ex[None, :] - ey[:, None]) ** 2                                       # :26-27
    C = np.empty((n, n))
    facs = []
    for i in range(n):                                                         # :35-38
        f = cho_factor(AAt + lam * np.diag(D[i]), lower=True)
        C[i] = cho_solve(f, BAt[i])
        facs.append(f)
    return (C, facs) if with_factors else C


def solve_adjoint(A, B, evals_x, evals_y, lam, gC):
    """(dA, dB) of sum(gC * C) for C = solve(A, B, ...)."""
    A, B, gC = np.asarray(A, np.float64), np.asarray(B, np.float64), np.asarray(gC, np.float64)
    C, facs = solve(A, B, evals_x, evals_y, lam, with_factors=True)
    W = np.stack([cho_solve(f, gC[i]) for i, f in enumerate(facs)])
    M = W.T @ C + C.T @ W
    return W.T @ B - M @ A, W @ A


def compute_correspondence(feat_x, feat_y, evals_x, evals_y, evecs_trans_x, evecs_trans_y, lambda_param=1e-3):
    """fmaps_model.py:11-40 in fp64: (n, n) (the reference returns (1, n, n))."""
    A = np.asarray(evecs_trans_x, np.float64) @ np.asarray(feat_x, np.float64)   # :22
    B = np.asarray(evecs_trans_y, np.float64) @ np.asarray(feat_y, np.float64)   # :23
    return solve(A, B, evals_x, evals_y, lambda_param)


def spectral(feat, evecs, mass, n):
    """fmaps_model.py:79's evecs.t()[:n] @ diag(mass) @ feat, without the diagonal matrix."""
    return np.asarray(evecs, np.float64)[:, :n].T @ (np.asarray(mass, np.float64)[:, None] * np.asarray(feat, np.float64))


def model_torch(params, shape1, shape2, n=30, lam=1e-3):
    """fmaps_model.py:62-83 in float64 torch on the CPU (the autograd gold of the model's parameter gradients):
    ``params`` the model's state dict (``feature_extractor.*``, float64 tensors, requires_grad as wanted), each shape
    ``(x, mass, evals, evecs, gradX, gradY)`` in float64 with sparse COO gradX / gradY.  The feature extractor is
    ``dn_oracle_torch.block_forward`` between first_lin and last_lin (layers.py:364-377, outputs at vertices, no
    dropout); the head is :79-81 without the diagonal matrix and :26-38 with a solve per row.  Returns (C, feat1,
    feat2)."""
    import torch
    import dn_oracle_torch as T
    pre = "feature_extractor."
    p = {k[len(pre):]: v for k, v in params.items() if k.startswith(pre)}
    n_block = len([k for k in p if k.endswith("diffusion.diffusion_time")])
    feats, specs = [], []
    for x, mass, evals, evecs, gX, gY in (shape1, shape2):
        h = torch.addmm(p["first_lin.bias"], x, p["first_lin.weight"].t())
        for b in range(n_block):
            bp = {k[len("block_%d." % b):]: v for k, v in p.items() if k.startswith("block_%d." % b)}
            h = T.block_forward(h[None], mass[None], evals[None], evecs[None], [gX], [gY], bp)[0]
        f = torch.addmm(p["last_lin.bias"], h, p["last_lin.weight"].t())
        feats.append(f)
        specs.append(evecs[:, :n].t() @ (mass[:, None] * f))
    A, B = specs
    ex, ey = shape1[2][:n], shape2[2][:n]
    D = (ex[None, :] - ey[:, None]) ** 2
    AAt, BAt = A @ A.t(), B @ A.t()
    C = torch.stack([torch.linalg.solve(AAt + lam * torch.diag(D[i]), BAt[i]) for i in range(n)])
    return C, feats[0], feats[1]


def fixture_model_gold(fx, n=30, lam=1e-3):
    """``model_torch`` on the two shapes and the float16 weights of ``tests/golden/fmaps_small``, float64 on the CPU:
    returns (C, feat1, feat2, params) with the params dict requiring grad, for autograd golds."""
    import torch
    d = torch.float64
    params = {k[2:]: torch.from_numpy(v.astype(np.float64)).requires_grad_(True) for k, v in fx.items()
              if k.startswith("p:")}

    def shape(tag):
        f = lambda k: torch.from_numpy(np.asarray(fx[tag + ":" + k]))
        V = f("mass").shape[0]
        sp = lambda i, v: torch.sparse_coo_tensor(f(i), f(v).to(d), (V, V)).coalesce()
        return (f("verts").to(d), f("mass").to(d), f("evals").to(d), f("evecs").to(d), sp("gradX_idx", "gradX_vals"),
                sp("gradY_idx", "gradY_vals"))

    C, f1, f2 = model_torch(params, shape("x"), shape("y"), n=n, lam=lam)
    return C, f1, f2, params


def nearest_neighbor(source, target):
    """For every row of ``source`` the fp64 argmin over the rows of ``target`` (lowest index on ties) of the squared
    distance, and the best and second-best squared distances."""
    s, t = np.asarray(source, np.float64), np.asarray(target, np.float64)
    idx = np.empty(len(s), np.int64)
    d1, d2 = np.empty(len(s)), np.empty(len(s))
    chunk = max(1, 2_000_000 // max(len(t), 1))
    tt = np.ascontiguousarray(t.T)
    for a in range(0, len(s), chunk):
        q = s[a:a + chunk]
        d = np.zeros((len(q), len(t)))
        for k in range(s.shape[1]):
            d += (q[:, k:k + 1] - tt[k][None, :]) ** 2
        i = np.argmin(d, axis=1)
        idx[a:a + chunk] = i
        r = np.arange(len(q))
        d1[a:a + chunk] = d[r, i]
        d[r, i] = np.inf
        d2[a:a + chunk] = d.min(axis=1) if d.shape[1] > 1 else np.inf
    return idx, d1, d2
