"""CPU restatement (numpy/scipy, fp64) of the reference's implicit heat diffusion, ``LearnedTimeDiffusion`` with
``method='implicit_dense'`` (layers.py:69-84).

TEST INFRASTRUCTURE ONLY, like ``dn_oracle``: the gold that ``ops.ImplicitDiffusionFn`` is checked against at sizes where
the reference's dense (B, C, V, V) Cholesky does not fit.  Pinned by ``tests/test_implicit_oracle.py`` against what the
live reference computed (``tests/golden/implicit_small.npz``, from ``oracle/make_golden_implicit.py``).  Citations are to
``/root/reference/src/diffusion_net/layers.py``.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp


def implicit_diffusion(x, mass, L, diffusion_time, grad_out=None):
    """layers.py:69-84 (method='implicit_dense') in fp64 for one mesh: per channel c, y_c = (M + t_c L)^-1 M x_c with
    t clamped at 1e-8 (:48-49), by a sparse direct solve (scipy ``splu``, one factorisation per channel) instead of the
    reference's dense Cholesky.  ``x`` (V, C) or (B, V, C) (B inputs on the same mesh), ``mass`` (V), ``L`` any scipy
    sparse (V, V) matrix.  Returns y, or with ``grad_out`` (shaped like x) the adjoint too, ``(y, grad_x, grad_time)``:
    w_c = A_c^-T g_c, grad_x = M w, grad_time_c = -w_c . (L y_c) (L symmetric), shaped (B, C) for B inputs."""
    import scipy.sparse.linalg as sla
    x = np.asarray(x, dtype=np.float64)
    xb = x[None] if x.ndim == 2 else x
    gb = None if grad_out is None else np.asarray(grad_out, dtype=np.float64).reshape(xb.shape)
    m = np.asarray(mass, dtype=np.float64)
    L = sp.csc_matrix(L, dtype=np.float64)
    t = np.maximum(np.asarray(diffusion_time, dtype=np.float64), 1e-8)
    y = np.empty_like(xb)
    w = np.empty_like(xb)
    for c in range(xb.shape[2]):
        lu = sla.splu((sp.diags(m) + t[c] * L).tocsc())
        for b in range(xb.shape[0]):
            y[b, :, c] = lu.solve(m * xb[b, :, c])
            if gb is not None:
                w[b, :, c] = lu.solve(gb[b, :, c], trans="T")
    shape = x.shape
    if gb is None:
        return y.reshape(shape)
    gt = -np.stack([np.einsum("vc,vc->c", w[b], L @ y[b]) for b in range(xb.shape[0])])
    return y.reshape(shape), (m[:, None] * w).reshape(shape), gt[0] if x.ndim == 2 else gt
