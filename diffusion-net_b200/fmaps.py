"""The functional-map correspondence model (reference ``experiments/functional_correspondence/fmaps_model.py``) and its
evaluation's pointwise map (``functional_correspondence.py:194-196``) on the GPU.

* ``compute_correspondence`` / ``FmapSolveFn``: the regularised functional-map solve, one launch forward and two
  backward (``dn_fmap_solve_fwd`` / ``_bwd``: an fp64 Cholesky per row), with no host synchronisation: a pair
  training step captures in ``graphs.GraphedTrainStep``.  Where the reference's ``torch.inverse`` raises on a singular
  system, the affected row of C is NaN here.
* ``FunctionalMapCorrespondenceWithDiffusionNetFeatures``: the reference module (same kwargs, ``feature_extractor.*``
  state_dict keys, forward).  The spectral projection is ``to_basis(feat, evecs[:, :n_fmap], mass)``: the reference's
  dense ``evecs.t()[:n_fmap] @ torch.diag(mass)`` (a V x V matrix) is never formed.
* ``pointwise_map`` / ``nearest_neighbor``: the vertex-to-vertex map by an exact fp32 nearest-neighbour search
  (``dn_nearest_neighbor``), instead of the reference's host KD-tree.
"""
from __future__ import annotations

import ctypes as C
import weakref

import torch
import torch.nn as nn

from . import _lib, ops
from .layers import DiffusionNet

MAX_FMAP = 128       # n cap of dn_fmap_solve_* and dn_nearest_neighbor


def _check_n(n, what):
    if n > MAX_FMAP:
        raise RuntimeError("diffusion_net_b200 {}: n = {} exceeds the supported maximum of {}".format(what, n, MAX_FMAP))


class FmapSolveFn(torch.autograd.Function):
    """fmaps_model.py:22-38 from the spectral features: C (n, n) with row i solving
    (A A^T + lambda diag((evals_x - evals_y[i])^2)) c_i = A B[i]^T.  Differentiable in A and B; the eigenvalues and lambda
    are data (SURVEY.md section 8a)."""

    @staticmethod
    @ops._device_guard
    def forward(ctx, A, B, evals_x, evals_y, lambda_param):
        ops._require_cuda(A, B, evals_x, evals_y)
        A, B, ex, ey = ops._f32c(A), ops._f32c(B), ops._f32c(evals_x), ops._f32c(evals_y)
        if A.dim() != 2 or A.shape != B.shape or ex.shape != (A.shape[0],) or ey.shape != (A.shape[0],):
            raise ValueError("fmap solve: A {} and B {} must be (n, d), evals_x {} and evals_y {} (n)".format(
                tuple(A.shape), tuple(B.shape), tuple(ex.shape), tuple(ey.shape)))
        n, d = A.shape
        _check_n(n, "functional-map solve")
        out = torch.empty(n, n, dtype=torch.float32, device=A.device)
        _lib.check(_lib.load().dn_fmap_solve_fwd(A.data_ptr(), B.data_ptr(), ex.data_ptr(), ey.data_ptr(), n, d,
                                                 float(lambda_param), out.data_ptr(), ops._stream()),
                   "dn_fmap_solve_fwd")
        ctx.lam = float(lambda_param)
        ctx.save_for_backward(A, B, ex, ey)
        return out

    @staticmethod
    @ops._device_guard
    def backward(ctx, g):
        A, B, ex, ey = ctx.saved_tensors
        g = ops._f32c(g)
        n, d = A.shape
        gA, gB = torch.empty_like(A), torch.empty_like(B)
        ws = torch.empty(16 * n * n, dtype=torch.uint8, device=A.device)
        _lib.check(_lib.load().dn_fmap_solve_bwd(A.data_ptr(), B.data_ptr(), ex.data_ptr(), ey.data_ptr(), n, d, ctx.lam,
                                                 g.data_ptr(), gA.data_ptr(), gB.data_ptr(), ws.data_ptr(), ws.numel(),
                                                 ops._stream()), "dn_fmap_solve_bwd")
        return gA, gB, None, None, None


def fmap_solve(A, B, evals_x, evals_y, lambda_param=1e-3):
    """C (n, n) from the spectral features A = F_hat, B = G_hat (n, d); see FmapSolveFn."""
    if torch.is_grad_enabled():
        ops._no_operator_grads(("evals_x", evals_x), ("evals_y", evals_y))
    return FmapSolveFn.apply(A, B, evals_x, evals_y, lambda_param)


# ------------------------------------------------------------------------------------------------
# the spectral projection: the basis padded with zero columns to a multiple of 4, so that the tensor-core to_basis
# kernels (K % 4 == 0) take n_fmap = 30; memoised on the identity and version of the source tensor, as
# ops.prepare_operators is, so a resident mesh pads once
# ------------------------------------------------------------------------------------------------
_basis_cache = {}


def _padded(src, n, transpose):
    """(V, ceil4(n)) contiguous fp32: the first n columns of ``src`` (V, >= n), or of ``src.T`` for ``src`` (n, V), then
    zero columns."""
    key = (id(src), n, transpose)
    hit = _basis_cache.get(key)
    if hit is not None and hit[0]() is src and hit[1] == src._version:
        return hit[2]
    cols = src[:n].t() if transpose else src[:, :n]
    kp = (n + 3) // 4 * 4
    out = torch.zeros(cols.shape[0], kp, dtype=torch.float32, device=src.device)
    out[:, :n] = cols
    _basis_cache[key] = (weakref.ref(src), src._version, out)
    weakref.finalize(src, _basis_cache.pop, key, None)
    return out


def _project(feat, basis_padded, n, mass):
    """(n, d) spectral features basis^T (mass * feat); the padded rows beyond n are dropped (a contiguous view)."""
    return ops.to_basis(feat, basis_padded, mass)[:n]


def compute_correspondence(feat_x, feat_y, evals_x, evals_y, evecs_trans_x, evecs_trans_y, lambda_param=1e-3):
    """Drop-in for the reference's ``compute_correspondence`` (fmaps_model.py:11-40): the same arguments (features (V, d),
    evals (n), evecs_trans (n, V), the reference's ``evecs.t()[:n] @ diag(mass)``) and the same (1, n, n) output.
    F_hat = evecs_trans @ feat runs on the to_basis kernels with basis evecs_trans^T and no mass; gradients reach feat_x
    and feat_y.  A singular row of the system is NaN here, where the reference's torch.inverse raises."""
    ops._require_cuda(feat_x, feat_y, evals_x, evals_y, evecs_trans_x, evecs_trans_y)
    n = evecs_trans_x.shape[0]
    if evecs_trans_y.shape[0] != n or evals_x.shape != (n,) or evals_y.shape != (n,):
        raise ValueError("compute_correspondence: evecs_trans_x {}, evecs_trans_y {}, evals_x {}, evals_y {} disagree".format(
            tuple(evecs_trans_x.shape), tuple(evecs_trans_y.shape), tuple(evals_x.shape), tuple(evals_y.shape)))
    _check_n(n, "compute_correspondence")
    A = _project(feat_x, _padded(evecs_trans_x, n, True), n, None)
    B = _project(feat_y, _padded(evecs_trans_y, n, True), n, None)
    return fmap_solve(A, B, evals_x, evals_y, lambda_param).unsqueeze(0)


class FunctionalMapCorrespondenceWithDiffusionNetFeatures(nn.Module):
    """fmaps_model.py:43-83: DiffusionNet features on both shapes, then the functional map between them.

    Same constructor as the reference, including its quirk: ``self.n_fmap = 30`` whatever ``n_fmap`` is passed (and
    ``lambda_`` is unused; ``lambda_param`` is the regulariser).  The state_dict keys are the reference's
    (``feature_extractor.*``), so its shipped checkpoints strict-load.  ``forward(shape1, shape2)`` takes the reference's
    11-tuples (verts, faces, frames, mass, L, evals, evecs, gradX, gradY, hks, vts) and returns (C_pred (1, n, n), feat1,
    feat2).  The spectral projection is ``to_basis(feat, evecs[:, :30], mass)``; no V x V matrix is formed."""

    def __init__(self, n_feat=128, n_fmap=30, lambda_=1e-3, input_features="xyz", lambda_param=1e-3):
        super().__init__()
        C_in = {'xyz': 3, 'hks': 16}[input_features]
        self.feature_extractor = DiffusionNet(C_in=C_in, C_out=n_feat, C_width=128, N_block=4, dropout=True)
        self.n_fmap = 30     # as the reference: the n_fmap argument is ignored
        self.input_features = input_features
        self.lambda_param = lambda_param

    def forward(self, shape1, shape2):
        verts1, faces1, frames1, mass1, L1, evals1, evecs1, gradX1, gradY1, hks1, vts1 = shape1
        verts2, faces2, frames2, mass2, L2, evals2, evecs2, gradX2, gradY2, hks2, vts2 = shape2
        if self.input_features == "xyz":
            features1, features2 = verts1, verts2
        elif self.input_features == "hks":
            features1, features2 = hks1, hks2
        feat1 = self.feature_extractor(features1, mass1, L=L1, evals=evals1, evecs=evecs1, gradX=gradX1, gradY=gradY1,
                                       faces=faces1)
        feat2 = self.feature_extractor(features2, mass2, L=L2, evals=evals2, evecs=evecs2, gradX=gradX2, gradY=gradY2,
                                       faces=faces2)
        n = self.n_fmap
        _check_n(n, "FunctionalMapCorrespondenceWithDiffusionNetFeatures")
        A = _project(feat1, _padded(evecs1, n, False), n, mass1)
        B = _project(feat2, _padded(evecs2, n, False), n, mass2)
        C_pred = fmap_solve(A, B, evals1[:n], evals2[:n], self.lambda_param).unsqueeze(0)
        return C_pred, feat1, feat2


# ------------------------------------------------------------------------------------------------
# pointwise map
# ------------------------------------------------------------------------------------------------
def nearest_neighbor(source, target):
    """int64 (Vs,): for every row of ``source`` (Vs, n) the index of the nearest row of ``target`` (Vt, n), n <= 128, by
    exact fp32 squared distances (dn_nearest_neighbor); ties go to the lowest index.  ``find_knn(source, target, k=1)``
    of the reference's geometry.py."""
    ops._require_cuda(source, target)
    source, target = ops._f32c(source), ops._f32c(target)
    if source.dim() != 2 or target.dim() != 2 or source.shape[1] != target.shape[1] or target.shape[0] == 0:
        raise ValueError("nearest_neighbor: source {} and target {} must be (Vs, n) and (Vt, n) with Vt > 0".format(
            tuple(source.shape), tuple(target.shape)))
    Vs, n = source.shape
    Vt = target.shape[0]
    _check_n(n, "nearest_neighbor")
    out = torch.empty(Vs, dtype=torch.int64, device=source.device)
    lib = _lib.load()
    with ops._on(source):
        ws = torch.empty(max(int(lib.dn_nearest_neighbor_workspace_bytes(Vs, Vt, n)), 1), dtype=torch.uint8,
                         device=source.device)
        _lib.check(lib.dn_nearest_neighbor(source.data_ptr(), Vs, target.data_ptr(), Vt, n, out.data_ptr(),
                                           ws.data_ptr(), ws.numel(), ops._stream()), "dn_nearest_neighbor")
    return out


def _apply_basis_exact(values, basis):
    """basis (V, K) @ values (K, Cc) on the exact fp32 SIMT engine (dn_from_basis), whatever ops' engine is."""
    V, K = basis.shape
    Cc = values.shape[1]
    out = torch.empty(V, Cc, dtype=torch.float32, device=values.device)
    with ops._on(values):
        ws = ops.workspace(V, K, Cc, values.device)
        _lib.check(_lib.load().dn_from_basis(values.data_ptr(), basis.data_ptr(), None, V, K, Cc, out.data_ptr(),
                                             ws.data_ptr(), ws.numel(), _lib.ENGINE_SIMT, ops._stream()),
                   "dn_from_basis")
    return out


def pointwise_map(C, evecs_x, evecs_y, n_fmap=30):
    """The evaluation's vertex-to-vertex map (functional_correspondence.py:194-196): int64 (V_y,), for every vertex of
    shape y the index of its image on shape x, i.e. the nearest row of Phi_x[:, :n] C^T to each row of Phi_y[:, :n].  The
    product runs on the exact fp32 SIMT kernel and the search is dn_nearest_neighbor."""
    ops._require_cuda(C, evecs_x, evecs_y)
    Cm = C.squeeze(0) if C.dim() == 3 else C
    n = int(n_fmap)
    if Cm.dim() != 2 or Cm.shape[0] < n or Cm.shape[1] < n or evecs_x.shape[1] < n or evecs_y.shape[1] < n:
        raise ValueError("pointwise_map: C {}, evecs_x {}, evecs_y {} do not hold n_fmap = {}".format(
            tuple(C.shape), tuple(evecs_x.shape), tuple(evecs_y.shape), n))
    _check_n(n, "pointwise_map")
    with torch.no_grad():
        ct = ops._f32c(Cm[:n, :n].t().contiguous())
        target = _apply_basis_exact(ct, ops._f32c(evecs_x[:, :n].contiguous()))
        return nearest_neighbor(evecs_y[:, :n].contiguous(), target)
