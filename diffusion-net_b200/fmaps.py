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
* ``PairBatch`` / ``forward_pairs`` / ``pointwise_map_batch``: the same over many shape pairs in one launch sequence
  (the training and evaluation loops of functional_correspondence.py): features once per shape (``forward_batch``),
  one batched projection, one batched solve, and the pointwise maps of all pairs, each pair's result what the per-pair
  calls give.
* ``PairDataset`` / ``PairSlot``: shuffled pairs of a device-resident ``MeshDataset``, their ground-truth maps from the
  template correspondences (faust_scape_dataset.py:186-190, ``dn_fmap_ground_truth``), and fixed-buffer pair slots on
  which a whole training step, pair draw and random rotations included, captures in one CUDA graph.
"""
from __future__ import annotations

import ctypes as C
import weakref
from operator import index as operator_index

import numpy as np
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
        _lib.call("dn_fmap_solve_fwd", A, B, ex, ey, n, d, float(lambda_param), out, ops._stream())
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
        _lib.call("dn_fmap_solve_bwd", A, B, ex, ey, n, d, ctx.lam, g, gA, gB, ws, ws.numel(), ops._stream())
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

    def forward_pairs(self, pair_batch, xs):
        """Every pair of a ``PairBatch`` in one launch sequence: (C_pred (P, n, n), feats), C_pred[p] what
        ``forward(shape_{x_p}, shape_{y_p})`` gives for that pair and feats the list of per-shape features.  ``xs``: the
        per-shape inputs (verts or HKS, per ``input_features``) as a list, or one tensor in the batch layout.  The
        features run once per shape through ``feature_extractor.forward_batch``'s route, so in training mode a shape
        used by several pairs gets ONE dropout mask per step (the reference draws one per forward call); then
        ``project_batched`` and ``fmap_solve_batched``.  The loss over all pairs backpropagates through each shape's
        features once, with the per-pair gradients summed in a fixed order.

        On a ``PairSlot`` (``PairDataset.slot``; ``xs`` one tensor in the slot layout, e.g. ``slot.pack(verts,
        rotations=...)``) the same launch sequence runs on the slot's fixed buffers, so the step captures in one CUDA
        graph; ``feats`` is then the (V_cap, n_feat) features in the slot layout (a slot has no per-shape split)."""
        n = self.n_fmap
        if pair_batch.n != n:
            raise ValueError("forward_pairs: the pair batch was built for n_fmap = {}, the model uses {}".format(
                pair_batch.n, n))
        mb = pair_batch.mesh_batch
        feat = self.feature_extractor._forward_batch_layout(mb, xs)
        F_hat = project_batched(feat, pair_batch)
        C_pred = fmap_solve_batched(F_hat, pair_batch.evals, pair_batch.pairs, n, self.lambda_param)
        if isinstance(pair_batch, PairSlot):
            return C_pred, feat
        return C_pred, mb.unpack(feat)


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
    with ops._on(source):
        ws = torch.empty(max(int(_lib.load().dn_nearest_neighbor_workspace_bytes(Vs, Vt, n)), 1), dtype=torch.uint8,
                         device=source.device)
        _lib.call("dn_nearest_neighbor", source, Vs, target, Vt, n, out, ws, ws.numel(), ops._stream())
    return out


def _apply_basis_exact(values, basis):
    """basis (V, K) @ values (K, Cc) on the exact fp32 SIMT engine (dn_from_basis), whatever ops' engine is."""
    V, K = basis.shape
    Cc = values.shape[1]
    out = torch.empty(V, Cc, dtype=torch.float32, device=values.device)
    with ops._on(values):
        ws = ops.workspace(V, K, Cc, values.device)
        _lib.call("dn_from_basis", values, basis, None, V, K, Cc, out, ws, ws.numel(), _lib.ENGINE_SIMT, ops._stream())
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


# ------------------------------------------------------------------------------------------------
# pair batches: the head over many shape pairs in one launch sequence
# ------------------------------------------------------------------------------------------------
MAX_PAIRS = 65535        # grid-y limit of the batched solve
MAX_SHAPES = 1024        # dn_mesh_batch_plan gives every mesh at least one of its 1024 to_basis CTAs


class PairList:
    """Ordered pairs (x_p, y_p) of indices into ``n_shapes`` shapes, on the device, with the shape -> (pair, role) CSR the
    batched solve's backward sums over: entries 2 p + role (role 0 = x, 1 = y), each shape's in increasing order
    (increasing p, the x role of a self-pair before its y role).  Built once per pair batch."""

    def __init__(self, pairs, n_shapes, device):
        self.pairs = [(int(a), int(b)) for a, b in pairs]
        self.n_shapes = S = int(n_shapes)
        self.n_pairs = P = len(self.pairs)
        if P == 0:
            raise ValueError("a pair batch needs at least one pair")
        if P > MAX_PAIRS:
            raise ValueError("a pair batch takes at most {} pairs, got {}".format(MAX_PAIRS, P))
        for p, (a, b) in enumerate(self.pairs):
            if not (0 <= a < S and 0 <= b < S):
                raise ValueError("pair {} = ({}, {}) indexes a shape outside [0, {})".format(p, a, b, S))
        self.role_begin, self.role_list = role_csr(self.pairs, S)
        i32 = dict(dtype=torch.int32, device=device)
        self.pair_x_host = [a for a, _ in self.pairs]
        self.pair_y_host = [b for _, b in self.pairs]
        self.pair_x = torch.tensor(self.pair_x_host, **i32)
        self.pair_y = torch.tensor(self.pair_y_host, **i32)
        self._role_begin = torch.tensor(self.role_begin, **i32)
        self._role_list = torch.tensor(self.role_list, **i32)


def role_csr(pairs, n_shapes):
    """(begin [S + 1], entries [2 P]) of the shape -> (pair, role) lists: shape s owns entries[begin[s]:begin[s + 1]],
    each 2 p + role (role 0 = x, 1 = y) in increasing order."""
    lists = [[] for _ in range(n_shapes)]
    for p, (a, b) in enumerate(pairs):
        lists[a].append(2 * p)
        lists[b].append(2 * p + 1)
    begin, entries = [0], []
    for lst in lists:
        entries.extend(lst)          # already increasing: p grows, and 2p precedes 2p + 1
        begin.append(len(entries))
    return begin, entries


class PairBatch:
    """S shapes and P ordered pairs of them for ``forward_pairs`` / ``pointwise_map_batch``.  ``items`` are
    ``batch.MeshBatch`` items (mass, evals, evecs, gradX, gradY, optional faces), all with the same K >= n_fmap;
    ``pairs`` a list of (i, j).  Self-pairs, repeated shapes and shapes in no pair are allowed.  Builds once: the
    MeshBatch, the (V, n rounded up to 8) projection basis in its layout (the first n eigenvectors, then zero columns:
    32 columns at n = 30, as in the single-pair path), the (S, n) eigenvalue stack, and the device pair arrays with
    their role CSR."""

    def __init__(self, items, pairs, n_fmap=30):
        from .batch import MeshBatch
        n = int(n_fmap)
        S = len(items)
        if S < 1:
            raise ValueError("PairBatch needs at least one shape")
        if S > MAX_SHAPES:
            raise ValueError("PairBatch: {} shapes exceed the {} the mesh-batch planner takes".format(S, MAX_SHAPES))
        pairs = list(pairs)
        if not pairs:
            raise ValueError("PairBatch needs at least one pair")
        for p, (a, b) in enumerate(pairs):
            if not (0 <= int(a) < S and 0 <= int(b) < S):
                raise ValueError("PairBatch: pair {} = ({}, {}) indexes a shape outside [0, {})".format(p, a, b, S))
        _check_n(n, "PairBatch")
        if n < 1:
            raise ValueError("PairBatch: n_fmap must be at least 1, got {}".format(n))
        K = min(int(it["evals"].shape[0]) for it in items)
        if K < n:
            raise ValueError("PairBatch: K = {} eigenpairs is fewer than n_fmap = {}".format(K, n))
        self._build(MeshBatch(items), pairs, n)

    @classmethod
    def _of(cls, mb, pairs, n):
        """The pair batch of an already gathered MeshBatch (``PairDataset.batch``; the caller checked the pairs)."""
        pb = cls.__new__(cls)
        pb._build(mb, pairs, n)
        return pb

    def _build(self, mb, pairs, n):
        self.n, self.n_shapes, self.n_pairs = n, mb.n_meshes, len(pairs)
        self.mesh_batch = mb
        S = mb.n_meshes
        self.device = mb.device
        self.pairs = PairList(pairs, S, mb.device)
        self.kp = kp = (n + 7) // 8 * 8
        self.basis = torch.zeros(mb.V, kp, dtype=torch.float32, device=mb.device)
        self.basis[:, :n] = mb.evecs[:, :n]
        self.evals = mb.evals[:, :n].contiguous()
        self.row_begin_host = mb.row_begin[:-1]
        self.n_rows_host = mb.n_rows


def _spectral_ws(pb, Cc):
    mb = pb.mesh_batch
    return ops.workspace(mb.V, pb.kp, Cc, mb.device, extra=ops.batched_diffusion_workspace_extra(mb.n_meshes, pb.kp, Cc))


class ProjectBatchedFn(torch.autograd.Function):
    """(S, kp, C) spectral features Phi_s^T M_s F_s of every shape of a PairBatch from the (V, C) per-vertex features in
    its batch layout (dn_to_basis_batched); backward M_s Phi_s G_s (dn_from_basis_batched), 0 on padding rows.  Two
    launches each way, whatever S is; tensor-core engines only."""

    @staticmethod
    @ops._device_guard
    def forward(ctx, feat, pb):
        mb = pb.mesh_batch
        feat = ops._f32c(feat)
        if feat.dim() != 2 or feat.shape[0] != mb.V:
            raise ValueError("project_batched: features {} are not in the pair batch's layout ({} rows)".format(
                tuple(feat.shape), mb.V))
        Cc = feat.shape[1]
        out = torch.empty(mb.n_meshes, pb.kp, Cc, dtype=torch.float32, device=feat.device)
        ws = _spectral_ws(pb, Cc)
        _lib.call("dn_to_basis_batched", feat, pb.basis, mb.mass, C.byref(mb.desc), mb.V, pb.kp, Cc, out, ws, ws.numel(),
                  ops._engine, ops._stream())
        ctx.pb = pb
        return out

    @staticmethod
    @ops._device_guard
    def backward(ctx, g):
        pb = ctx.pb
        mb = pb.mesh_batch
        g = ops._f32c(g)
        Cc = g.shape[2]
        gx = torch.empty(mb.V, Cc, dtype=torch.float32, device=g.device)
        ws = _spectral_ws(pb, Cc)
        _lib.call("dn_from_basis_batched", g, pb.basis, mb.mass, C.byref(mb.desc), mb.V, pb.kp, Cc, gx, ws, ws.numel(),
                  ops._engine, ops._stream())
        return gx, None


def project_batched(feat, pair_batch):
    """(S, kp, C): every shape's spectral features from ``feat`` (V, C) in ``pair_batch``'s layout; rows n .. kp - 1 are
    zero (zero basis columns).  Differentiable in ``feat``."""
    ops._require_cuda(feat)
    return ProjectBatchedFn.apply(feat, pair_batch)


class FmapSolveBatchedFn(torch.autograd.Function):
    """The functional-map solve of every pair of a PairList: C (P, n, n), C[p] = FmapSolveFn's C for A = F_hat[x_p][:n],
    B = F_hat[y_p][:n] and the shapes' first n eigenvalues, bitwise.  One launch forward, three backward
    (dn_fmap_solve_{fwd,bwd}_batched); the gradient of a shape is the per-pair gradients summed in a fixed order."""

    @staticmethod
    @ops._device_guard
    def forward(ctx, F_hat, evals, pairs, n, lambda_param):
        F_hat, evals = ops._f32c(F_hat), ops._f32c(evals)
        if F_hat.dim() != 3 or F_hat.shape[0] != pairs.n_shapes or F_hat.shape[1] < n or evals.dim() != 2 or \
                evals.shape[0] != pairs.n_shapes or evals.shape[1] < n:
            raise ValueError("fmap_solve_batched: F_hat {} must be (S, >= n, d) and evals {} (S, >= n) for S = {}, "
                             "n = {}".format(tuple(F_hat.shape), tuple(evals.shape), pairs.n_shapes, n))
        S, m, d = F_hat.shape
        out = torch.empty(pairs.n_pairs, n, n, dtype=torch.float32, device=F_hat.device)
        _lib.call("dn_fmap_solve_fwd_batched", F_hat, m * d, evals, evals.shape[1], S, pairs.pair_x, pairs.pair_y,
                  pairs.n_pairs, n, d, float(lambda_param), out, ops._stream())
        ctx.pairs, ctx.n, ctx.lam = pairs, n, float(lambda_param)
        ctx.save_for_backward(F_hat, evals)
        return out

    @staticmethod
    @ops._device_guard
    def backward(ctx, g):
        F_hat, evals = ctx.saved_tensors
        pairs, n = ctx.pairs, ctx.n
        g = ops._f32c(g)
        S, m, d = F_hat.shape
        gF = torch.zeros_like(F_hat)
        ws = torch.empty(int(_lib.load().dn_fmap_solve_batched_workspace_bytes(pairs.n_pairs, n, d)), dtype=torch.uint8,
                         device=F_hat.device)
        _lib.call("dn_fmap_solve_bwd_batched", F_hat, m * d, evals, evals.shape[1], S, pairs.pair_x, pairs.pair_y,
                  pairs.n_pairs, pairs._role_begin, pairs._role_list, n, d, ctx.lam, g, gF, ws, ws.numel(),
                  ops._stream())
        return gF, None, None, None, None


def fmap_solve_batched(F_hat, evals, pairs, n, lambda_param=1e-3):
    """C (P, n, n) for every pair of ``pairs`` (a PairList) from the stacked spectral features ``F_hat`` (S, >= n, d; the
    first n rows of each shape used) and eigenvalues ``evals`` (S, >= n).  Differentiable in F_hat."""
    ops._require_cuda(F_hat, evals)
    _check_n(int(n), "functional-map solve")
    if torch.is_grad_enabled():
        ops._no_operator_grads(("evals", evals))
    return FmapSolveBatchedFn.apply(F_hat, evals, pairs, int(n), lambda_param)


def pointwise_map_batch(C_pred, pair_batch, n_fmap=30):
    """``pointwise_map`` for every pair of ``pair_batch``: a list of P int64 tensors (V_{y_p},), the p-th bitwise equal to
    ``pointwise_map(C_pred[p], evecs_{x_p}, evecs_{y_p}, n_fmap)``.  C_pred is (P, >= n, >= n).  The products and the
    searches of all pairs run in chunks of up to 64 pairs, 2 or 3 launches per chunk (dn_fmap_pointwise_map_batched)."""
    ops._require_cuda(C_pred)
    n = int(n_fmap)
    pb = pair_batch
    mb = pb.mesh_batch
    P = pb.n_pairs
    if C_pred.dim() != 3 or C_pred.shape[0] != P or C_pred.shape[1] < n or C_pred.shape[2] < n or mb.K < n:
        raise ValueError("pointwise_map_batch: C_pred {} does not hold {} pairs of n_fmap = {} (K = {})".format(
            tuple(C_pred.shape), P, n, mb.K))
    _check_n(n, "pointwise_map_batch")
    px, py = _lib.int_array(pb.pairs.pair_x_host), _lib.int_array(pb.pairs.pair_y_host)
    rb, nr = _lib.int_array(pb.row_begin_host), _lib.int_array(pb.n_rows_host)
    counts = [pb.n_rows_host[y] for y in pb.pairs.pair_y_host]
    with torch.no_grad(), ops._on(C_pred):
        Cm = ops._f32c(C_pred[:, :n, :n].contiguous())
        out = torch.empty(sum(counts), dtype=torch.int64, device=C_pred.device)
        wsb = int(_lib.load().dn_fmap_pointwise_map_batched_workspace_bytes(n, P, px, py, rb, nr, pb.n_shapes))
        if wsb < 0:
            _lib.check(wsb, "dn_fmap_pointwise_map_batched_workspace_bytes")
        ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=C_pred.device)
        _lib.call("dn_fmap_pointwise_map_batched", Cm, n, mb.evecs, mb.K, rb, nr, pb.n_shapes, px, py, P, out, ws,
                  ws.numel(), ops._stream())
    return list(torch.split(out, counts))


# ------------------------------------------------------------------------------------------------
# pair datasets: shuffled pairs of a MeshDataset, their ground-truth maps, and pair slots for CUDA-graph training
# ------------------------------------------------------------------------------------------------
_GT_BAD_PAIR, _GT_SINGULAR = 1, 2


def _ground_truth_into(pds, ids, out, status, ws):
    """dn_fmap_ground_truth of device int64 pair ids into ``out`` (P, n, n); ``ws`` sized for P."""
    _lib.call("dn_fmap_ground_truth", pds.ds.evecs, pds.ds.K, pds.n, pds._vts_rows, pds._vts_begin, pds.ds.n_meshes,
              pds.pairs, pds.n_table, ids, ids.shape[0], pds.max_m, out, status, ws, ws.numel(), ops._stream())
    return out


def _gt_workspace(pds, P):
    b = int(_lib.load().dn_fmap_ground_truth_workspace_bytes(P, pds.n, pds.max_m))
    if b < 0:
        _lib.check(b, "dn_fmap_ground_truth_workspace_bytes")
    return torch.empty(b, dtype=torch.uint8, device=pds.device)


def _raise_gt_status(st, n_table):
    kind, pos, pid = st
    if kind == _GT_BAD_PAIR:
        raise IndexError("pair index {} at position {} is outside the dataset's {} pairs".format(pid, pos, n_table))
    if kind == _GT_SINGULAR:
        raise RuntimeError("pair {} at position {}: the ground-truth system A^T A is singular (its correspondences "
                           "do not determine an n x n map); its C_gt is NaN".format(pid, pos))


class PairDataset:
    """Ordered shape pairs of a ``batch.MeshDataset`` with their correspondences, for the functional-map model's
    training loop (functional_correspondence.py:100-143) on the device.

    ``ds``: the MeshDataset (K >= n_fmap eigenpairs); ``vts``: one int64 tensor per mesh, the vertex of that mesh
    matching each template vertex (faust_scape_dataset.py's ``vts``; repeats allowed); ``pairs``: the table of allowed
    ordered pairs (x, y), e.g. ``itertools.permutations(range(80), 2)`` as the reference trains FAUST.  Checked once on
    the host: indices, vertices inside their mesh, ``len(vts[x]) == len(vts[y])`` for every pair.  The correspondences,
    rebased to dataset rows and concatenated, and the pair table stay on the device.

    * ``batch(pair_ids)``: the eager ``PairBatch`` of those pairs (``ds.batch(xs + ys)`` with pairs (p, P + p)), for
      ``forward_pairs`` and ``pointwise_map_batch``.
    * ``ground_truth(pair_ids)``: (P, n, n) ground-truth maps (``dn_fmap_ground_truth``).
    * ``slot(n_pairs)``: a ``PairSlot`` whose whole training step, pair draw included, captures in one CUDA graph.

    The ground truth is the reference's least squares C_gt = X^T, X = argmin ||Phi_x[vts_x, :n] X -
    Phi_y[vts_y, :n]||, solved by fp64 normal equations.  Where the reference's ``lstsq`` returns some solution for a
    rank-deficient system (fewer than n distinct correspondence rows, say), that pair's C_gt here is NaN and a status
    is set that ``check()`` (or ``PairSlot.check()``) raises on."""

    def __init__(self, ds, vts, pairs, n_fmap=30):
        n = int(n_fmap)
        _check_n(n, "PairDataset")
        if n < 1:
            raise ValueError("PairDataset: n_fmap must be at least 1, got {}".format(n))
        if ds.K < n:
            raise ValueError("PairDataset: K = {} eigenpairs is fewer than n_fmap = {}".format(ds.K, n))
        vts = list(vts)
        if len(vts) != ds.n_meshes:
            raise ValueError("PairDataset: {} correspondence tensors for {} meshes".format(len(vts), ds.n_meshes))
        host = []
        for s, v in enumerate(vts):
            v = torch.as_tensor(v)
            if v.dim() != 1 or v.dtype.is_floating_point or v.dtype.is_complex or v.dtype == torch.bool:
                raise ValueError("PairDataset: vts[{}] must be a 1-D integer tensor, got {} of shape {}".format(
                    s, v.dtype, tuple(v.shape)))
            v = v.cpu().to(torch.int64)
            if v.numel() and (int(v.min()) < 0 or int(v.max()) >= ds.n_rows[s]):
                raise IndexError("PairDataset: vts[{}] holds a vertex outside the mesh's {} vertices".format(
                    s, ds.n_rows[s]))
            host.append(v)
        counts = [int(v.numel()) for v in host]
        table = torch.as_tensor([[int(a), int(b)] for a, b in pairs], dtype=torch.int64).reshape(-1, 2)
        if table.shape[0] == 0:
            raise ValueError("PairDataset needs at least one pair")
        S = ds.n_meshes
        for p, (a, b) in enumerate(table.tolist()):
            if not (0 <= a < S and 0 <= b < S):
                raise ValueError("PairDataset: pair {} = ({}, {}) indexes a mesh outside [0, {})".format(p, a, b, S))
            if counts[a] != counts[b]:
                raise ValueError("PairDataset: pair {} = ({}, {}) has {} and {} correspondences; the ground truth needs "
                                 "as many on both shapes".format(p, a, b, counts[a], counts[b]))
        self.ds, self.n, self.device = ds, n, ds.device
        self.n_table = int(table.shape[0])
        self.pair_x_host = table[:, 0].tolist()
        self.pair_y_host = table[:, 1].tolist()
        self.max_m = max(counts[a] for a in self.pair_x_host)
        self.pairs = table.to(ds.device)
        self._vts_rows = torch.cat([v + r0 for v, r0 in zip(host, ds.row_begin)]).to(ds.device)
        self._vts_begin = torch.tensor([0] + np.cumsum(counts).tolist(), dtype=torch.int64).to(ds.device)
        self.status = torch.zeros(3, dtype=torch.int64, device=ds.device)

    def __len__(self):
        return self.n_table

    def _host_ids(self, ids, what):
        if torch.is_tensor(ids):
            ids = ids.tolist()
        ids = [int(i) for i in ids]
        if not ids:
            raise ValueError("PairDataset.{} needs at least one pair index".format(what))
        bad = [(q, i) for q, i in enumerate(ids) if not 0 <= i < self.n_table]
        if bad:
            raise IndexError("PairDataset.{}: pair index {} at position {} is outside the dataset's {} pairs".format(
                what, bad[0][1], bad[0][0], self.n_table))
        return ids

    def batch(self, pair_ids):
        """The ``PairBatch`` of pairs ``pair_ids`` (host ints; repeats allowed): shapes x_0 .. x_{P-1}, y_0 ..
        y_{P-1} drawn by one ``ds.batch`` and pairs (p, P + p)."""
        ids = self._host_ids(pair_ids, "batch")
        if 2 * len(ids) > MAX_SHAPES:
            raise ValueError("PairDataset.batch: {} pairs need {} shapes, more than the {} a pair batch takes".format(
                len(ids), 2 * len(ids), MAX_SHAPES))
        P = len(ids)
        mb = self.ds.batch([self.pair_x_host[i] for i in ids] + [self.pair_y_host[i] for i in ids])
        return PairBatch._of(mb, [(p, P + p) for p in range(P)], self.n)

    def ground_truth(self, pair_ids):
        """(P, n, n) float32 ground-truth maps of pairs ``pair_ids``: host ints (checked here) or a CUDA int64 tensor
        (checked on the device: an invalid index gives a NaN map and sets the status ``check()`` reads).  Two
        launches, no host synchronisation for device ids."""
        if torch.is_tensor(pair_ids) and pair_ids.device.type != "cpu":
            if pair_ids.dtype != torch.int64 or pair_ids.dim() != 1 or pair_ids.device != self.device:
                raise ValueError("PairDataset.ground_truth: device pair ids must be a 1-D int64 tensor on {}".format(
                    self.device))
            ids = pair_ids.contiguous()
        else:
            ids = torch.tensor(self._host_ids(pair_ids, "ground_truth"), dtype=torch.int64).to(self.device)
        P = ids.shape[0]
        if not 1 <= P <= MAX_PAIRS:
            raise ValueError("PairDataset.ground_truth takes 1 .. {} pairs, got {}".format(MAX_PAIRS, P))
        out = torch.empty(P, self.n, self.n, dtype=torch.float32, device=self.device)
        with ops._on(out):
            return _ground_truth_into(self, ids, out, self.status, _gt_workspace(self, P))

    def check(self):
        """Raise if a ground_truth call since the last check met an invalid pair index (IndexError) or a singular
        system (RuntimeError), and clear the status.  One device-to-host read."""
        st = self.status.tolist()
        if st[0]:
            self.status.zero_()
        _raise_gt_status(st, self.n_table)

    def slot(self, n_pairs, max_rows=None, max_entries=None):
        """A ``PairSlot`` of ``n_pairs`` pairs (see there)."""
        return PairSlot(self, n_pairs, max_rows, max_entries)


class PairSlot:
    """``n_pairs`` pairs of a ``PairDataset`` on buffers that never move, refilled on the device from any pair indices,
    so that the functional-map model's whole training step (pair draw, rotations, features, projection, solve, ground
    truth, loss and backward) captures in one CUDA graph (``graphs.GraphedTrainStep``)::

        slot = pds.slot(P)
        ids = torch.zeros(P, dtype=torch.int64, device="cuda")
        def step(model, ids):
            slot.fill(ids)
            x = slot.pack(verts, rotations=dn.batch.random_rotations(2 * P, device="cuda"))
            C_pred, _ = model.forward_pairs(slot, x)
            return (C_pred - slot.ground_truth()).square().mean()
        g = dn.graphs.GraphedTrainStep(model, step, (ids,))
        for chunk in torch.randint(len(pds), (n_steps, P), device="cuda"):
            ids.copy_(chunk); g.zero_grads(model); g.replay(); opt.step()

    It wraps a ``batch.BatchSlot`` of 2 P meshes filled with ``cat(pair_x[ids], pair_y[ids])`` (``mesh_batch``), with
    the fixed ``PairList`` (p, P + p) (so the solve's shape -> (pair, role) lists never change), a fixed (V_cap, kp)
    projection basis refreshed at every fill and a fixed (P, n, n) ground-truth buffer.  The default capacity is 2 P
    times the dataset's largest padded mesh and gradient entry count: a pair draw repeats shapes, which
    ``BatchSlot``'s default (any distinct meshes) does not cover.

    A pair index outside the table gives every mesh of the slot an invalid id: the step computes NaN (loss and
    gradients), and ``check()`` raises IndexError; the next valid fill recovers.  Dropout masks are drawn over the
    whole slot layout, as ``forward_pairs`` draws them on a ``PairBatch``."""

    def __init__(self, pds, n_pairs, max_rows=None, max_entries=None):
        from .batch import BatchSlot
        P = operator_index(n_pairs)
        if P < 1 or 2 * P > MAX_SHAPES:
            raise ValueError("PairDataset.slot takes 1 .. {} pairs, got {}".format(MAX_SHAPES // 2, P))
        ds = pds.ds
        pad_max = max((r + 127) // 128 * 128 for r in ds.n_rows)
        self.pds, self.n, self.n_pairs, self.n_shapes, self.device = pds, pds.n, P, 2 * P, ds.device
        self.mesh_batch = BatchSlot(ds, 2 * P, 2 * P * pad_max if max_rows is None else max_rows,
                                    2 * P * max(ds._grad_nnz) if max_entries is None else max_entries)
        self.pairs = PairList([(p, P + p) for p in range(P)], 2 * P, ds.device)
        self.kp = kp = (self.n + 7) // 8 * 8
        self.basis = torch.zeros(self.mesh_batch.V, kp, dtype=torch.float32, device=ds.device)
        self.evals = self.mesh_batch.evals       # (2 P, K): the solve reads the first n of every row
        self.ids = torch.zeros(P, dtype=torch.int64, device=ds.device)
        self.C_gt = torch.zeros(P, self.n, self.n, dtype=torch.float32, device=ds.device)
        self.status = torch.zeros(3, dtype=torch.int64, device=ds.device)
        self._ws = _gt_workspace(pds, P)

    def fill(self, ids):
        """Draw pairs ``ids``: a CUDA int64 tensor of n_pairs pair indices (checked on the device, nothing read back)
        or host ints (checked here).  A few small torch ops map the pairs to their 2 P meshes (an invalid index to
        an invalid mesh id), then ``BatchSlot.fill`` and one copy of the basis.  Returns the slot."""
        P = self.n_pairs
        if torch.is_tensor(ids) and ids.device.type != "cpu":
            if ids.dtype != torch.int64 or tuple(ids.shape) != (P,) or ids.device != self.device:
                raise ValueError("PairSlot.fill: device ids must be an int64 tensor of shape ({},) on {}".format(
                    P, self.device))
            if ids.data_ptr() != self.ids.data_ptr():
                self.ids.copy_(ids)
        else:
            h = self.pds._host_ids(ids, "slot fill")
            if len(h) != P:
                raise ValueError("PairSlot.fill: {} pair indices for a slot of {} pairs".format(len(h), P))
            self.ids.copy_(torch.tensor(h, dtype=torch.int64).pin_memory(), non_blocking=True)
        valid = (self.ids >= 0) & (self.ids < self.pds.n_table)
        xy = torch.index_select(self.pds.pairs, 0, torch.where(valid, self.ids, 0))
        xy = torch.where(valid.unsqueeze(1), xy, -1)
        mesh_ids = self.mesh_batch.ids
        mesh_ids[:P].copy_(xy[:, 0])
        mesh_ids[P:].copy_(xy[:, 1])
        self.mesh_batch.fill(mesh_ids)
        self.basis[:, :self.n].copy_(self.mesh_batch.evecs[:, :self.n])
        return self

    def pack(self, t, rotations=None):
        """``BatchSlot.pack`` of the slot's 2 P meshes (x shapes first, then y shapes); ``rotations`` (2 P, 3, 3)."""
        return self.mesh_batch.pack(t, rotations=rotations)

    def ground_truth(self):
        """The (P, n, n) ground-truth maps of the drawn pairs, written into the slot's fixed buffer (two launches)."""
        with ops._on(self.C_gt):
            return _ground_truth_into(self.pds, self.ids, self.C_gt, self.status, self._ws)

    def check(self):
        """Raise if a fill since the last check had an invalid pair index (IndexError) or exceeded the capacity
        (ValueError), or a ground truth was singular (RuntimeError), and clear the status.  One device-to-host read."""
        st = torch.cat([self.status, self.mesh_batch.status]).tolist()
        gt, ms = st[:3], st[3:]
        if gt[0]:
            self.status.zero_()
        if ms[0]:
            self.mesh_batch.status.zero_()
        if gt[0] == _GT_BAD_PAIR or ms[0] == 1:
            if gt[0] == _GT_BAD_PAIR:
                _raise_gt_status(gt, self.pds.n_table)
            raise IndexError("PairSlot.fill: the pair index at position {} is outside the dataset's {} pairs".format(
                ms[1] % self.n_pairs, self.pds.n_table))
        if ms[0]:
            raise ValueError("PairSlot.fill: the drawn pairs exceed the slot's capacity of {} rows and {} gradient "
                             "entries".format(self.mesh_batch.V, self.mesh_batch.entry_capacity))
        _raise_gt_status(gt, self.pds.n_table)
