"""The k lowest eigenpairs of a mesh's ``(L + eps I) phi = lambda M phi`` on the GPU: the problem the reference hands to
``scipy.sparse.linalg.eigsh(L + eps I, k, M, sigma=eps)`` (geometry.py:340-352), solved by Chebyshev-filtered subspace
iteration (Zhou & Saad) on ``A = M^-1/2 (L + eps I) M^-1/2``, with ``phi = M^-1/2 y``.

Every O(V) step runs in the library's fp64 kernels (dn_eig.cu): the filter's sparse products, the tall-skinny Gram
matrices, the block rotations and the residual norms.  Only B x B dense work (Cholesky / eigh of the Rayleigh-Ritz
matrices, B = k + guard) uses ``torch.linalg`` on the device.

One outer iteration: filter the active block with a Chebyshev polynomial that damps ``[theta_B, bound]`` (theta_B the
largest Ritz value of the block, bound Gershgorin's), orthonormalise it against the locked pairs and itself (CholQR2,
SVQB when the Gram matrix is too ill-conditioned for Cholesky), Rayleigh-Ritz, lock the leading converged pairs.
Converged: ``||A y - theta y|| <= RES_TOL * theta_{k-1}`` (but never below ``RES_FLOOR * bound``, the rounding level of
one product with A).  The degree of each filter is what the slowest unconverged wanted pair needs to reach that bound,
clamped to [MIN_DEGREE, MAX_DEGREE].  With B == V one Rayleigh-Ritz step is exact."""
from __future__ import annotations

import math

import numpy as np
import torch

from . import _lib, ops

RES_TOL = 1e-9
RES_FLOOR = 1e-14
MIN_DEGREE, MAX_DEGREE = 10, 60
MAX_ITERATIONS = 500


def block_size(V, k):
    """B = min(V, k + guard), guard = max(16, k / 4); for V = None the unclamped k + guard (a mesh batch's width)."""
    B = k + max(16, k // 4)
    return B if V is None else min(V, B)


def chebyshev_coefficients(degree, lo, cut, hi):
    """Yields (alpha, beta, gamma) for each of the ``degree`` steps of the scaled Chebyshev filter that damps [cut, hi]
    (``lo`` estimates the bottom of the spectrum, for scaling only): step 0 is ``Y1 = alpha A Y0 + beta Y0``, step
    d > 0 ``Y_{d+1} = alpha A Y_d + beta Y_d + gamma Y_{d-1}``.  (lo, cut, hi) are floats, or float64 arrays with one
    entry per mesh; either way each entry goes through the same float64 operations, so a mesh's coefficients do not
    depend on which form computed them.  A generator, so that a caller can launch each step as soon as it has its
    coefficients."""
    e, c = (hi - cut) / 2.0, (hi + cut) / 2.0
    sigma = e / (lo - c)
    sigma1 = sigma
    yield sigma1 / e, -c * sigma1 / e, 0.0 * e             # gamma is unused without Y_prev; e > 0, so +0.0
    for _ in range(1, degree):
        sigma2 = 1.0 / (2.0 / sigma1 - sigma)
        a = 2.0 * sigma2 / e
        yield a, -c * a, -sigma * sigma2
        sigma = sigma2


def filter_degree(theta, res, tol, cut, hi):
    """The degree of the next filter: what the slowest of the wanted pairs (Ritz values ``theta``, residual norms
    ``res``) with ``res > tol`` needs to reach ``tol`` when [cut, hi] is damped, clamped to [MIN_DEGREE, MAX_DEGREE]."""
    e, c = (hi - cut) / 2.0, (hi + cut) / 2.0
    need = MIN_DEGREE
    for th, r in zip(theta, res):
        if r > tol:
            t = abs((th - c) / e)
            if t > 1.0 + 1e-12:
                need = max(need, math.ceil(math.acosh(r / tol) / math.acosh(t)))
            else:
                need = MAX_DEGREE
    return min(need, MAX_DEGREE)


def _svqb(G):
    """SVQB (Stathopoulos & Wu) of Gram matrices G (..., n, n): C with C^T G C = I on G's numerical range."""
    d = G.diagonal(dim1=-2, dim2=-1).clamp_min(1e-300).rsqrt()
    S, U = torch.linalg.eigh(d[..., :, None] * G * d[..., None, :])
    S = torch.maximum(S, S.amax(dim=-1, keepdim=True) * 1e-15)
    return d[..., :, None] * U * S.rsqrt()[..., None, :]


class LaplaceOperator:
    """The device arrays of ``A = A_vals + diag(A_diag)`` (dn_mesh_laplacian) plus the mass and the spectral bound."""

    def __init__(self, V, rowptr, colidx, avals, adiag, mass, bound):
        self.V, self.rowptr, self.colidx, self.avals, self.adiag, self.mass = V, rowptr, colidx, avals, adiag, mass
        self.bound = float(bound)


class _Solver:
    def __init__(self, op, k, B, seed):
        self.op, self.k, self.B, self.V = op, k, B, op.V
        self.lib = _lib.load()
        dev = op.mass.device
        self.dev = dev
        f64 = torch.float64
        gen = torch.Generator(device=dev)
        gen.manual_seed(seed)
        self.Q = torch.randn(self.V, B, generator=gen, device=dev, dtype=f64)
        self.T = [torch.empty(self.V, B, device=dev, dtype=f64) for _ in range(2)]
        self.W = torch.empty(self.V, B, device=dev, dtype=f64)
        self.W2 = torch.empty(self.V, B, device=dev, dtype=f64)
        self.ws = torch.empty(max(512 * B * B, 4096), dtype=torch.uint8, device=dev)
        self.steps = 0
        self.col_steps = 0               # sum over filter steps of the columns filtered (bench_operators' byte model)

    # ---- kernels on column slices [c0, B) of the V x B buffers ----------------------------------------------------
    def _p(self, buf, c0=0):
        return buf.data_ptr() + 8 * c0

    def filt(self, src, prev, dst, c0, alpha, beta, gamma):
        op = self.op
        _lib.call("dn_eig_filter", op.rowptr, op.colidx, op.avals, op.adiag, self.V, self.B - c0, self._p(src, c0),
                  self._p(prev, c0) if prev is not None else None, self.B, alpha, beta, gamma, self._p(dst, c0),
                  ops._stream())

    def gram(self, X, xc0, xn, Y, yc0, yn):
        out = torch.empty(xn, yn, dtype=torch.float64, device=self.dev)
        _lib.call("dn_eig_gram", self._p(X, xc0), self.B, self._p(Y, yc0), self.B, self.V, xn, yn, out, self.ws,
                  self.ws.numel(), ops._stream())
        return out

    def rotate(self, X, xc0, kd, Cm, Z, zc0, n, beta=0.0):
        _lib.call("dn_eig_rotate", self._p(X, xc0), self.B, Cm.contiguous(), n, self.V, kd, n, beta, self._p(Z, zc0),
                  self.B, ops._stream())

    def residuals(self, Wb, Qb, c0, theta):
        n = self.B - c0
        out = torch.empty(n, dtype=torch.float64, device=self.dev)
        _lib.call("dn_eig_residual_norms", self._p(Wb, c0), self.B, self._p(Qb, c0), self.B, theta.contiguous(), self.V,
                  n, out, self.ws, self.ws.numel(), ops._stream())
        return out

    # ---- the steps of one outer iteration ------------------------------------------------------------------------
    def chebyshev(self, c0, degree, lo, cut, hi):
        """Scaled Chebyshev filter of degree ``degree`` on columns [c0, B) of Q, damping [cut, hi]; ``lo`` estimates
        the bottom of the spectrum (scaling only).  Returns the buffer holding the result."""
        coef = chebyshev_coefficients(degree, lo, cut, hi)
        bufs = [self.Q, self.T[0], self.T[1]]
        prev, cur = 0, 1
        self.filt(bufs[prev], None, bufs[cur], c0, *next(coef))
        for step in coef:
            nxt = 3 - prev - cur
            self.filt(bufs[cur], bufs[prev], bufs[nxt], c0, *step)
            prev, cur = cur, nxt
        self.steps += degree
        self.col_steps += degree * (self.B - c0)
        return bufs[cur]

    def orthonormalize(self, Y, c0):
        """Columns [c0, B) of Y made orthonormal and orthogonal to the locked columns [0, c0) of Q; returns the buffer
        (never Q) that holds them."""
        n = self.B - c0
        for _ in range(2):
            if c0 > 0:                                   # Y_a -= Q_l (Q_l^T Y_a)
                G = self.gram(self.Q, 0, c0, Y, c0, n)
                self.rotate(self.Q, 0, c0, -G, Y, c0, n, beta=1.0)
            G = self.gram(Y, c0, n, Y, c0, n)
            G = 0.5 * (G + G.T)
            R, info = torch.linalg.cholesky_ex(G, upper=True)
            if int(info) == 0:
                Cm = torch.linalg.solve_triangular(R, torch.eye(n, dtype=G.dtype, device=G.device), upper=True)
            else:
                Cm = _svqb(G)
            Z = next(b for b in (self.T[0], self.T[1], self.W2) if b is not Y)
            self.rotate(Y, c0, n, Cm, Z, c0, n)
            Y = Z
        return Y

    def rayleigh_ritz(self, Z, c0):
        """Rayleigh-Ritz on the orthonormal columns [c0, B) of Z: Ritz vectors into Q, A times them into W2."""
        n = self.B - c0
        self.filt(Z, None, self.W, c0, 1.0, 0.0, 0.0)
        H = self.gram(Z, c0, n, self.W, c0, n)
        theta, U = torch.linalg.eigh(0.5 * (H + H.T))
        self.rotate(Z, c0, n, U, self.Q, c0, n)
        self.rotate(self.W, c0, n, U, self.W2, c0, n)
        return theta, self.residuals(self.W2, self.Q, c0, theta)


def _event():
    e = torch.cuda.Event(enable_timing=True)
    e.record()
    return e


def lowest_eigenpairs(op, k, seed=0, stats=None):
    """(evals (k) fp64 ascending and clipped at 0, evecs (V, k) fp64 M-orthonormal) of ``(L + eps I, M)``.
    Eigenvector signs: the largest-magnitude entry of every column is positive (lowest vertex index on ties).
    Deterministic: a seeded start block and fixed-order reductions, so two calls give bitwise-equal results.
    ``stats`` (dict, optional) receives iterations, total filter degree, block size and stage times (ms).
    Raises ValueError("failed to compute eigendecomp ...") if the iteration cap is reached, and for k >= V, where the
    reference's ``eigsh(..., sigma=eps)`` refuses (k must be below the matrix order) and it ends in that error."""
    V = op.V
    dev = op.mass.device
    if k <= 0:
        return (torch.zeros(0, dtype=torch.float64, device=dev), torch.zeros(V, 0, dtype=torch.float64, device=dev))
    if k >= V:
        raise ValueError("failed to compute eigendecomp: k_eig = {} is not below the vertex count {}".format(k, V))
    B = block_size(V, k)
    s = _Solver(op, k, B, seed)
    t0 = _event()
    Z = s.orthonormalize(s.Q, 0)
    theta, res = s.rayleigh_ritz(Z, 0)
    rr_ms, filter_ms = [(t0, _event())], []
    theta_all = theta
    converged = torch.zeros(B, dtype=torch.bool, device=dev)
    nl, it = 0, 0
    while True:
        if B == V:
            converged[:] = True
        k_th = float(theta_all.sort().values[k - 1])
        tol = max(RES_TOL * abs(k_th), RES_FLOOR * op.bound)
        converged[nl:] = res <= tol
        order = torch.sort(theta_all, stable=True).indices
        if bool(converged[order[:k]].all()):
            break
        if it >= MAX_ITERATIONS:
            raise ValueError("failed to compute eigendecomp: {} filter iterations ({} steps) did not reach residual {:.1e}"
                             .format(it, s.steps, tol))
        # lock the leading converged active pairs (Q's active columns are sorted by Ritz value)
        lead = 0
        conv_a = converged[nl:].tolist()
        while lead < len(conv_a) and conv_a[lead] and nl + lead < k:
            lead += 1
        th_a = theta_all[nl:]
        res_a = res[lead:]
        nl += lead
        th_host = th_a.tolist()
        cut, lo = th_host[-1], th_host[0]
        if cut >= op.bound:
            raise ValueError("failed to compute eigendecomp: the block's Ritz values reach the spectral bound")
        degree = filter_degree(th_host[lead:lead + k - nl], res_a[:k - nl].tolist(), tol, cut, op.bound)
        f0 = _event()
        Y = s.chebyshev(nl, degree, lo, cut, op.bound)
        f1 = _event()
        Z = s.orthonormalize(Y, nl)
        theta, res = s.rayleigh_ritz(Z, nl)
        rr_ms.append((f1, _event()))
        filter_ms.append((f0, f1))
        theta_all = torch.cat((theta_all[:nl], theta))
        converged = torch.cat((converged[:nl], torch.zeros(B - nl, dtype=torch.bool, device=dev)))
        it += 1
    idx = torch.sort(theta_all, stable=True).indices[:k]
    cols = idx.to(torch.int32).contiguous()
    evecs = torch.empty(V, k, dtype=torch.float64, device=dev)
    _lib.check(s.lib.dn_eig_finalize(*_lib.addresses((s.Q, B, cols, k, op.mass, V, evecs, s.ws, s.ws.numel(),
                                                      ops._stream()))), "dn_eig_finalize")
    evals = theta_all[idx].clamp_min(0.0)
    if stats is not None:
        torch.cuda.synchronize(dev)
        stats.update(iterations=it, filter_steps=s.steps, filter_col_steps=s.col_steps, block=B, bound=op.bound,
                     res_tol=tol, nnz=int(op.colidx.numel()),
                     filter_ms=sum(a.elapsed_time(b) for a, b in filter_ms),
                     rr_ms=sum(a.elapsed_time(b) for a, b in rr_ms))
    return evals, evecs


# ----------------------------------------------------------------------------------------------------------------------
# the same iteration for a batch of small meshes, as one launch sequence
# ----------------------------------------------------------------------------------------------------------------------
TILE_ROWS, SLICE_ROWS = _lib.EIG_TILE_ROWS, _lib.EIG_SLICE_ROWS


class BatchPlan:
    """``dn_eig_batch`` for meshes of ``Vs`` vertices laid out one after the other: the struct and its device arrays."""

    def __init__(self, Vs, device):
        Vs = np.asarray(Vs, dtype=np.int64)
        n = len(Vs)
        begin = lambda c: np.concatenate(([0], np.cumsum(c)))
        tiles, slices = -(-Vs // TILE_ROWS), -(-Vs // SLICE_ROWS)
        self.row_begin = begin(Vs)
        if self.row_begin[-1] >= 2 ** 31 - 1:
            raise ValueError("a batch of {} rows exceeds the int32 row index".format(int(self.row_begin[-1])))
        parts = [self.row_begin, np.repeat(np.arange(n), tiles), begin(tiles), np.repeat(np.arange(n), slices), begin(slices)]
        offs = begin([len(p) for p in parts])
        self.arrays = torch.from_numpy(np.concatenate(parts).astype(np.int32)).to(device)   # kept alive next to the struct
        ptr = [self.arrays.data_ptr() + 4 * int(o) for o in offs[:5]]
        self.n, self.V, self.n_slices = n, int(self.row_begin[-1]), int(slices.sum())
        self.struct = _lib.dn_eig_batch(n, int(tiles.sum()), self.n_slices, *ptr)


class _BatchSolver:
    """_Solver's kernels on the concatenated V x B blocks of the meshes of a batch (full blocks: nothing is locked)."""

    def __init__(self, ops_, k, B, seed):
        import ctypes
        self.k, self.B, self.n = k, B, len(ops_)
        dev = self.dev = ops_[0].mass.device
        f64 = torch.float64
        self.plan = BatchPlan([op.V for op in ops_], dev)
        self.bt = ctypes.byref(self.plan.struct)
        V, rb = self.plan.V, self.plan.row_begin
        # one block-diagonal CSR with batch-global columns
        nz = [0]
        for op in ops_:
            nz.append(nz[-1] + int(op.colidx.numel()))
        self.rowptr = torch.cat([op.rowptr[:-1] + nz[b] for b, op in enumerate(ops_)] +
                                [torch.tensor([nz[-1]], dtype=torch.int32, device=dev)]).to(torch.int32)
        self.colidx = torch.cat([op.colidx + int(rb[b]) for b, op in enumerate(ops_)]).to(torch.int32)
        self.avals = torch.cat([op.avals for op in ops_])
        self.adiag = torch.cat([op.adiag for op in ops_])
        self.mass = torch.cat([op.mass for op in ops_])
        # every mesh starts from the block lowest_eigenpairs would start from: its start does not depend on the batch
        self.Q = torch.empty(V, B, device=dev, dtype=f64)
        gen = torch.Generator(device=dev)
        for b, op in enumerate(ops_):
            gen.manual_seed(seed)
            self.Q[int(rb[b]):int(rb[b + 1])] = torch.randn(op.V, B, generator=gen, device=dev, dtype=f64)
        self.T = [torch.empty(V, B, device=dev, dtype=f64) for _ in range(2)]
        self.W = torch.empty(V, B, device=dev, dtype=f64)
        self.W2 = torch.empty(V, B, device=dev, dtype=f64)
        self.ws = torch.empty(max(8 * self.plan.n_slices * B * B, 8 * self.n * B, 4096), dtype=torch.uint8, device=dev)
        self.active = torch.ones(self.n, dtype=torch.int32, device=dev)
        self.act = torch.arange(self.n, device=dev)                  # indices of the active meshes
        self.G = torch.zeros(self.n, B, B, dtype=f64, device=dev)    # Gram / rotation stacks, all meshes
        self.Cm = torch.zeros(self.n, B, B, dtype=f64, device=dev)
        self.eye = torch.eye(B, dtype=f64, device=dev)
        self.unit = torch.tensor([[1.0] * self.n, [0.0] * self.n, [0.0] * self.n], dtype=f64, device=dev)
        self.steps = 0
        self.dense_ev = []

    def set_active(self, flags):
        self.active = torch.tensor([int(f) for f in flags], dtype=torch.int32, device=self.dev)
        self.act = torch.tensor([b for b, f in enumerate(flags) if f], dtype=torch.int64, device=self.dev)

    def filt(self, src, prev, dst, coef):
        """coef: (3, n) device rows alpha, beta, gamma"""
        _lib.call("dn_eig_filter_batched", self.rowptr, self.colidx, self.avals, self.adiag, self.bt, self.B, src, prev,
                  self.B, coef[0], coef[1], coef[2], self.active, dst, ops._stream())

    def gram(self, X, Y):
        _lib.call("dn_eig_gram_batched", X, self.B, Y, self.B, self.bt, self.B, self.B, self.active, self.G, self.ws,
                  self.ws.numel(), ops._stream())
        G = self.G[self.act]
        return 0.5 * (G + G.transpose(1, 2))

    def rotate(self, X, Cm, Z):
        _lib.call("dn_eig_rotate_batched", X, self.B, Cm, self.bt, self.B, self.B, 0.0, self.active, Z, self.B,
                  ops._stream())

    def _dense(self, fn):
        a = _event()
        r = fn()
        self.dense_ev.append((a, _event()))
        return r

    def chebyshev(self, degree, lo, cut, hi):
        """_Solver.chebyshev with every mesh's own (lo, cut, hi): the coefficients of all steps go up in one copy."""
        coef = torch.from_numpy(np.array(list(chebyshev_coefficients(degree, lo, cut, hi)))).to(self.dev)
        bufs = [self.Q, self.T[0], self.T[1]]
        prev, cur = 0, 1
        self.filt(bufs[prev], None, bufs[cur], coef[0])
        for d in range(1, degree):
            nxt = 3 - prev - cur
            self.filt(bufs[cur], bufs[prev], bufs[nxt], coef[d])
            prev, cur = cur, nxt
        self.steps += degree
        return bufs[cur]

    def orthonormalize(self, Y):
        """CholQR2 per mesh on (n_active, B, B) stacks; SVQB for exactly the meshes whose Cholesky fails (one host read
        of the info vector per pass)."""
        for _ in range(2):
            G = self.gram(Y, Y)

            def dense():
                R, info = torch.linalg.cholesky_ex(G, upper=True)
                bad = torch.nonzero(info).flatten()                  # host read
                R[bad] = self.eye
                Cm = torch.linalg.solve_triangular(R, self.eye.expand_as(R), upper=True)
                if bad.numel():
                    Cm[bad] = _svqb(G[bad])
                self.Cm[self.act] = Cm
            self._dense(dense)
            Z = next(b for b in (self.T[0], self.T[1], self.W2) if b is not Y)
            self.rotate(Y, self.Cm, Z)
            Y = Z
        return Y

    def rayleigh_ritz(self, Z, theta_all, res_all):
        """Ritz vectors of the active meshes into Q, A times them into W2; their rows of theta_all / res_all updated."""
        self.filt(Z, None, self.W, self.unit)
        H = self.gram(Z, self.W)

        def dense():
            theta, U = torch.linalg.eigh(H)
            self.Cm[self.act] = U
            theta_all[self.act] = theta
        self._dense(dense)
        self.rotate(Z, self.Cm, self.Q)
        self.rotate(self.W, self.Cm, self.W2)
        _lib.call("dn_eig_residual_norms_batched", self.W2, self.B, self.Q, self.B, theta_all, self.bt, self.B,
                  self.active, res_all, self.ws, self.ws.numel(), ops._stream())


def lowest_eigenpairs_batch(ops_, k, seed=0, stats=None, first=0):
    """``lowest_eigenpairs`` for a list of ``LaplaceOperator`` (the meshes of one dataset, a few hundred to some ten
    thousand vertices each): a list of its ``(evals, evecs)`` pairs, in order.

    The meshes whose block has the full width ``B = k + guard`` are iterated together on their concatenated rows: each
    filter step, Gram matrix, rotation and residual is one launch over all of them (dn_eig_*_batched), the B x B dense
    steps are batched ``torch.linalg`` calls on an (n_active, B, B) stack, and the host reads the Ritz values and
    residuals of all meshes in one copy per outer iteration (plus the Cholesky info vector of each of the two
    orthonormalisation passes).  Same constants and the same per-mesh convergence test as ``lowest_eigenpairs``; what
    differs: nothing is locked (every active mesh iterates its full block -- at these sizes the filter is the cheap
    part, and ragged widths would need a launch per width), and one filter degree per outer iteration serves the whole
    batch, the largest any active mesh asks for (each mesh keeps its own damped interval [cut_b, bound_b]; the scaled
    recurrence makes a higher degree than needed harmless).  A converged mesh turns inactive: its Ritz vectors stay
    where they are and no later launch touches its rows.  A mesh's start block, tile and slice cuts are its own, so
    every kernel gives it the bits it would get alone; only the shared degree ties it to its batch, which moves its
    eigenpairs within the solver's tolerance.  Two calls on the same list give bitwise-equal results.

    A mesh with ``V < k + guard`` (a narrower block) is solved by ``lowest_eigenpairs``; ``k >= V`` raises its
    ValueError, prefixed with ``mesh {i}: `` like every other per-mesh failure (i counts from ``first``, the index of
    ``ops_[0]`` in the caller's list).
    ``stats`` (dict, optional) receives iterations, filter_steps, block, n_stacked and filter / Rayleigh-Ritz / dense
    ``torch.linalg`` times in ms (the dense time is part of the Rayleigh-Ritz time)."""
    n, k = len(ops_), int(k)
    for i, op in enumerate(ops_):
        if 0 < k and k >= op.V:
            raise ValueError("mesh {}: failed to compute eigendecomp: k_eig = {} is not below the vertex count {}"
                             .format(first + i, k, op.V))
    out = [None] * n
    if k <= 0:
        return [lowest_eigenpairs(op, k, seed=seed) for op in ops_]
    B = block_size(None, k)
    stack = [i for i, op in enumerate(ops_) if op.V >= B]
    for i, op in enumerate(ops_):
        if op.V < B:
            try:
                out[i] = lowest_eigenpairs(op, k, seed=seed)
            except ValueError as e:
                raise ValueError("mesh {}: {}".format(first + i, e)) from None
    it, s = 0, None
    if stack:
        sops = [ops_[i] for i in stack]
        m = len(sops)
        s = _BatchSolver(sops, k, B, seed)
        dev = s.dev
        bound = np.array([op.bound for op in sops])
        theta_all = torch.zeros(m, B, dtype=torch.float64, device=dev)
        res_all = torch.zeros(m, B, dtype=torch.float64, device=dev)
        t0 = _event()
        s.rayleigh_ritz(s.orthonormalize(s.Q), theta_all, res_all)
        rr_ev, filter_ev = [(t0, _event())], []
        active = np.ones(m, dtype=bool)
        while True:
            host = torch.stack((theta_all, res_all)).cpu().numpy()      # the outer iteration's one read of both
            th, res = host[0], host[1]
            tol = np.maximum(RES_TOL * np.abs(th[:, k - 1]), RES_FLOOR * bound)
            active &= ~(res[:, :k] <= tol[:, None]).all(axis=1)
            if not active.any():
                break
            who = [stack[b] for b in np.nonzero(active)[0]]
            if it >= MAX_ITERATIONS:
                raise ValueError("mesh {}: failed to compute eigendecomp: {} filter iterations ({} steps) did not reach "
                                 "residual {:.1e}".format(first + who[0], it, s.steps, tol[active][0]))
            cut, lo = th[:, -1].copy(), th[:, 0].copy()
            if (cut[active] >= bound[active]).any():
                b = int(np.nonzero(active & (cut >= bound))[0][0])
                raise ValueError("mesh {}: failed to compute eigendecomp: the block's Ritz values reach the spectral bound"
                                 .format(first + stack[b]))
            cut[~active], lo[~active] = 0.5 * bound[~active], 0.0       # placeholders: inactive rows are not touched
            degree = max(filter_degree(th[b, :k], res[b, :k], tol[b], cut[b], bound[b]) for b in np.nonzero(active)[0])
            s.set_active(active)
            f0 = _event()
            Y = s.chebyshev(degree, lo, cut, bound)
            f1 = _event()
            s.rayleigh_ritz(s.orthonormalize(Y), theta_all, res_all)
            rr_ev.append((f1, _event()))
            filter_ev.append((f0, f1))
            it += 1
        # eigh returns every mesh's Ritz values ascending and nothing was locked: the k lowest are the first k columns
        cols = torch.arange(k, dtype=torch.int32, device=dev).repeat(m, 1).contiguous()
        evecs = torch.empty(s.plan.V, k, dtype=torch.float64, device=dev)
        _lib.call("dn_eig_finalize_batched", s.Q, B, cols, k, s.mass, s.bt, evecs, s.ws, s.ws.numel(), ops._stream())
        evals = theta_all[:, :k].clamp_min(0.0)
        rb = s.plan.row_begin
        for b, i in enumerate(stack):
            out[i] = (evals[b], evecs[int(rb[b]):int(rb[b + 1])])
    if stats is not None:
        stats.update(iterations=it, filter_steps=s.steps if s else 0, block=B, n_stacked=len(stack))
        if s:
            torch.cuda.synchronize(s.dev)
            ms = lambda evs: sum(a.elapsed_time(b) for a, b in evs)
            stats.update(filter_ms=ms(filter_ev), rr_ms=ms(rr_ev), dense_ms=ms(s.dense_ev))
    return out
