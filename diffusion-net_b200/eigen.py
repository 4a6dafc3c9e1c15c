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

import torch

from . import _lib, ops

RES_TOL = 1e-9
RES_FLOOR = 1e-14
MIN_DEGREE, MAX_DEGREE = 10, 60
MAX_ITERATIONS = 500


def block_size(V, k):
    """B = min(V, k + guard), guard = max(16, k / 4)."""
    return min(V, k + max(16, k // 4))


class LaplaceOperator:
    """The device arrays of ``A = A_vals + diag(A_diag)`` (dn_mesh_laplacian) plus the mass and the spectral bound."""

    def __init__(self, V, rowptr, colidx, avals, adiag, mass, bound):
        self.V, self.rowptr, self.colidx, self.avals, self.adiag, self.mass = V, rowptr, colidx, avals, adiag, mass
        self.bound = float(bound)


def _check(code, what):
    _lib.check(code, what)


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
        _check(self.lib.dn_eig_filter(op.rowptr.data_ptr(), op.colidx.data_ptr(), op.avals.data_ptr(),
                                      op.adiag.data_ptr(), self.V, self.B - c0, self._p(src, c0),
                                      self._p(prev, c0) if prev is not None else None, self.B, alpha, beta, gamma,
                                      self._p(dst, c0), ops._stream()), "dn_eig_filter")

    def gram(self, X, xc0, xn, Y, yc0, yn):
        out = torch.empty(xn, yn, dtype=torch.float64, device=self.dev)
        _check(self.lib.dn_eig_gram(self._p(X, xc0), self.B, self._p(Y, yc0), self.B, self.V, xn, yn, out.data_ptr(),
                                    self.ws.data_ptr(), self.ws.numel(), ops._stream()), "dn_eig_gram")
        return out

    def rotate(self, X, xc0, kd, Cm, Z, zc0, n, beta=0.0):
        Cm = Cm.contiguous()
        _check(self.lib.dn_eig_rotate(self._p(X, xc0), self.B, Cm.data_ptr(), n, self.V, kd, n, beta, self._p(Z, zc0),
                                      self.B, ops._stream()), "dn_eig_rotate")

    def residuals(self, Wb, Qb, c0, theta):
        n = self.B - c0
        out = torch.empty(n, dtype=torch.float64, device=self.dev)
        theta = theta.contiguous()
        _check(self.lib.dn_eig_residual_norms(self._p(Wb, c0), self.B, self._p(Qb, c0), self.B, theta.data_ptr(),
                                              self.V, n, out.data_ptr(), self.ws.data_ptr(), self.ws.numel(),
                                              ops._stream()), "dn_eig_residual_norms")
        return out

    # ---- the steps of one outer iteration ------------------------------------------------------------------------
    def chebyshev(self, c0, degree, lo, cut, hi):
        """Scaled Chebyshev filter of degree ``degree`` on columns [c0, B) of Q, damping [cut, hi]; ``lo`` estimates
        the bottom of the spectrum (scaling only).  Returns the buffer holding the result."""
        e, c = (hi - cut) / 2.0, (hi + cut) / 2.0
        sigma = e / (lo - c)
        sigma1 = sigma
        bufs = [self.Q, self.T[0], self.T[1]]
        prev, cur = 0, 1
        self.filt(bufs[prev], None, bufs[cur], c0, sigma1 / e, -c * sigma1 / e, 0.0)
        for _ in range(2, degree + 1):
            nxt = 3 - prev - cur
            sigma2 = 1.0 / (2.0 / sigma1 - sigma)
            a = 2.0 * sigma2 / e
            self.filt(bufs[cur], bufs[prev], bufs[nxt], c0, a, -c * a, -sigma * sigma2)
            prev, cur, sigma = cur, nxt, sigma2
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
            else:                                        # SVQB (Stathopoulos & Wu)
                d = G.diagonal().clamp_min(1e-300).rsqrt()
                S, U = torch.linalg.eigh(d[:, None] * G * d[None, :])
                S = S.clamp_min(S.max() * 1e-15)
                Cm = d[:, None] * U * S.rsqrt()[None, :]
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
        e, c = (op.bound - cut) / 2.0, (op.bound + cut) / 2.0
        need = MIN_DEGREE
        r_host = res_a.tolist()
        for i, th in enumerate(th_host[lead:]):
            if nl + i >= k:
                break
            r = r_host[i]
            if r > tol:
                t = abs((th - c) / e)
                if t > 1.0 + 1e-12:
                    need = max(need, math.ceil(math.acosh(r / tol) / math.acosh(t)))
                else:
                    need = MAX_DEGREE
        degree = min(max(need, MIN_DEGREE), MAX_DEGREE)
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
    _check(s.lib.dn_eig_finalize(s.Q.data_ptr(), B, cols.data_ptr(), k, op.mass.data_ptr(), V, evecs.data_ptr(),
                                 s.ws.data_ptr(), s.ws.numel(), ops._stream()), "dn_eig_finalize")
    evals = theta_all[idx].clamp_min(0.0)
    if stats is not None:
        torch.cuda.synchronize(dev)
        stats.update(iterations=it, filter_steps=s.steps, filter_col_steps=s.col_steps, block=B, bound=op.bound,
                     res_tol=tol, nnz=int(op.colidx.numel()),
                     filter_ms=sum(a.elapsed_time(b) for a, b in filter_ms),
                     rr_ms=sum(a.elapsed_time(b) for a, b in rr_ms))
    return evals, evecs
