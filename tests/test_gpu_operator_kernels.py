"""The mesh-operator kernels one by one, against plain fp64 numpy / scipy, at the shapes where their launches change and
on the degenerate meshes real scans contain; the eigensolver's driver where it branches.

Bounds: with gamma_m = m eps / (1 - m eps), eps = 2^-53, a dot product or sum of m terms computed in fp64 is within
gamma_m * sum|terms| of the exact value, per entry.  The kernel and the numpy gold each carry such an error, so the
tests allow 2 gamma_m sum|terms|.  Every bound is shown to be tight: the same test perturbs the gold by dropping one
term of the sum (one row, one column or one split) and requires that perturbation to exceed the bound at least 100x
somewhere (``_assert_rejects``).

Sections: 1. each dn_eig_* kernel (filter, gram, rotate, residual norms, finalize); 2. dn_mesh_laplacian,
dn_vertex_frames and dn_build_grad on degenerate meshes; 3. lowest_eigenpairs where the driver branches (B == V,
B > 160, disconnected meshes, SVQB, no convergence); 4. the same driver on the CPU with the five kernels replaced by
dense fp64 products, plus the host-side input checks."""
import ctypes
import functools
import os
import sys
import types

import numpy as np
import pytest
import scipy.linalg as sl
import scipy.sparse as sp
import scipy.sparse.linalg as sla
import torch

from conftest import ROOT
from test_gpu_operators import _kprime, _projector_err

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle as O  # noqa: E402
import dn_oracle_ops as OO  # noqa: E402
from ref_import import _cotan_laplacian, _vertex_areas  # noqa: E402

import diffusion_net_b200 as dn  # noqa: E402
from diffusion_net_b200 import eigen  # noqa: E402

gpu = pytest.mark.gpu
EPS = 2.0 ** -53
U32 = 2.0 ** -24
DN_OK, DN_ERR_WORKSPACE = 0, -3
SHIFT = 1e-8                                     # geometry.EPS: the mass shift and the eigenproblem shift


def gamma(m):
    m = np.asarray(m, dtype=np.float64)
    return m * EPS / (1.0 - m * EPS)


def _assert_rejects(gold, perturbed, bound, what):
    """Dropping one term of the sum moves the gold by more than 100x the bound on at least one entry."""
    ratio = float(np.max(np.abs(np.asarray(perturbed) - np.asarray(gold)) / np.asarray(bound)))
    assert ratio >= 100.0, "{}: dropping one term moves the gold by only {:.3g} x the bound".format(what, ratio)


def _assert_within(got, gold, bound, what):
    err = np.abs(np.asarray(got, dtype=np.float64) - gold)
    bound = np.broadcast_to(bound, err.shape)
    ratio = np.divide(err, bound, out=np.where(err > 0, np.inf, 0.0), where=bound > 0)
    assert np.all(err <= bound), "{}: worst err / bound = {:.3g}".format(what, float(ratio.max()))
    print("MEASURED {} max_abs_err={:.3e} max_err_over_bound={:.3e}".format(what, float(err.max(initial=0.0)),
                                                                             float(ratio.max(initial=0.0))))


def _splits(V):
    return int(min(max(V // 4096, 1), 64))


# ------------------------------------------------------------------------------------------------
# meshes (seeded; fp64 vertices)
# ------------------------------------------------------------------------------------------------
def _np_mesh(make):
    v, f = make
    return np.asarray(v, dtype=np.float64), np.asarray(f, dtype=np.int64)


def degenerate_mesh():
    """A jittered 8 x 9 patch plus: a face with a repeated index, a duplicate face, an edge shared by three faces, an
    obtuse fan, a sliver whose cotangents are ~1e8 (dyadic coordinates, so every cross product is exact), a component
    of three collinear vertices (zero normal: the wiggle remedy fires) and an unreferenced last vertex (no face: the
    random-normal remedy fires)."""
    v, f = _np_mesh(dn.synthetic.patch_mesh(8, 9, seed=3))
    verts, faces = [v], [f, [[10, 10, 11]], f[:1]]
    n = len(v)
    i, j = 3 * 9 + 4, 4 * 9 + 4                                    # an interior edge of the patch
    verts.append([(v[i] + v[j]) / 2 + [0.0, 0.0, 0.3]])
    faces.append([[i, j, n]])
    n += 1
    ang = np.radians([0.0, 110.0, 220.0, 330.0])                   # centre angles 110, 110, 110, 30 degrees
    rad = np.array([1.0, 0.7, 1.3, 0.9])
    ring = np.stack((2.0 + rad * np.cos(ang), rad * np.sin(ang), 0.1 * rad), 1)
    verts += [[[2.0, 0.0, 0.0]], ring]
    faces.append([[n, n + 1 + a, n + 1 + (a + 1) % 4] for a in range(4)])
    n += 5
    verts.append([[4.0, 0.0, 0.0], [5.0, 0.0, 0.0], [4.5, 2.0 ** -29, 0.0]])    # |cot| = 2.5e8 and 1.3e8
    faces.append([[n, n + 1, n + 2]])
    n += 3
    verts.append([[6.0, 0.0, 1.0], [7.0, 0.0, 1.0], [8.0, 0.0, 1.0]])
    faces.append([[n, n + 1, n + 2]])
    n += 3
    verts.append([[0.0, 0.0, 5.0]])
    return np.concatenate([np.asarray(x, np.float64) for x in verts]), np.concatenate([np.asarray(x) for x in faces])


def two_components_mesh():
    v, f = _np_mesh(dn.synthetic.torus_mesh(12, 16, seed=1))
    v2, f2 = _np_mesh(dn.synthetic.patch_mesh(7, 9, seed=2))
    verts = np.concatenate((v, v2 + [3.0, 0.0, 0.0], [[0.0, 0.0, 9.0]]))
    return verts, np.concatenate((f, f2 + len(v)))


def fan_mesh(valence=2000):
    """One vertex of valence ``valence`` (a closed cone), plus a 3 x 3 patch sharing nothing with it."""
    t = 2 * np.pi * np.arange(valence) / valence
    ring = np.stack((np.cos(t), np.sin(t), 0.05 * np.sin(7 * t)), 1)
    verts = np.concatenate(([[0.0, 0.0, 0.4]], ring))
    faces = np.stack((np.zeros(valence, np.int64), 1 + np.arange(valence), 1 + (np.arange(valence) + 1) % valence), 1)
    return verts, faces


def two_tori_mesh():
    """Two disjoint 12 x 16 tori and an unreferenced last vertex: two eps-eigenvalues and the isolated one 1 / mean."""
    v, f = _np_mesh(dn.synthetic.torus_mesh(12, 16, seed=1))
    verts = np.concatenate((v, v + [5.0, 0.0, 0.0], [[0.0, 9.0, 0.0]]))
    return verts, np.concatenate((f, f + len(v)))


GEOM_MESHES = {
    "degenerate": degenerate_mesh,
    "two_components": two_components_mesh,
    "fan2000": fan_mesh,
    "torus200k": lambda: _np_mesh(dn.synthetic.torus_mesh(400, 500, seed=0)),
}

SOLVER_MESHES = {
    "patch6x7": lambda: _np_mesh(dn.synthetic.patch_mesh(6, 7, seed=3)),
    "patch8x9": lambda: _np_mesh(dn.synthetic.patch_mesh(8, 9, seed=3)),
    "ico4": lambda: _np_mesh(dn.synthetic.icosphere_mesh(4, seed=2)),
    "two_tori": two_tori_mesh,
}
SOLVER_CASES = {                                   # name -> (mesh, k): where eigen.lowest_eigenpairs branches
    "patch6x7_k26": ("patch6x7", 26),              # B == V: one Rayleigh-Ritz step
    "patch6x7_k41": ("patch6x7", 41),
    "patch8x9_k56": ("patch8x9", 56),
    "patch8x9_k71": ("patch8x9", 71),
    "ico4_k180": ("ico4", 180),                    # B = 225: NC = 8
    "ico4_k210": ("ico4", 210),                    # B = 262: a second, 6-column filter slice
    "ico4_k256": ("ico4", 256),                    # B = 320
    "two_tori_k48": ("two_tori", 48),              # two eps-eigenvalues and the isolated vertex's 1 / mean
}


def oracle_operator(verts, faces):
    """(L, mass, A) of the reference's problem in fp64: the cotan Laplacian and lumped mass of ``ref_import``, and
    A = M^-1/2 (L + eps I) M^-1/2."""
    L = _cotan_laplacian(verts, faces, denom_eps=1e-10)
    m = _vertex_areas(verts, faces)
    m += SHIFT * m.mean()
    d = sp.diags(1.0 / np.sqrt(m))
    A = (d @ (L + SHIFT * sp.identity(len(m))) @ d).tocsr()
    return L, m, A


@functools.lru_cache(maxsize=None)
def dense_gold(mesh):
    """(verts, faces, L, mass, all eigenvalues, all M-orthonormal eigenvectors) of ``(L + eps I, M)``, dense fp64."""
    verts, faces = SOLVER_MESHES[mesh]()
    L, m, _ = oracle_operator(verts, faces)
    lam, phi = sl.eigh((L + SHIFT * sp.identity(len(m))).toarray(), np.diag(m))
    return verts, faces, L, m, lam, phi


# ------------------------------------------------------------------------------------------------
# GPU plumbing
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    dn._lib.load()
    return torch.device("cuda")


def _lib():
    return dn._lib.load()


def _p(t, c0=0):
    return t.data_ptr() + t.element_size() * c0


def _np(t):
    return t.detach().cpu().numpy()


def _bits(a):
    return np.asarray(a, dtype=np.float64).view(np.int64)


SENTINEL = np.array([0x7FF8DEADBEEF0001], dtype=np.int64).view(np.float64)[0]      # a NaN with a payload


def _sentinel_buf(V, ld, dev):
    return torch.full((V, ld), SENTINEL, dtype=torch.float64, device=dev)


def _assert_sentinel_kept(buf, c0, n, what):
    b = _bits(_np(buf))
    outside = np.ones(b.shape[1], bool)
    outside[c0:c0 + n] = False
    assert np.all(b[:, outside] == _bits(SENTINEL)), what + ": a column outside the slice was written"


# ------------------------------------------------------------------------------------------------
# 1. eigensolver kernels
# ------------------------------------------------------------------------------------------------
def _random_csr(V, rs):
    """Random CSR of a V x V operator: 0..8 entries per row, row V // 2 empty (only the diagonal shift)."""
    cnt = rs.randint(0, 9, V)
    cnt[V // 2] = 0
    rowptr = np.concatenate(([0], np.cumsum(cnt))).astype(np.int32)
    colidx = rs.randint(0, V, int(rowptr[-1])).astype(np.int32)
    return rowptr, colidx, rs.randn(int(rowptr[-1])), rs.randn(V)


# (V, n, c0, pad, with_prev): n covers every NC (1..8) and 1..3 column slices of 256; c0 > 0 with ld = c0 + n + pad
FILTER_CASES = ([(20000, n, 0, 0, n % 2 == 0) for n in (1, 32, 33, 161, 200, 256, 257, 320, 600)] +
                [(20000, 320, 64, 0, True), (20000, 200, 57, 3, False), (20000, 262, 58, 0, True),
                 (1, 33, 0, 0, False), (1, 1, 2, 1, True), (7, 257, 5, 2, True), (9, 600, 0, 0, False),
                 (9, 40, 3, 1, True)])


@gpu
@pytest.mark.parametrize("V,n,c0,pad,with_prev", FILTER_CASES)
def test_eig_filter(cuda, V, n, c0, pad, with_prev):
    rs = np.random.RandomState(V + 7 * n + c0)
    rowptr, colidx, avals, adiag = _random_csr(V, rs)
    ld = c0 + n + pad
    Y, Yp = rs.randn(V, ld), rs.randn(V, ld)
    alpha, beta, gamma_ = 1.3, -0.7, 0.4
    t = lambda a, dt=torch.float64: torch.from_numpy(np.ascontiguousarray(a)).to(cuda, dt)
    pad = lambda a: np.concatenate((a, np.zeros(1, a.dtype)))    # V = 1: no entries, but valid pointers
    d_rp, d_ci, d_av, d_ad, d_Y, d_Yp = (t(rowptr, torch.int32), t(pad(colidx), torch.int32), t(pad(avals)), t(adiag),
                                         t(Y), t(Yp))
    out = _sentinel_buf(V, ld, cuda)
    rc = _lib().dn_eig_filter(_p(d_rp), _p(d_ci), _p(d_av), _p(d_ad), V, n, _p(d_Y, c0),
                              _p(d_Yp, c0) if with_prev else None, ld, alpha, beta, gamma_, _p(out, c0),
                              dn.ops._stream())
    assert rc == DN_OK
    S = sp.csr_matrix((avals, colidx, rowptr), shape=(V, V))
    y, yp = Y[:, c0:c0 + n], Yp[:, c0:c0 + n]
    ay = S @ y + adiag[:, None] * y
    gold = alpha * ay + beta * y + (gamma_ * yp if with_prev else 0.0)
    terms = (abs(alpha) * (abs(S) @ abs(y) + abs(adiag)[:, None] * abs(y)) + abs(beta) * abs(y)
             + (abs(gamma_) * abs(yp) if with_prev else 0.0))
    m = np.diff(rowptr)[:, None] + 4                   # row entries + diagonal + the three-term combination
    bound = 2 * gamma(m) * terms
    got = _np(out)
    _assert_within(got[:, c0:c0 + n], gold, bound, "eig_filter V={} n={}".format(V, n))
    _assert_sentinel_kept(out, c0, n, "eig_filter")
    r = int(np.argmax(np.abs(adiag)))                  # drop one term: the diagonal of one row
    pert = gold.copy()
    pert[r] -= alpha * adiag[r] * y[r]
    _assert_rejects(gold, pert, bound, "eig_filter")


# (V, m, n, layout): splits clamp(V // 4096, 1, 64): 1, 1, 1, 1, 2, 3 (ragged), 64, 64 (ragged tail)
GRAM_CASES = [(0, 65, 320, "sep"), (1, 1, 1, "self"), (1, 320, 63, "off"), (4095, 63, 65, "off"),
              (4095, 64, 64, "self"), (8191, 64, 64, "sep"), (8192, 65, 320, "off"), (12289, 320, 320, "self"),
              (12289, 1, 63, "sep"), (262144, 64, 65, "off"), (262145, 65, 64, "sep"), (262145, 1, 320, "off")]


@gpu
@pytest.mark.parametrize("V,m,n,layout", GRAM_CASES)
def test_eig_gram(cuda, V, m, n, layout):
    """out = X^T Y over V rows; X and Y separate, one buffer (the self-Gram), or column ranges of one buffer."""
    rs = np.random.RandomState(V % 1000 + m + n)
    if layout == "self":
        ld, cx, cy = n + 5, 2, 2
    elif layout == "off":
        ld, cx, cy = m + n + 7, 3, m + 5
    else:
        ld, cx, cy = None, 0, 0
    if ld is None:
        X, Y = rs.randn(V, m), rs.randn(V, n)
        dX, dY = torch.from_numpy(X).to(cuda), torch.from_numpy(Y).to(cuda)
        ldx, ldy = m, n
    else:
        W = rs.randn(V, ld)
        X, Y = W[:, cx:cx + m], W[:, cy:cy + n]
        dX = dY = torch.from_numpy(W).to(cuda)
        ldx = ldy = ld
    out = torch.full((m, n), float("nan"), dtype=torch.float64, device=cuda)
    wsb = 8 * _splits(V) * m * n
    ws = torch.empty(max(wsb, 8), dtype=torch.uint8, device=cuda)
    call = lambda nbytes: _lib().dn_eig_gram(_p(dX, cx), ldx, _p(dY, cy), ldy, V, m, n, _p(out), _p(ws), nbytes,
                                             dn.ops._stream())
    if V > 0:
        assert call(wsb - 8) == DN_ERR_WORKSPACE
    assert call(wsb) == DN_OK
    got = _np(out)
    if V == 0:
        assert np.all(_bits(got) == 0)
        return
    gold = X.T @ Y
    bound = 2 * gamma(V) * (np.abs(X).T @ np.abs(Y))
    _assert_within(got, gold, bound, "eig_gram V={} m={} n={} {}".format(V, m, n, layout))
    r = V - 1                                          # drop one row (the ragged tail's last)
    _assert_rejects(gold, gold - np.outer(X[r], Y[r]), bound, "eig_gram row")
    P = _splits(V)
    if P > 1:                                          # drop the last split
        lo = (P - 1) * ((V + P - 1) // P)
        _assert_rejects(gold, gold - X[lo:].T @ Y[lo:], bound, "eig_gram split")


# (kd, n, V, beta)
ROTATE_CASES = [(1, 64, 20000, 0.0), (31, 65, 63, 1.0), (32, 1, 64, -0.5), (33, 320, 65, 0.0), (300, 65, 20000, -0.5),
                (300, 320, 20000, 1.0), (33, 64, 1, 1.0), (31, 320, 20000, 0.0), (32, 65, 20000, -0.5),
                (1, 1, 1, 0.0), (300, 1, 64, 1.0)]


def _check_rotate(X, C, Z0, beta, got, what):
    gold = X @ C + (beta * Z0 if beta != 0.0 else 0.0)
    terms = np.abs(X) @ np.abs(C) + (abs(beta) * np.abs(Z0) if beta != 0.0 else 0.0)
    bound = 2 * gamma(X.shape[1] + 1) * terms
    _assert_within(got, gold, bound, what)
    k = int(np.argmax(np.abs(C).sum(1)))               # drop one column of X
    _assert_rejects(gold, gold - np.outer(X[:, k], C[k]), bound, what)


@gpu
@pytest.mark.parametrize("kd,n,V,beta", ROTATE_CASES)
def test_eig_rotate(cuda, kd, n, V, beta):
    """Z = beta Z + X C; with beta = 0 Z is pre-filled with NaN and must not be read."""
    rs = np.random.RandomState(kd * 1000 + n + V)
    X, C = rs.randn(V, kd), rs.randn(kd, n)
    ldz, cz = n + 3, 1
    Z0 = rs.randn(V, n)
    dZ = _sentinel_buf(V, ldz, cuda)
    dZ[:, cz:cz + n] = float("nan") if beta == 0.0 else torch.from_numpy(Z0).to(cuda)
    dX, dC = torch.from_numpy(X).to(cuda), torch.from_numpy(C).to(cuda)
    assert _lib().dn_eig_rotate(_p(dX), kd, _p(dC), n, V, kd, n, beta, _p(dZ, cz), ldz, dn.ops._stream()) == DN_OK
    got = _np(dZ)[:, cz:cz + n]
    assert np.all(np.isfinite(got))
    _check_rotate(X, C, Z0, beta, got, "eig_rotate kd={} n={} V={} beta={}".format(kd, n, V, beta))
    _assert_sentinel_kept(dZ, cz, n, "eig_rotate")


@gpu
def test_eig_rotate_disjoint_columns_of_one_buffer(cuda):
    """The locked-column projection when the Chebyshev output lands in Q: X = columns [0, c0) and Z = columns
    [c0, B) of one V x B buffer, beta = 1."""
    rs = np.random.RandomState(5)
    V, B, c0 = 20000, 130, 33
    Q = rs.randn(V, B)
    C = rs.randn(c0, B - c0)
    dQ, dC = torch.from_numpy(Q).to(cuda), torch.from_numpy(C).to(cuda)
    assert _lib().dn_eig_rotate(_p(dQ), B, _p(dC), B - c0, V, c0, B - c0, 1.0, _p(dQ, c0), B,
                                dn.ops._stream()) == DN_OK
    got = _np(dQ)
    assert np.array_equal(_bits(got[:, :c0]), _bits(Q[:, :c0]))
    _check_rotate(Q[:, :c0], C, Q[:, c0:], 1.0, got[:, c0:], "eig_rotate disjoint columns")


@gpu
def test_eig_rotate_kd0_leaves_z(cuda):
    rs = np.random.RandomState(6)
    Z = torch.from_numpy(rs.randn(300, 70)).to(cuda)
    before = Z.clone()
    assert _lib().dn_eig_rotate(None, 0, None, 70, 300, 0, 70, 1.0, _p(Z), 70, dn.ops._stream()) == DN_OK
    assert np.array_equal(_bits(_np(Z)), _bits(_np(before)))


# (n, V): V at the split boundaries
RESID_CASES = [(1, 1), (31, 4095), (33, 8192), (320, 12289), (33, 262145), (31, 262144), (320, 8191)]


@gpu
@pytest.mark.parametrize("n,V", RESID_CASES)
def test_eig_residual_norms(cuda, n, V):
    """out[c] = || W[:, c] - theta[c] Q[:, c] ||, theta[0] = 0; W and Q column slices of ld-wide buffers."""
    rs = np.random.RandomState(n + V)
    ld, c0 = n + 4, 3
    Wb, Qb = rs.randn(V, ld), rs.randn(V, ld)
    theta = rs.uniform(0.1, 3.0, n)
    theta[0] = 0.0
    dW, dQ, dth = (torch.from_numpy(a).to(cuda) for a in (Wb, Qb, theta))
    out = torch.full((n,), float("nan"), dtype=torch.float64, device=cuda)
    wsb = 8 * _splits(V) * n
    ws = torch.empty(wsb, dtype=torch.uint8, device=cuda)
    assert _lib().dn_eig_residual_norms(_p(dW, c0), ld, _p(dQ, c0), ld, _p(dth), V, n, _p(out), _p(ws), wsb - 8,
                                        dn.ops._stream()) == DN_ERR_WORKSPACE
    assert _lib().dn_eig_residual_norms(_p(dW, c0), ld, _p(dQ, c0), ld, _p(dth), V, n, _p(out), _p(ws), wsb,
                                        dn.ops._stream()) == DN_OK
    W, Q = Wb[:, c0:c0 + n], Qb[:, c0:c0 + n]
    D = W - theta[None, :] * Q
    s = (D * D).sum(0)
    gold = np.sqrt(s)
    # d carries gamma_2 (|W| + |theta Q|) in each computation; the sum of V squares gamma_V; the root one rounding
    e = gamma(2) * (np.abs(W) + np.abs(theta[None, :] * Q))
    ds = gamma(V) * ((np.abs(D) + e) ** 2).sum(0) + (2 * np.abs(D) * e + e * e).sum(0)
    bound = 2 * (ds / gold + EPS * gold)
    _assert_within(_np(out), gold, bound, "eig_residual_norms n={} V={}".format(n, V))
    r = int(np.argmax(np.abs(D[:, 0])))                # drop one row
    _assert_rejects(gold, np.sqrt(s - D[r] ** 2), bound, "eig_residual_norms")


def finalize_np(Y, cols, mass):
    """dn_eig_finalize restated: phi = M^-1/2 Y[:, cols], each column's sign set by its largest |phi| (lowest row on
    ties, +1 for a zero column)."""
    x = Y[:, cols] / np.sqrt(mass)[:, None]
    idx = np.argmax(np.abs(x), axis=0)                 # first maximum: the lowest row
    sign = np.where(x[idx, np.arange(len(cols))] < 0.0, -1.0, 1.0)
    return sign[None, :] * x


@gpu
@pytest.mark.parametrize("V", [5, 1000, 70000])
def test_eig_finalize_bitwise(cuda, V):
    rs = np.random.RandomState(V)
    B, k = 40, 25
    Y = rs.uniform(-0.5, 0.5, (V, B))
    mass = rs.uniform(0.5, 2.0, V)                     # non-uniform
    cols = rs.permutation(B)[:k].astype(np.int32)
    # ties in |phi| between a lower and an upper row of opposite signs, in different threads (3 / 300) and in one
    # thread's stride (5 / 261, 7 / 263); on the smallest V the first and last rows
    ties = [(0, 3, 300, -1.0), (1, 5, 261, 1.0), (2, 7, 263, -1.0)]  # (column slot, lower row, upper row, lower's sign)
    ties = [(s, a, b, sg) if b < V else (s, 0, V - 1, sg) for s, a, b, sg in ties]
    for slot, a, b, sg in ties:
        mass[b] = mass[a]
        Y[a, cols[slot]] = sg * 3.0 * np.sqrt(mass[a])
        Y[b, cols[slot]] = -Y[a, cols[slot]]
    Y[:, cols[3]] = 0.0                                # a zero column: +1
    want = finalize_np(Y, cols, mass)
    for slot, a, b, sg in ties:                        # the lower row decided
        assert want[a, slot] > 0 and want[b, slot] < 0
    dY, dc, dm = (torch.from_numpy(np.ascontiguousarray(x)).to(cuda) for x in (Y, cols, mass))
    out = torch.full((V, k), float("nan"), dtype=torch.float64, device=cuda)
    ws = torch.empty(8 * k, dtype=torch.uint8, device=cuda)
    assert _lib().dn_eig_finalize(_p(dY), B, _p(dc), k, _p(dm), V, _p(out), _p(ws), 8 * k - 8,
                                  dn.ops._stream()) == DN_ERR_WORKSPACE
    assert _lib().dn_eig_finalize(_p(dY), B, _p(dc), k, _p(dm), V, _p(out), _p(ws), 8 * k, dn.ops._stream()) == DN_OK
    assert np.array_equal(_bits(_np(out)), _bits(want))


# ------------------------------------------------------------------------------------------------
# 2. geometry kernels on degenerate meshes
# ------------------------------------------------------------------------------------------------
def _cotan_terms(verts, faces):
    """The terms of the reference's coo Laplacian (``ref_import``: four per face corner) as (rows, cols, w, mag):
    mag = (|w| + 1/2) kappa with kappa = 1 + |u||v| / (|u x v| + denom_eps) bounds how far rounding inside one
    cotangent (dot, cross, norm, divide) moves it -- 1 / sin of the corner's angle, ~1e8 on a sliver."""
    rows, cols, ws, mags = [], [], [], []
    for c in range(3):
        i, j, k = faces[:, c], faces[:, (c + 1) % 3], faces[:, (c + 2) % 3]
        u, v = verts[j] - verts[i], verts[k] - verts[i]
        den = np.linalg.norm(np.cross(u, v), axis=1) + 1e-10
        w = 0.5 * np.einsum("ij,ij->i", u, v) / den
        kappa = 1.0 + np.linalg.norm(u, axis=1) * np.linalg.norm(v, axis=1) / den
        rows += [j, k, j, k]
        cols += [k, j, j, k]
        ws += [-w, -w, w, w]
        mags += [(np.abs(w) + 0.5) * kappa] * 4
    return np.concatenate(rows), np.concatenate(cols), np.concatenate(ws), np.concatenate(mags)


def _device_laplacian(verts, faces, dev):
    v64 = torch.from_numpy(verts).to(dev)
    f64 = torch.from_numpy(faces).to(dev)
    return dn.geometry.mesh_laplacian(v64, f64)


@gpu
@pytest.mark.parametrize("mesh", sorted(GEOM_MESHES))
def test_mesh_laplacian(cuda, mesh):
    verts, faces = GEOM_MESHES[mesh]()
    V, F = len(verts), len(faces)
    # the C-ABI refuses a workspace one byte short of 120 F + 12 V + 2048 before enqueueing anything
    dummy = torch.zeros(8, dtype=torch.float64, device=cuda)
    need = 120 * F + 12 * V + 2048
    assert _lib().dn_mesh_laplacian(_p(dummy), _p(dummy), F, V, SHIFT, *[_p(dummy)] * 8, _p(dummy), need - 1,
                                    dn.ops._stream()) == DN_ERR_WORKSPACE
    rowptr, colidx, lvals, mass, avals, adiag, bound = _device_laplacian(verts, faces, cuda)
    again = _device_laplacian(verts, faces, cuda)
    for a, b in zip((rowptr, colidx, lvals, mass, avals, adiag), again[:6]):
        assert torch.equal(a, b)
    assert bound == again[6]
    Lg = _cotan_laplacian(verts, faces, denom_eps=1e-10)       # scipy CSC, explicit zeros kept
    rp, ci = _np(rowptr), _np(colidx)
    assert np.array_equal(rp, Lg.indptr) and np.array_equal(ci, Lg.indices)   # symmetric: CSC arrays = CSR arrays
    Lm = sp.csr_matrix((_np(lvals), ci, rp), shape=(V, V))
    Lt = Lm.T.tocsr()
    assert np.array_equal(Lt.indptr, rp) and np.array_equal(Lt.indices, ci)
    assert np.array_equal(_bits(Lt.data), _bits(Lm.data))    # bitwise symmetric
    gold = Lg.tocsr()
    r, c, w, mag = _cotan_terms(verts, faces)
    csr = lambda vals: sp.coo_matrix((vals, (r, c)), shape=(V, V)).tocsr()
    m_cnt, sum_mag = csr(np.ones(len(r))).data, csr(mag).data   # same pattern as gold, CSR order
    bound_L = 2 * gamma(m_cnt + 16) * sum_mag
    _assert_within(Lm.data, gold.data, bound_L, "mesh_laplacian L " + mesh)
    t = int(np.argmax(np.where(r != c, np.abs(w) / mag, 0.0)))   # drop one off-diagonal term (one face corner)
    _assert_rejects(gold.data, csr(np.where(np.arange(len(w)) == t, 0.0, w)).data, bound_L, "mesh_laplacian L")
    # mass: barycentric areas (each face gives its vertices two sixths) + eps * mean; a face's area carries the
    # rounding of its cross product relative to |e1||e2|, not to its area (thin triangles of the valence-2000 fan)
    area = _vertex_areas(verts, faces)
    gm = area + SHIFT * area.mean()
    deg = np.bincount(faces.reshape(-1), minlength=V)
    e1, e2 = verts[faces[:, 1]] - verts[faces[:, 0]], verts[faces[:, 2]] - verts[faces[:, 0]]
    fa = 0.5 * np.linalg.norm(np.cross(e1, e2), axis=1)
    fmag = fa + 0.5 * np.linalg.norm(e1, axis=1) * np.linalg.norm(e2, axis=1)
    amag = np.zeros(V)
    for i in range(3):
        np.add.at(amag, faces[:, i], fmag / 3)
    bound_m = 2 * gamma(2 * deg + 16) * amag + 2 * gamma(V + 4) * SHIFT * area.mean()
    _assert_within(_np(mass), gm, bound_m, "mesh_laplacian mass " + mesh)
    f_big = int(np.argmax(fa))                                # drop one face's third from one vertex
    pert = gm.copy()
    pert[faces[f_big, 0]] -= fa[f_big] / 3
    _assert_rejects(gm, pert, bound_m, "mesh_laplacian mass")
    # A = M^-1/2 (L + eps I) M^-1/2 as A_vals (pattern of L) + A_diag (eps / m)
    d = 1.0 / np.sqrt(gm)
    rows = np.repeat(np.arange(V), np.diff(gold.indptr))
    ga = d[rows] * d[gold.indices] * gold.data
    mrel = bound_m / gm
    bound_a = d[rows] * d[gold.indices] * bound_L + (gamma(8) + mrel[rows] + mrel[gold.indices]) * np.abs(ga)
    _assert_within(_np(avals), ga, bound_a, "mesh_laplacian A_vals " + mesh)
    gdiag = SHIFT / gm
    _assert_within(_np(adiag), gdiag, (gamma(4) + 2 * mrel) * gdiag, "mesh_laplacian A_diag " + mesh)
    # Gershgorin bound: the max absolute row sum of A (shift included), and above the largest eigenvalue of A
    A = sp.csr_matrix((ga, gold.indices, gold.indptr), shape=(V, V)) + sp.diags(gdiag)
    absA = abs(A)
    rowsum = np.asarray(absA.sum(1)).ravel()
    r = int(np.argmax(rowsum))
    err_row = (sp.csr_matrix((bound_a, gold.indices, gold.indptr), shape=(V, V)) @ np.ones(V))[r]
    tol = err_row + (gamma(8) + 2 * mrel[r]) * gdiag[r] + gamma(int(absA[r].nnz) + 2) * rowsum[r]
    assert abs(bound - rowsum.max()) <= tol + 1e-300
    if V <= 5000:
        lmax = float(sla.eigsh(A, k=1, which="LA", return_eigenvectors=False)[0])
        assert bound >= lmax * (1 - 1e-10)


def _summed_face_normals(verts, faces):
    """Per vertex: the sum of its unit face normals, and sum over those faces of |fn| (1 + |e1||e2| / |e1 x e2|), the
    size of the terms times how much rounding inside one cross product can turn its direction."""
    c = verts[faces]
    e1, e2 = c[:, 1] - c[:, 0], c[:, 2] - c[:, 0]
    cr = np.cross(e1, e2)
    fn = OO._normalize(cr)
    crn = np.linalg.norm(cr, axis=1)
    cond = 1.0 + np.linalg.norm(e1, axis=1) * np.linalg.norm(e2, axis=1) / np.where(crn > 0, crn, 1.0)
    out, mag = np.zeros(verts.shape), np.zeros(len(verts))
    for i in range(3):
        np.add.at(out, faces[:, i], fn)
        np.add.at(mag, faces[:, i], np.linalg.norm(fn, axis=1) * cond)
    return out, mag


@gpu
@pytest.mark.parametrize("mesh", ["degenerate", "fan2000", "two_components"])
def test_vertex_frames(cuda, mesh):
    verts, faces = GEOM_MESHES[mesh]()
    V, F = len(verts), len(faces)
    v64, f64 = torch.from_numpy(verts).to(cuda), torch.from_numpy(faces).to(cuda)
    # the first pass marks exactly the vertices whose summed face normal is zero (the oracle's NaN rows)
    nrm = torch.empty(V, 3, dtype=torch.float64, device=cuda)
    fr = torch.empty(V, 3, 3, dtype=torch.float64, device=cuda)
    nbad = torch.zeros(1, dtype=torch.int32, device=cuda)
    ws = torch.empty(12 * F + 8 * V + 1024, dtype=torch.uint8, device=cuda)
    assert _lib().dn_vertex_frames(_p(v64), _p(f64), F, V, None, _p(nrm), _p(fr), _p(nbad), _p(ws), ws.numel(),
                                   dn.ops._stream()) == DN_OK
    summed, mag = _summed_face_normals(verts, faces)
    zero = np.linalg.norm(summed, axis=1) == 0
    assert np.array_equal(np.isnan(_np(nrm)).any(1), zero)
    assert int(nbad.item()) == int(zero.sum())
    if mesh == "degenerate":
        assert zero.sum() == 4                                 # the collinear component and the lone vertex
    frames = _np(dn.geometry._vertex_frames(v64, f64, None, torch.float64, verts))
    gold = OO.tangent_frames(verts, faces)
    n_gold = gold[:, 2]
    # the basis switch at |n_x| = 0.9 is discontinuous: a vertex within rounding of it is not comparable
    keep = np.abs(np.abs(n_gold[:, 0]) - 0.9) >= 1e-12
    deg = np.bincount(faces.reshape(-1), minlength=V)
    kappa = np.where(zero, 1.0, mag / np.maximum(np.linalg.norm(summed, axis=1), 1e-300))
    bound = (gamma(8 * deg + 64) * kappa)[:, None, None] * np.ones((1, 3, 3))
    _assert_within(frames[keep], gold[keep], bound[keep], "vertex_frames " + mesh)


def _grad_edges(rs):
    """User edges: a valence-2000 row, one neighbour, collinear neighbours, a self loop and a duplicate, a vertex with
    no outgoing edge, random rows; shuffled."""
    V = 2100
    e = [(0, j) for j in range(1, 2001)]
    e += [(1, 2)]
    e += [(2, 3), (2, 4), (2, 5)]
    e += [(3, 3), (3, 4), (3, 4), (3, 6)]
    for v in range(5, V):
        e += [(v, int(j)) for j in rs.choice(V, 3, replace=False) if j != v]
    e = np.array(e, dtype=np.int64).T
    e = e[:, rs.permutation(e.shape[1])]
    et = rs.randn(e.shape[1], 2).astype(np.float32)
    et[e[0] == 2] = np.array([[1.0], [-2.0], [0.5]], np.float32) * np.array([[0.6, 0.8]], np.float32)
    return V, e, et


@gpu
def test_build_grad_user_edges(cuda):
    rs = np.random.RandomState(11)
    V, e, et = _grad_edges(rs)
    g = dn.geometry.build_grad_operators(torch.empty(V, 3, device=cuda), torch.empty(V, 3, 3, device=cuda),
                                         torch.from_numpy(e).to(cuda), edge_tangent=torch.from_numpy(et).to(cuda))
    rowptr, colidx, vals = (t.numpy() for t in g.to_host_csr())
    vals = vals.astype(np.float64)
    mine = sp.csr_matrix((vals[:, 0] + 1j * vals[:, 1], colidx, rowptr), shape=(V, V))
    mine.sum_duplicates()
    gold = O.build_grad(V, e, et.astype(np.float64)).tocsr()
    gold.sum_duplicates()
    assert np.array_equal(mine.indptr, gold.indptr) and np.array_equal(mine.indices, gold.indices)
    rows = np.repeat(np.arange(V), np.diff(gold.indptr))
    rowmax = np.maximum.reduceat(np.abs(gold.data), gold.indptr[:-1])
    bound = 2 * U32 * rowmax[rows]
    for part in (np.real, np.imag):
        _assert_within(part(mine.data), part(gold.data), bound, "build_grad")
    assert np.diff(gold.indptr)[4] == 1                       # vertex 4: no outgoing edge, only itself (coef 0)
    keep = ~((e[0] == 0) & (e[1] == 7))                       # drop one edge of the valence-2000 row
    pert = O.build_grad(V, e[:, keep], et[keep].astype(np.float64)).tocsr()
    row0, prow0 = gold[0].toarray().ravel(), pert[0].toarray().ravel()
    b0 = 2 * U32 * np.abs(row0).max()
    _assert_rejects(row0.real, prow0.real, b0, "build_grad")
    _assert_rejects(row0.imag, prow0.imag, b0, "build_grad")
    # the drop-in returns the same matrix
    M = dn.geometry.build_grad(np.zeros((V, 3)), e, et).tocsr()
    M.sum_duplicates()
    assert abs(M - mine).max() == 0


# ------------------------------------------------------------------------------------------------
# 3. the solver where the driver branches
# ------------------------------------------------------------------------------------------------
def _device_op(verts, faces, dev):
    rowptr, colidx, lvals, mass, avals, adiag, bound = _device_laplacian(verts, faces, dev)
    return eigen.LaplaceOperator(len(verts), rowptr, colidx, avals, adiag, mass, bound)


def _check_solution(lam, phi, mesh, k, what, rel=1e-8):
    """Eigenvalues within ``rel`` lambda_{k-1} of dense eigh, the projector onto the leading k' (ending at a relative
    gap >= 1e-3) within Davis-Kahan's residual / gap, M-orthonormality, and the fp64 residual of every pair:
    ||M^-1/2 (L phi + eps phi - lambda M phi)|| = ||A y - theta y|| <= 1e-8 lambda_{k-1} (the solver stops at 1e-9)."""
    _, _, L, m, glam, gphi = dense_gold(mesh)
    scale = glam[k - 1]
    err = np.abs(lam - np.clip(glam[:k], 0.0, None)).max()
    print("MEASURED {} eval_err_over_lambda_k={:.3e}".format(what, err / scale))
    assert err <= rel * scale, (what, err / scale)
    kp = _kprime(glam, k)
    assert kp > 0
    assert _projector_err(phi[:, :kp], gphi[:, :kp], m) <= 100 * 1e-9 * scale / (glam[kp] - glam[kp - 1])
    assert np.abs(phi.T @ (phi * m[:, None]) - np.eye(k)).max() <= 1e-9
    R = (L @ phi + SHIFT * phi - (phi * m[:, None]) * lam[None, :]) / np.sqrt(m)[:, None]
    assert np.all(np.linalg.norm(R, axis=0) <= 1e-8 * scale)


def _solve_twice(op, k):
    a = eigen.lowest_eigenpairs(op, k)
    b = eigen.lowest_eigenpairs(op, k)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    return _np(a[0]), _np(a[1])


@gpu
@pytest.mark.parametrize("case", sorted(SOLVER_CASES))
def test_lowest_eigenpairs_branches(cuda, case):
    mesh, k = SOLVER_CASES[case]
    verts, faces = dense_gold(mesh)[:2]
    lam, phi = _solve_twice(_device_op(verts, faces, cuda), k)
    _check_solution(lam, phi, mesh, k, "lowest_eigenpairs " + case)


@gpu
def test_lowest_eigenpairs_svqb(cuda, monkeypatch):
    """Every Cholesky reports failure, so each orthonormalisation takes the SVQB branch."""
    calls = []
    real = torch.linalg.cholesky_ex

    def failing(G, upper=False):
        calls.append(G.shape[0])
        R, info = real(G, upper=upper)
        return R, torch.ones_like(info)
    monkeypatch.setattr(torch.linalg, "cholesky_ex", failing)
    verts, faces = dense_gold("patch8x9")[:2]
    lam, phi = _solve_twice(_device_op(verts, faces, cuda), 30)
    assert len(calls) >= 4
    _check_solution(lam, phi, "patch8x9", 30, "lowest_eigenpairs svqb")


@gpu
def test_lowest_eigenpairs_no_convergence(cuda, monkeypatch):
    monkeypatch.setattr(eigen, "MAX_ITERATIONS", 0)
    verts, faces = _np_mesh(dn.synthetic.icosphere_mesh(3, seed=5))
    with pytest.raises(ValueError, match="failed to compute eigendecomp"):
        eigen.lowest_eigenpairs(_device_op(verts, faces, cuda), 40)


@gpu
def test_compute_operators_k_eig_at_vertex_count(cuda):
    verts, faces = dn.synthetic.patch_mesh(6, 7, seed=3)
    with pytest.raises(ValueError, match="failed to compute eigendecomp"):
        dn.geometry.compute_operators(verts, faces, 42, device=cuda)
    out = dn.geometry.compute_operators(verts, faces, 41, device=cuda)
    assert out[3].shape == (41,)


# ------------------------------------------------------------------------------------------------
# 4. the driver on the CPU, and the host-side input checks (no GPU)
# ------------------------------------------------------------------------------------------------
class _DenseSolver(eigen._Solver):
    """eigen._Solver with the five kernels replaced by plain fp64 products on the CPU."""

    def __init__(self, op, k, B, seed):
        self.op, self.k, self.B, self.V = op, k, B, op.V
        self.dev = torch.device("cpu")
        gen = torch.Generator().manual_seed(seed)
        self.Q = torch.randn(self.V, B, generator=gen, dtype=torch.float64)
        self.T = [torch.empty(self.V, B, dtype=torch.float64) for _ in range(2)]
        self.W = torch.empty(self.V, B, dtype=torch.float64)
        self.W2 = torch.empty(self.V, B, dtype=torch.float64)
        self.steps = self.col_steps = 0
        self.ws = torch.empty(1)
        self.lib = types.SimpleNamespace(dn_eig_finalize=self._finalize)

    def filt(self, src, prev, dst, c0, alpha, beta, gamma_):
        Y = src[:, c0:].numpy()
        r = alpha * (self.op.A @ Y) + beta * Y
        if prev is not None:
            r = r + gamma_ * prev[:, c0:].numpy()
        dst[:, c0:] = torch.from_numpy(r)

    def gram(self, X, xc0, xn, Y, yc0, yn):
        return X[:, xc0:xc0 + xn].T @ Y[:, yc0:yc0 + yn]

    def rotate(self, X, xc0, kd, Cm, Z, zc0, n, beta=0.0):
        r = X[:, xc0:xc0 + kd] @ Cm
        Z[:, zc0:zc0 + n] = r if beta == 0.0 else beta * Z[:, zc0:zc0 + n] + r

    def residuals(self, Wb, Qb, c0, theta):
        return (Wb[:, c0:] - theta[None, :] * Qb[:, c0:]).norm(dim=0)

    def _finalize(self, y_ptr, ldy, cols_ptr, k, mass_ptr, V, out_ptr, *rest):
        arr = lambda p, n, t: np.ctypeslib.as_array((t * n).from_address(p))
        Y = arr(y_ptr, V * ldy, ctypes.c_double).reshape(V, ldy)
        cols = arr(cols_ptr, k, ctypes.c_int32)
        out = arr(out_ptr, V * k, ctypes.c_double).reshape(V, k)
        out[:] = finalize_np(Y, cols, arr(mass_ptr, V, ctypes.c_double))
        return 0


def test_driver_on_cpu(monkeypatch):
    """eigen.lowest_eigenpairs, unmodified, over dense fp64 kernels: a driver regression fails here on any machine."""
    monkeypatch.setattr(eigen, "_Solver", _DenseSolver)
    monkeypatch.setattr(eigen, "_event", lambda: None)
    monkeypatch.setattr(dn.ops, "_stream", lambda: None)
    for case in sorted(SOLVER_CASES):
        mesh, k = SOLVER_CASES[case]
        verts, faces = dense_gold(mesh)[:2]
        L, m, A = oracle_operator(verts, faces)
        op = types.SimpleNamespace(V=len(m), mass=torch.from_numpy(m), A=A,
                                   bound=float(abs(A).sum(1).max()), colidx=torch.zeros(1))
        lam, phi = (t.numpy() for t in eigen.lowest_eigenpairs(op, k))
        _check_solution(lam, phi, mesh, k, "driver on cpu " + case, rel=1e-12)


def test_lowest_eigenpairs_refuses_k_at_vertex_count():
    """The reference's eigsh(..., sigma=eps) refuses k >= V, and its retries end in this ValueError."""
    V = 12
    op = eigen.LaplaceOperator(V, None, None, None, None, torch.ones(V, dtype=torch.float64), 1.0)
    for k in (V, V + 1):
        with pytest.raises(ValueError, match="failed to compute eigendecomp"):
            eigen.lowest_eigenpairs(op, k)


def test_build_grad_refuses_bad_edges():
    V = 6
    verts, frames = torch.zeros(V, 3), torch.zeros(V, 3, 3)
    good = torch.tensor([[0, 1, 2], [1, 2, 3]])
    for bad in ([[0, 6], [1, 2]], [[0, 1], [1, 6]], [[-1, 1], [1, 2]], [[0, 1], [-3, 2]]):
        with pytest.raises(IndexError):
            dn.geometry.build_grad_operators(verts, frames, torch.tensor(bad))
        with pytest.raises(IndexError):
            dn.geometry.build_grad(np.zeros((V, 3)), np.array(bad), np.zeros((2, 2), np.float32))
    for et in (np.zeros((2, 2), np.float32), np.zeros((3, 3), np.float32), np.zeros((3,), np.float32)):
        with pytest.raises(ValueError):
            dn.geometry.build_grad_operators(verts, frames, good, edge_tangent=torch.from_numpy(et))
        with pytest.raises(ValueError):
            dn.geometry.build_grad(np.zeros((V, 3)), good.numpy(), et)
