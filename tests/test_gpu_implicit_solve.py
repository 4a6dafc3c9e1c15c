"""The implicit heat-diffusion solve (dn_implicit.cu's ``implicit_cg_kernel``, through dn_implicit_diffusion_fwd / _bwd)
against fp64, at every column group, at the row counts where its cooperative grid changes shape, per column, and at
the edges of its C-ABI; then the implicit net at tensor-core widths against fp64 autograd.

Gold: ``oracle/dn_oracle_implicit.implicit_diffusion`` (a scipy ``splu`` per distinct time, and its adjoint) on the
fp32-rounded L and mass the kernel sees, promoted to fp64.  With u = 2^-24, eps = 2^-53 and A_c = M + t_c L, per
column c of an fp32 result y (forward, b = M x) or w (backward, b = g; recovered as grad_x / m):

  residual  ||b_c - A_c y_c||_2 <= 2 rtol ||b_c||_2 + u (1 + 2u) || |A_c| |y_c| ||_2 + gamma_{n+2} || |A_c| |y_c| ||_2
            the solver's stopping test (2x for drift between the recurrence and the true residual), the final rounding
            to fp32 (componentwise, so never looser than ||A_c||_2 u ||y_c||_2), and the CPU's own fp64 evaluation
            (n = the longest row).  Needs no direct solve, so it also runs at V = 200k.
  error     ||y_c - y*_c||_inf <= (residual_c + ||b_c - A_c y*_c||_2) / lambda_min(A_c) + u ||y*_c||_inf
            lambda_min from the same factorisation (eigsh, shift-invert at 0) or eigvalsh at small V, once per
            distinct t_c.  L rounded to fp32 is not exactly PSD (L 1 != 0 by about u |L_vv|), so lambda_min >= min m
            is not assumed.
  grad_time[c] = -w_c . (L y_c) with y the fp32 forward output the kernel reads: the gold uses w*, and the bound
            propagates w's error bound through ||L y_c||_2, adds the fp64 sums' gamma terms and u |gold| for the store.

``test_bounds_reject_structural_errors`` (CPU) applies four structural errors to the gold and requires each to exceed
the residual bound 100x somewhere in its cases.

Why the grid cases: ``launch_nc`` sizes the grid as min(resident CTAs, ceil(V / 8), 1024); rows go round-robin over
all warps and every reduction is a per-CTA partial summed over the CTAs in index order.  The resident count comes from
the occupancy API inside the launch (on an H100 about 132, 264 or 396 CTAs, depending on the instantiation's
registers), so the tori bracket 8x each of those counts and go past 8192 rows."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import scipy.linalg as sl
import scipy.sparse as sp
import scipy.sparse.linalg as sla
import torch

from conftest import ROOT
from test_gpu_implicit import _checkpoint_times, _close, _sparse
from test_gpu_operator_kernels import fan_mesh, two_components_mesh, two_tori_mesh

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle_implicit as OI  # noqa: E402  (checker only)
import dn_oracle_torch as T  # noqa: E402  (checker only)
from ref_import import _cotan_laplacian, _vertex_areas  # noqa: E402

import diffusion_net_b200 as dn  # noqa: E402

gpu = pytest.mark.gpu
U = 2.0 ** -24
EPS = 2.0 ** -53
RTOL = dn.ops.IMPLICIT_RTOL
MAX_ITER = dn.ops.IMPLICIT_MAX_ITER
DN_OK, DN_ERR_INVALID_ARGUMENT, DN_ERR_UNSUPPORTED, DN_ERR_WORKSPACE = 0, -1, -2, -3
F_SENT = np.array([0x7FA1B2C3], dtype=np.int32).view(np.float32)[0]            # NaNs with a payload
D_SENT = np.array([0x7FF8DEADBEEF0001], dtype=np.int64).view(np.float64)[0]
COLUMNS = [1, 31, 32, 33, 63, 65, 96, 100, 129, 160, 191, 200, 224, 255, 256]


def gamma(n):
    return n * EPS / (1.0 - n * EPS)


def _bits32(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


# ---------------------------------------------------------------------------------------------------------------
# meshes: (L, m) as the kernel sees them, fp32-rounded and promoted to fp64
# ---------------------------------------------------------------------------------------------------------------
def _ops(verts, faces):
    """Cotan L and lumped mass (+ 1e-8 mean, as get_operators) of the mesh scaled to unit max radius."""
    v = np.asarray(verts, dtype=np.float64)
    v = v - v.mean(0)
    v /= np.linalg.norm(v, axis=1).max()
    f = np.asarray(faces, dtype=np.int64)
    L = sp.csr_matrix(_cotan_laplacian(v, f, denom_eps=1e-10)).astype(np.float32).astype(np.float64)
    m = _vertex_areas(v, f)
    m = (m + 1e-8 * m.mean()).astype(np.float32).astype(np.float64)
    L.sort_indices()
    return L, m


def _path(V, seed=0):
    """A hand-built SPD L: a weighted path graph's Laplacian plus 0.1 I (V = 1 is the 1 x 1 matrix [0.1])."""
    rs = np.random.RandomState(seed)
    w = (0.5 + rs.rand(max(V - 1, 0))).astype(np.float32).astype(np.float64)
    d = np.zeros(V) + 0.1
    d[:-1] += w
    d[1:] += w
    L = sp.diags([d, -w, -w], [0, 1, -1], shape=(V, V), format="csr").astype(np.float32).astype(np.float64)
    L.sort_indices()
    return L, (0.5 + rs.rand(V)).astype(np.float32).astype(np.float64)


def _torus(n, m, seed=1):
    v, f = dn.synthetic.torus_mesh(n, m, seed=seed)
    return _ops(v.numpy(), f.numpy())


MESHES = {
    "path1": lambda: _path(1), "path7": lambda: _path(7), "path8": lambda: _path(8), "path9": lambda: _path(9),
    "patch80": lambda: _ops(*(t.numpy() for t in dn.synthetic.patch_mesh(8, 10, seed=2))),
    "torus1200": lambda: _torus(30, 40),
    # 8x the resident CTAs (about 132, 264 and 396 on an H100) minus and plus a few rows
    "torus1040": lambda: _torus(26, 40), "torus1071": lambda: _torus(21, 51),
    "torus2100": lambda: _torus(30, 70), "torus2125": lambda: _torus(25, 85),
    "torus3150": lambda: _torus(45, 70), "torus3186": lambda: _torus(54, 59),
    "torus8184": lambda: _torus(88, 93), "torus8200": lambda: _torus(82, 100),
    "torus20k": lambda: _torus(100, 200, seed=0),
    "two_components": lambda: _ops(*two_components_mesh()),
    "unreferenced": lambda: _ops(*two_tori_mesh()),         # an empty L row, mass 1e-8 mean
    "fan2000": lambda: _ops(*fan_mesh()),                   # one row of 2001 entries
}
_mesh_cache = {}


def _mesh(name):
    if name not in _mesh_cache:
        _mesh_cache[name] = MESHES[name]()
    return _mesh_cache[name]


def _times(C, kind="checkpoint"):
    t = _checkpoint_times(512)
    if kind == "checkpoint":
        return np.resize(t, C).astype(np.float32)
    if kind == "few":                                       # 16 distinct times: the grid cases keep the gold cheap
        return np.resize(t[:16], C).astype(np.float32)
    if kind == "edges":                                     # clamped entries, and columns that freeze far apart
        return np.resize(np.concatenate(([-1.0, 0.0, 1e-9, 0.5, 5.0], t[:11])), C).astype(np.float32)
    raise ValueError(kind)


def _data(V, C, seed):
    rs = np.random.RandomState(seed)
    return rs.randn(V, C).astype(np.float32), rs.randn(V, C).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------
# gold and bounds (CPU)
# ---------------------------------------------------------------------------------------------------------------
def _tc(t):
    return np.maximum(np.asarray(t, dtype=np.float64), np.float32(1e-8)).astype(np.float64)


def _apply(L, m, t, y, absolute=False):
    """A_c y_c per column in fp64 (|A_c| |y_c| with ``absolute``)."""
    y = np.asarray(y, dtype=np.float64)
    if absolute:
        return m[:, None] * np.abs(y) + abs(L) @ np.abs(y) * _tc(t)[None]
    return m[:, None] * y + (L @ y) * _tc(t)[None]


def residual_bound(L, m, t, b, y):
    """(||b_c - A_c y_c||_2, its bound) per column."""
    n = int(np.diff(L.indptr).max(initial=0)) + 2
    res = np.linalg.norm(b - _apply(L, m, t, y), axis=0)
    ay = np.linalg.norm(_apply(L, m, t, y, absolute=True), axis=0)
    return res, 2 * RTOL * np.linalg.norm(b, axis=0) + (U * (1 + 2 * U) + gamma(n)) * ay


def _lambda_min(L, m, t, lus):
    """lambda_min(M + t L) for each distinct clamped t, reusing the oracle's factorisations."""
    out = {}
    for tv in np.unique(_tc(t)):
        A = (sp.diags(m) + tv * L).tocsc()
        if A.shape[0] <= 600:
            out[tv] = float(sl.eigvalsh(A.toarray())[0])
        else:
            lu = lus[float(max(tv, 1e-8))]              # the oracle clamps at fp64 1e-8, the kernel at fp32 1e-8
            op = sla.LinearOperator(A.shape, matvec=lu.solve, dtype=np.float64)
            out[tv] = float(sla.eigsh(A, k=1, sigma=0.0, which="LM", OPinv=op, return_eigenvectors=False)[0])
        assert out[tv] > 0, (tv, out[tv])
    return np.array([out[v] for v in _tc(t)])


class Gold:
    """y*, w* (= A^-1 g) and lambda_min of one (mesh, x, t, g) case."""

    def __init__(self, L, m, x, t, g=None, lam=True):
        self.L, self.m, self.t = L, m, np.asarray(t, dtype=np.float32)
        self.b = m[:, None] * x.astype(np.float64)
        self.g = None if g is None else g.astype(np.float64)
        lus = {}
        if not lam:                                         # residual checks only: no direct solve
            self.y = self.w = self.lam = None
            return
        if g is None:
            self.y = OI.implicit_diffusion(x, m, L, self.t, lus=lus)
        else:
            self.y, gx, _ = OI.implicit_diffusion(x, m, L, self.t, grad_out=g, lus=lus)
            self.w = gx / m[:, None]
        self.lam = _lambda_min(L, m, self.t, lus)

    def error_bound(self, b, y, gold):
        res, rb = residual_bound(self.L, self.m, self.t, b, y)
        gres = np.linalg.norm(b - _apply(self.L, self.m, self.t, gold), axis=0)
        return res, rb, (res + gres) / self.lam + U * np.abs(gold).max(0)


def _within(what, err, bound):
    err, bound = np.asarray(err, dtype=np.float64), np.asarray(bound, dtype=np.float64)
    ratio = float(np.max(err / np.maximum(bound, 1e-300)))
    assert np.all(err <= bound), "{}: worst err / bound = {:.3g} (column {})".format(what, ratio,
                                                                                    int(np.argmax(err / bound)))
    print("MEASURED {} max_err_over_bound={:.3e}".format(what, ratio))
    return ratio


def check_forward(gold, y, what):
    """Residual and (where lambda is known) error bounds of the fp32 forward output y against ``gold``."""
    y = np.asarray(y, dtype=np.float64)
    if gold.lam is None:
        res, rb = residual_bound(gold.L, gold.m, gold.t, gold.b, y)
        _within(what + " fwd residual", res, rb)
        return
    res, rb, eb = gold.error_bound(gold.b, y, gold.y)
    _within(what + " fwd residual", res, rb)
    _within(what + " fwd error", np.abs(y - gold.y).max(0), eb)


def check_backward(gold, y, gx, gt, what, gt0=None):
    """grad_x = M w and grad_time against w* and -w* . (L y) (y: the fp32 forward output the kernel read)."""
    L, m = gold.L, gold.m
    w = np.asarray(gx, dtype=np.float64) / m[:, None]
    ly = L @ np.asarray(y, dtype=np.float64)
    if gold.lam is None:
        res, rb = residual_bound(L, m, gold.t, gold.g, w)
        _within(what + " bwd residual", res, rb)
        return
    res, rb, eb = gold.error_bound(gold.g, w, gold.w)
    _within(what + " bwd residual", res, rb)
    _within(what + " bwd error", np.abs(w - gold.w).max(0), eb)
    gt_gold = -np.einsum("vc,vc->c", gold.w, ly)
    ay = np.linalg.norm(_apply(L, m, gold.t, w, absolute=True), axis=0)
    gres = np.linalg.norm(gold.g - _apply(L, m, gold.t, gold.w), axis=0)
    w_err = (res + U * (1 + 2 * U) * ay + gres) / gold.lam          # ||w_fp64 - w*||_2 (w_fp64: before the store)
    n = L.shape[0] + int(np.diff(L.indptr).max(initial=0))
    sums = 2 * gamma(n) * np.einsum("vc,vc->c", np.abs(w), abs(L) @ np.abs(np.asarray(y, dtype=np.float64)))
    bound = w_err * np.linalg.norm(ly, axis=0) + sums + U * (1 + 2 * U) * (np.abs(gt_gold) + w_err * np.linalg.norm(
        ly, axis=0) + sums)
    got = np.asarray(gt, dtype=np.float64) - (0.0 if gt0 is None else gt0)
    _within(what + " grad_time", np.abs(got - gt_gold), bound)


def check_status(st, C, zero_cols=()):
    its, rel = st[2:2 + C], st[2 + C:]
    assert st[0] == 0
    assert np.all(rel <= RTOL), rel.max()
    assert st[1] == its.max()
    assert np.all(its == np.round(its)) and np.all(its >= 0)
    for c in zero_cols:
        assert its[c] == 0 and rel[c] == 0, (c, its[c], rel[c])


# ---------------------------------------------------------------------------------------------------------------
# GPU plumbing: the C-ABI called directly, every output prefilled with a sentinel
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    dn._lib.load()
    return torch.device("cuda")


class Dev:
    """One mesh on the device: its LaplacianCSR (from a coalesced COO of the fp32 L, or ``Lt`` as given) and mass."""

    def __init__(self, L, m, Lt=None):
        Lc = L.tocoo()
        self.V = L.shape[0]
        self.Lt = Lt if Lt is not None else _sparse(Lc.row, Lc.col, Lc.data.astype(np.float32), self.V, "cuda")
        self.lap = dn.ops.LaplacianCSR(self.Lt)
        self.mass = torch.from_numpy(m.astype(np.float32)).cuda()


def _sent32(shape):
    return torch.full(shape, int(_bits32([F_SENT])[0]), dtype=torch.int32, device="cuda").view(torch.float32)


def _sent64(n):
    return torch.full((n,), int(np.float64(D_SENT).view(np.int64)), dtype=torch.int64, device="cuda").view(
        torch.float64)


def _ws(V, Cc, short=0):
    return torch.empty(int(dn._lib.load().dn_implicit_diffusion_workspace_bytes(V, Cc)) - short, dtype=torch.uint8,
                       device="cuda")


def fwd(dev, x, t, max_iter=MAX_ITER, rtol=RTOL):
    """(rc, y, time after the call, status) of dn_implicit_diffusion_fwd."""
    lib = dn._lib.load()
    V, Cc = x.shape
    xd = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()
    td = torch.from_numpy(np.array(t, dtype=np.float32)).cuda()
    y, st, ws = _sent32((V, Cc)), _sent64(2 + 2 * Cc), _ws(V, Cc)
    rc = lib.dn_implicit_diffusion_fwd(C.byref(dev.lap.csr[0]), xd.data_ptr(), dev.mass.data_ptr(), td.data_ptr(), V,
                                       Cc, float(rtol), int(max_iter), y.data_ptr(), st.data_ptr(), ws.data_ptr(),
                                       ws.numel(), dn.ops._stream())
    torch.cuda.synchronize()
    return rc, y.cpu().numpy(), td.cpu().numpy(), st.cpu().numpy()


def bwd(dev, g, t, y, gt0=None, max_iter=MAX_ITER, rtol=RTOL):
    """(rc, grad_x, grad_time, time after the call, status) of dn_implicit_diffusion_bwd; grad_time starts at gt0."""
    lib = dn._lib.load()
    V, Cc = g.shape
    gd, td, yd = (torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda() for a in (g, t, y))
    gx, st, ws = _sent32((V, Cc)), _sent64(2 + 2 * Cc), _ws(V, Cc)
    gt = torch.from_numpy(np.zeros(Cc, np.float32) if gt0 is None else np.array(gt0, dtype=np.float32)).cuda()
    rc = lib.dn_implicit_diffusion_bwd(C.byref(dev.lap.csr[0]), gd.data_ptr(), dev.mass.data_ptr(), td.data_ptr(),
                                       yd.data_ptr(), V, Cc, float(rtol), int(max_iter), gx.data_ptr(), gt.data_ptr(),
                                       st.data_ptr(), ws.data_ptr(), ws.numel(), dn.ops._stream())
    torch.cuda.synchronize()
    return rc, gx.cpu().numpy(), gt.cpu().numpy(), td.cpu().numpy(), st.cpu().numpy()


def run_case(L, m, x, t, g, what, lam=True, zero_cols=()):
    """Forward and backward of one case on the GPU, every bound and status check; returns the GPU results."""
    dev = Dev(L, m)
    rc, y, t_after, st = fwd(dev, x, t)
    assert rc == DN_OK
    assert np.array_equal(_bits32(t_after), _bits32(np.maximum(t, np.float32(1e-8))))   # fmaxf(t, 1e-8f), bitwise
    check_status(st, x.shape[1], zero_cols)
    rc, gx, gt, t_b, st_b = bwd(dev, g, t_after, y)
    assert rc == DN_OK
    assert np.array_equal(_bits32(t_b), _bits32(t_after))                                 # the backward leaves time
    check_status(st_b, x.shape[1], zero_cols)
    print("{}: {} / {} iterations (fwd / bwd)".format(what, int(st[1]), int(st_b[1])))
    gold = Gold(L, m, x, t, g, lam=lam)
    check_forward(gold, y, what)
    check_backward(gold, y, gx, gt, what)
    return y, gx, gt, st, st_b


# ---------------------------------------------------------------------------------------------------------------
# 1. every column group, every grid shape, times and meshes
# ---------------------------------------------------------------------------------------------------------------
# NC = 1..8 and partial lane groups; 16 distinct times keep the gold's factorisations few, except at C = 1, 33, 256
CASES = {"c{}".format(c): ("torus1200", c, "checkpoint" if c in (1, 33, 256) else "few") for c in COLUMNS}
CASES.update({
    "path1": ("path1", 33, "few"), "path7": ("path7", 33, "few"), "path8": ("path8", 33, "few"),
    "path9": ("path9", 1, "few"), "path9_c256": ("path9", 256, "few"), "patch80": ("patch80", 65, "checkpoint"),
    "torus1040": ("torus1040", 256, "few"), "torus1071": ("torus1071", 256, "few"),      # NC = 8: 1 CTA / SM
    "torus2100": ("torus2100", 64, "few"), "torus2125": ("torus2125", 64, "few"),        # NC = 2: 2 CTAs / SM
    "torus3150": ("torus3150", 32, "few"), "torus3186": ("torus3186", 32, "few"),        # NC = 1: 3 CTAs / SM
    "torus8184": ("torus8184", 128, "few"), "torus8200": ("torus8200", 128, "few"),
    "torus20k": ("torus20k", 128, "checkpoint"),
    "edge_times": ("torus1200", 40, "edges"),
    "two_components": ("two_components", 33, "checkpoint"),
    "unreferenced": ("unreferenced", 33, "checkpoint"),
    "fan2000": ("fan2000", 65, "checkpoint"),
})


@gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_solve_within_bounds(cuda, case):
    mesh, Cc, kind = CASES[case]
    L, m = _mesh(mesh)
    x, g = _data(L.shape[0], Cc, seed=Cc)
    t = _times(Cc, kind)
    zero = [c for c in (2, 5) if c < Cc and L.shape[0] > 1]          # b_c = 0: never starts
    for c in zero:
        x[:, c] = 0.0
        g[:, c] = 0.0
    run_case(L, m, x, t, g, case, zero_cols=zero)


@gpu
def test_200k_residual(cuda):
    """V = 200k at the checkpoint's times, forward and backward: the residual bound only (no direct solve)."""
    L, m = _torus(400, 500, seed=0)
    x, g = _data(L.shape[0], 128, seed=7)
    run_case(L, m, x, _times(128), g, "torus200k", lam=False)


@gpu
def test_uncoalesced_laplacian_is_bitwise_the_coalesced(cuda):
    """An uncoalesced COO L (every entry split into two exact halves, shuffled) builds the same CSR: bitwise outputs."""
    L, m = _mesh("patch80")
    Lc = L.tocoo()
    rs = np.random.RandomState(0)
    rows, cols = np.concatenate((Lc.row, Lc.row)), np.concatenate((Lc.col, Lc.col))
    vals = np.concatenate((Lc.data, Lc.data)).astype(np.float32) * np.float32(0.5)
    p = rs.permutation(len(rows))
    idx = torch.from_numpy(np.stack((rows[p], cols[p])).astype(np.int64))
    Lu = torch.sparse_coo_tensor(idx, torch.from_numpy(vals[p]), L.shape).cuda()
    assert not Lu.is_coalesced()
    x, g = _data(L.shape[0], 40, seed=1)
    t = _times(40)
    outs = []
    for dev in (Dev(L, m), Dev(L, m, Lt=Lu)):
        _, y, _, st = fwd(dev, x, t)
        _, gx, gt, _, st_b = bwd(dev, g, np.maximum(t, np.float32(1e-8)), y)
        outs.append((y, gx, gt, st, st_b))
    for a, b in zip(*outs):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


# ---------------------------------------------------------------------------------------------------------------
# 2. column independence, bitwise
# ---------------------------------------------------------------------------------------------------------------
def _both(dev, x, t, g):
    _, y, t_after, st = fwd(dev, x, t)
    _, gx, gt, _, st_b = bwd(dev, g, t_after, y)
    return y, gx, gt, st, st_b


@gpu
@pytest.mark.parametrize("Cc", [33, 200])
def test_columns_are_independent_bitwise(cuda, Cc):
    L, m = _mesh("torus1200")
    dev = Dev(L, m)
    x, g = _data(L.shape[0], Cc, seed=11)
    t = _times(Cc, "edges")
    y, gx, gt, st, st_b = _both(dev, x, t, g)
    # a permutation of the columns permutes every output, status included
    p = np.random.RandomState(1).permutation(Cc)
    y2, gx2, gt2, st2, st2_b = _both(dev, x[:, p], t[p], g[:, p])
    for a, b in ((y[:, p], y2), (gx[:, p], gx2), (gt[p], gt2)):
        assert np.array_equal(_bits32(a), _bits32(b))
    for s, s2 in ((st, st2), (st_b, st2_b)):
        assert s2[0] == s[0] and s2[1] == s[1]
        assert np.array_equal(s[2:2 + Cc][p], s2[2:2 + Cc]) and np.array_equal(s[2 + Cc:][p], s2[2 + Cc:])
    # every column but c changed: column c is unchanged
    c = Cc // 2
    rs = np.random.RandomState(2)
    x3, g3 = rs.randn(*x.shape).astype(np.float32), rs.randn(*g.shape).astype(np.float32)
    t3 = (_times(Cc)[::-1] * np.float32(1.7)).copy()
    x3[:, c], g3[:, c], t3[c] = x[:, c], g[:, c], t[c]
    y3, gx3, gt3, st3, st3_b = _both(dev, x3, t3, g3)
    assert np.array_equal(_bits32(y3[:, c]), _bits32(y[:, c]))
    assert np.array_equal(_bits32(gx3[:, c]), _bits32(gx[:, c]))
    assert _bits32(gt3[c:c + 1]) == _bits32(gt[c:c + 1])
    assert st3[2 + c] == st[2 + c] and st3[2 + Cc + c] == st[2 + Cc + c]


@gpu
def test_column_result_does_not_depend_on_the_column_count(cuda):
    """At V = 80 the grid is ceil(V / 8) = 10 CTAs for every instantiation (fewer than any SM count holds), so the
    grid, and with it every reduction order, is the same at C = 1 and C = 256.  Column 0 must then be bitwise the same:
    any difference is a column reading another column's data (or a lane group's mask), not rounding."""
    L, m = _mesh("patch80")
    dev = Dev(L, m)
    x, g = _data(L.shape[0], 256, seed=12)
    t = _times(256)
    full = _both(dev, x, t, g)
    one = _both(dev, x[:, :1].copy(), t[:1].copy(), g[:, :1].copy())
    assert np.array_equal(_bits32(full[0][:, 0]), _bits32(one[0][:, 0]))
    assert np.array_equal(_bits32(full[1][:, 0]), _bits32(one[1][:, 0]))
    assert _bits32(full[2][:1]) == _bits32(one[2][:1])
    assert full[3][2] == one[3][2] and full[4][2] == one[4][2]


# ---------------------------------------------------------------------------------------------------------------
# 3. C-ABI contracts
# ---------------------------------------------------------------------------------------------------------------
@gpu
def test_grad_time_accumulates(cuda):
    L, m = _mesh("torus1200")
    dev = Dev(L, m)
    x, g = _data(L.shape[0], 65, seed=13)
    t = _times(65)
    _, y, t_after, _ = fwd(dev, x, t)
    _, _, r, _, _ = bwd(dev, g, t_after, y)
    g0 = np.random.RandomState(3).randn(65).astype(np.float32)
    _, _, acc, _, _ = bwd(dev, g, t_after, y, gt0=g0)
    assert np.array_equal(_bits32(acc), _bits32(g0 + r))                # fl32(g0 + r), bitwise


@gpu
def test_unconverged_solve_writes_nothing(cuda):
    L, m = _mesh("torus1200")
    dev = Dev(L, m)
    x, g = _data(L.shape[0], 33, seed=14)
    t = _times(33, "edges")
    _, y_ok, t_ok, _ = fwd(dev, x, t)
    rc, y, t_after, st = fwd(dev, x, t, max_iter=2)
    assert rc == DN_OK and st[0] > 0 and st[1] == 2
    assert np.all(_bits32(y) == _bits32(F_SENT))
    assert np.array_equal(_bits32(t_after), _bits32(t_ok))             # the clamp is written anyway
    g0 = np.full(33, 0.25, np.float32)
    rc, gx, gt, _, st_b = bwd(dev, g, t_ok, y_ok, gt0=g0, max_iter=2)
    assert rc == DN_OK and st_b[0] > 0
    assert np.all(_bits32(gx) == _bits32(F_SENT))
    assert np.array_equal(gt, g0)                                       # not accumulated


def _abi_refusals(L_ptrs, V, ptr):
    """Every refusal of dn_implicit_diffusion_fwd / _bwd, with the launch counter unchanged.  ``ptr(n)`` returns a
    pointer to n bytes; nothing behind it is read before the argument checks fail."""
    lib = dn._lib.load()
    csr = dn._lib.dn_csr(*L_ptrs)
    n0 = lib.dn_kernel_launch_count()

    def call(Cc, rtol=RTOL, max_iter=MAX_ITER, short=0, backward=False):
        ws = int(lib.dn_implicit_diffusion_workspace_bytes(V, Cc))
        p = ptr(4 * V * max(Cc, 1))
        args = (C.byref(csr), p, ptr(4 * V), ptr(4 * max(Cc, 1)))
        tail = (V, Cc, float(rtol), int(max_iter), p, ptr(8 * (2 + 2 * max(Cc, 1))), ptr(ws), ws - short, None)
        if backward:
            return lib.dn_implicit_diffusion_bwd(*args, p, *tail[:5], ptr(4 * max(Cc, 1)), *tail[5:])
        return lib.dn_implicit_diffusion_fwd(*args, *tail)

    for bw in (False, True):
        assert call(33, short=1, backward=bw) == DN_ERR_WORKSPACE
        assert call(257, backward=bw) == DN_ERR_UNSUPPORTED
        assert call(33, rtol=-1e-8, backward=bw) == DN_ERR_INVALID_ARGUMENT
        assert call(33, rtol=float("nan"), backward=bw) == DN_ERR_INVALID_ARGUMENT
        assert call(33, max_iter=0, backward=bw) == DN_ERR_INVALID_ARGUMENT
        assert call(0, backward=bw) == DN_ERR_INVALID_ARGUMENT
    assert lib.dn_implicit_diffusion_workspace_bytes(V, 0) == -1
    assert lib.dn_kernel_launch_count() == n0                           # nothing was enqueued


def test_abi_refusals_enqueue_nothing():
    """Runs without a device: the checks refuse before touching any pointer (these point into host buffers)."""
    keep = []

    def ptr(n):
        keep.append(np.zeros(max(int(n), 1), np.uint8))
        return keep[-1].ctypes.data

    _abi_refusals((ptr(4 * 81), ptr(4 * 300), ptr(8 * 300), 300), 80, ptr)


@gpu
@pytest.mark.parametrize("Cc", [33, 200])
def test_two_calls_bitwise_20k(cuda, Cc):
    L, m = _mesh("torus20k")
    dev = Dev(L, m)
    x, g = _data(L.shape[0], Cc, seed=15)
    t = _times(Cc)
    a, b = _both(dev, x, t, g), _both(dev, x, t, g)
    for u, v in zip(a, b):
        assert np.array_equal(u.view(np.uint8), v.view(np.uint8))


# ---------------------------------------------------------------------------------------------------------------
# 4. non-finite columns: NaN out, promptly, the other columns untouched
# ---------------------------------------------------------------------------------------------------------------
PROMPT = 8          # iterations a non-finite column may take before it is frozen


def _nan_setup():
    L, m = _mesh("torus1200")
    dev = Dev(L, m)
    x, g = _data(L.shape[0], 40, seed=16)
    t = _times(40, "edges")
    return L, m, dev, x, g, t


def _assert_nan_column(a, c, what):
    assert np.all(np.isnan(a[..., c])), what + ": the column is not all NaN"


def _assert_others_bitwise(a, ref, c, what):
    keep = np.ones(a.shape[-1], bool)
    keep[c] = False
    assert np.array_equal(_bits32(a[..., keep]), _bits32(ref[..., keep])), what + ": another column changed"


@gpu
def test_nan_in_one_column(cuda):
    L, m, dev, x, g, t = _nan_setup()
    y, gx, gt, st, st_b = _both(dev, x, t, g)
    tc = np.maximum(t, np.float32(1e-8))
    # forward: a NaN in x column 5
    xn = x.copy()
    xn[17, 5] = np.nan
    rc, yn, _, stn = fwd(dev, xn, t)
    assert rc == DN_OK and stn[0] == 0 and stn[2 + 5] <= PROMPT and np.isnan(stn[2 + 40 + 5])
    _assert_nan_column(yn, 5, "fwd")
    _assert_others_bitwise(yn, y, 5, "fwd")
    # backward: a NaN in g column 5, against the same call without it
    gn = g.copy()
    gn[17, 5] = np.nan
    rc, gxn, gtn, _, stn_b = bwd(dev, gn, tc, y)
    assert rc == DN_OK and stn_b[0] == 0 and stn_b[2 + 5] <= PROMPT and np.isnan(stn_b[2 + 40 + 5])
    _assert_nan_column(gxn, 5, "grad_x")
    _assert_others_bitwise(gxn, gx, 5, "grad_x")
    assert np.isnan(gtn[5])
    _assert_others_bitwise(gtn[None], gt[None], 5, "grad_time")
    # through ops: a NaN upstream gradient reaches grad_time instead of vanishing
    ltd = dn.LearnedTimeDiffusion(40, method="implicit_dense").cuda()
    with torch.no_grad():
        ltd.diffusion_time.copy_(torch.from_numpy(t))
    xt = torch.from_numpy(x).cuda().requires_grad_(True)
    (ltd(xt, dev.Lt, dev.mass, None, None) * torch.from_numpy(gn).cuda()).sum().backward()
    assert torch.isnan(ltd.diffusion_time.grad[5]) and torch.isnan(xt.grad[:, 5]).all()
    assert torch.isfinite(ltd.diffusion_time.grad[:5]).all()


@gpu
def test_nan_mass_makes_everything_nan_promptly(cuda):
    L, m, dev, x, g, t = _nan_setup()
    dev.mass[3] = float("nan")
    rc, y, _, st = fwd(dev, x, t)
    assert rc == DN_OK and st[0] == 0 and st[1] <= PROMPT
    assert np.all(np.isnan(y)) and np.all(np.isnan(st[2 + 40:]))
    rc, gx, gt, _, st_b = bwd(dev, g, np.maximum(t, np.float32(1e-8)), np.zeros_like(x))
    assert rc == DN_OK and st_b[0] == 0 and st_b[1] <= PROMPT
    assert np.all(np.isnan(gx)) and np.all(np.isnan(gt))


@gpu
def test_inf_in_one_column(cuda):
    L, m, dev, x, g, t = _nan_setup()
    y, _, _, _, _ = _both(dev, x, t, g)
    xi = x.copy()
    xi[17, 7] = np.inf
    rc, yi, _, st = fwd(dev, xi, t)
    assert rc == DN_OK and st[0] == 0 and st[2 + 7] <= PROMPT and np.isnan(st[2 + 40 + 7])
    _assert_nan_column(yi, 7, "fwd")
    _assert_others_bitwise(yi, y, 7, "fwd")


@gpu
def test_nan_in_laplacian_freezes_promptly(cuda):
    """A NaN L value reaches every column through p.q: each is NaN after its first iteration, not at max_iter."""
    L, m = _mesh("patch80")
    Ln = L.copy()
    Ln.data[len(Ln.data) // 2] = np.nan
    dev = Dev(Ln, m)
    x, _ = _data(L.shape[0], 33, seed=17)
    rc, y, _, st = fwd(dev, x, _times(33))
    assert rc == DN_OK and st[0] == 0 and st[1] <= PROMPT
    assert np.all(np.isnan(y))


# ---------------------------------------------------------------------------------------------------------------
# 5. a (B, V, C) stack of two different meshes, through the layer and through a 2-block net
# ---------------------------------------------------------------------------------------------------------------
def _two_meshes():
    (La, ma), (Lb, mb) = _torus(30, 40, seed=1), _torus(30, 40, seed=9)
    assert La.shape == Lb.shape and abs(La - Lb).max() > 1e-3
    return [(La, ma), (Lb, mb)]


@gpu
def test_stack_of_different_meshes(cuda):
    meshes = _two_meshes()
    V, Cc = meshes[0][0].shape[0], 48
    devs = [Dev(L, m) for L, m in meshes]
    t = _times(Cc, "edges")
    rs = np.random.RandomState(18)
    x, g = rs.randn(2, V, Cc).astype(np.float32), rs.randn(2, V, Cc).astype(np.float32)
    ltd = dn.LearnedTimeDiffusion(Cc, method="implicit_dense").cuda()
    with torch.no_grad():
        ltd.diffusion_time.copy_(torch.from_numpy(t))
    xt = torch.from_numpy(x).cuda().requires_grad_(True)
    y = ltd(xt, torch.stack([d.Lt for d in devs]), torch.stack([d.mass for d in devs]), None, None)
    (y * torch.from_numpy(g).cuda()).sum().backward()
    gt_sum = 0.0
    for b, (L, m) in enumerate(meshes):
        gy, ggx, ggt = OI.implicit_diffusion(x[b], m, L, t, grad_out=g[b])
        _close(y[b].detach().cpu().numpy(), gy)
        _close(xt.grad[b].cpu().numpy(), ggx)
        gt_sum = gt_sum + ggt
    _close(ltd.diffusion_time.grad.cpu().numpy(), gt_sum)


# ---------------------------------------------------------------------------------------------------------------
# 6. the implicit net at tensor-core widths, and on a stack of two meshes, against fp64 autograd
# ---------------------------------------------------------------------------------------------------------------
class _Implicit64(torch.autograd.Function):
    """fp64 implicit diffusion of one mesh for the torch oracle's ``diffuse`` hook: the oracle's solve and adjoint.
    The backward appends sum_v |w_c| |(L y_c)| per channel to ``sink``: the size of the time gradient's dot product
    before it cancels."""

    @staticmethod
    def forward(ctx, x, t, m, L, sink):
        y = OI.implicit_diffusion(x[0].numpy(), m, L, t.numpy())
        ctx.save_for_backward(x, t)
        ctx.m, ctx.L, ctx.y, ctx.sink = m, L, y, sink
        return torch.from_numpy(y).unsqueeze(0)

    @staticmethod
    def backward(ctx, g):
        x, t = ctx.saved_tensors
        _, gx, gt = OI.implicit_diffusion(x[0].numpy(), ctx.m, ctx.L, t.numpy(), grad_out=g[0].numpy())
        ctx.sink.append(np.einsum("vc,vc->c", np.abs(gx / ctx.m[:, None]), np.abs(ctx.L @ ctx.y)))
        return torch.from_numpy(gx).unsqueeze(0), torch.from_numpy(gt), None, None, None


def _net_gold(net, masks, meshes, xs, Rs, check_kinks, engine):
    """Sum over meshes of sum(out * R) through the fp64 composition of the oracle with the implicit solve; returns the
    per-mesh outputs, the input gradients, the parameter gradients and, per block, sum_v |w| |L y| over the meshes."""
    D = torch.float64
    prm = {k: v.detach().cpu().to(D).requires_grad_(True) for k, v in net.state_dict().items()}
    NB = len(net.blocks)
    outs, x64s, loss, sinks = [], [], 0.0, {b: [] for b in range(len(net.blocks))}
    for i, ((L, m, gX, gY), x) in enumerate(zip(meshes, xs)):
        x64 = x.detach().cpu().to(D).requires_grad_(True)
        h = torch.addmm(prm["first_lin.bias"], x64, prm["first_lin.weight"].t()).unsqueeze(0)
        m64 = torch.from_numpy(m).unsqueeze(0)
        for b in range(NB):
            bp = {k[len("block_%d." % b):]: v for k, v in prm.items() if k.startswith("block_%d." % b)}
            pre = []
            h = T.block_forward(h, m64, None, None, [gX.cpu().to(D)], [gY.cpu().to(D)], bp,
                                relu_masks=[mk[i] for mk in masks[b]], pre_acts=pre,
                                diffuse=lambda xi, t, b=b: _Implicit64.apply(xi, t, m, L, sinks[b]))
            check_kinks([mk[i] for mk in masks[b]], pre, engine)
        out = torch.addmm(prm["last_lin.bias"], h[0], prm["last_lin.weight"].t())
        loss = loss + (out * Rs[i].cpu().to(D)).sum()
        outs.append(out.detach())
        x64s.append(x64)
    loss.backward()
    return outs, [x.grad for x in x64s], {k: v.grad for k, v in prm.items()}, {b: sum(s) for b, s in sinks.items()}


def _mlp_hidden(out, weight0):
    """Per mesh, in mesh order: the ReLU patterns (hidden > 0) saved by the MLPFn nodes whose first weight is
    ``weight0`` (a stack runs one node per mesh; the meshes' first sources are slices of one tensor, in order)."""
    nodes, seen, stack = [], {}, [out.grad_fn]
    while stack:
        f = stack.pop()
        if f is None or id(f) in seen:
            continue
        seen[id(f)] = f
        if "MLPFn" in type(f).__name__:
            n_src, n_layers = f.meta[0], f.meta[1]
            sv = f.saved_tensors
            if sv[n_src].data_ptr() == weight0.data_ptr():
                h0 = n_src + n_layers
                nodes.append((sv[0].data_ptr(), [(h > 0).cpu() for h in sv[h0:h0 + f.n_hidden]]))
        stack.extend(nf for nf, _ in f.next_functions)
    return [hs for _, hs in sorted(nodes, key=lambda n: n[0])]


def _implicit_net_case(engine, C_width, meshes_np, seed, label):
    import test_gpu_backward as GB
    dn.set_engine(engine)
    chk = GB.Checker("implicit_net/{}/{}".format(label, engine))
    try:
        C_out, NB = 5, 2
        meshes, xs, Rs, Ls, ms, gXs, gYs = [], [], [], [], [], [], []
        for verts, faces in meshes_np:
            _, mass, Lt, _, _, gX, gY = dn.geometry.compute_operators(verts, faces, 16, device="cuda")
            Lc = Lt.coalesce()
            idx = Lc.indices().cpu().numpy()
            L = sp.csr_matrix((Lc.values().cpu().numpy().astype(np.float64), (idx[0], idx[1])), shape=Lt.shape)
            meshes.append((L, mass.cpu().numpy().astype(np.float64), gX, gY))
            xs.append(verts.cuda())
            Ls.append(Lt), ms.append(mass), gXs.append(gX), gYs.append(gY)
            Rs.append(torch.randn(verts.shape[0], C_out, generator=torch.Generator().manual_seed(seed + len(Rs))))
        torch.manual_seed(seed)
        net = dn.DiffusionNet(C_in=3, C_out=C_out, C_width=C_width, N_block=NB, dropout=False,
                              diffusion_method="implicit_dense").cuda().train()
        with torch.no_grad():
            for n_, p_ in net.named_parameters():
                if n_.endswith("diffusion_time"):
                    p_.uniform_(1e-3, 0.3)
        stack = len(meshes) > 1
        if stack:
            kw = dict(L=torch.stack(Ls), gradX=torch.stack(gXs), gradY=torch.stack(gYs))
            x_in, mass_in = torch.stack(xs).requires_grad_(True), torch.stack(ms)
        else:
            kw = dict(L=Ls[0], gradX=gXs[0], gradY=gYs[0])
            x_in, mass_in = xs[0].clone().requires_grad_(True), ms[0]
        with torch.no_grad():                           # inference: the composed no-grad path
            y0 = net(x_in, mass_in, **kw)
        out = net(x_in, mass_in, **kw)
        # masks[b][layer][mesh]: our ReLU pattern, from each mesh's MLPFn node (meshes in the order of their sources)
        masks = {b: [list(hs) for hs in zip(*_mlp_hidden(out, net.blocks[b].mlp.linears()[0].weight))]
                 for b in range(NB)}
        assert all(len(masks[b][0]) == len(meshes) for b in range(NB))
        R = torch.stack(Rs) if stack else Rs[0]
        (out * R.cuda()).sum().backward()
        gold, gold_gx, gold_gp, dots = _net_gold(net, masks, meshes, xs, Rs, GB._check_kinks, engine)
        tol = GB.TOL[engine]
        outs = list(out) if stack else [out]
        outs0 = list(y0) if stack else [y0]
        gxs = list(x_in.grad) if stack else [x_in.grad]
        for i in range(len(meshes)):
            chk("out[{}] no_grad".format(i), outs0[i], gold[i], tol[0])
            chk("out[{}]".format(i), outs[i], gold[i], tol[0])
            chk("grad_x[{}]".format(i), gxs[i], gold_gx[i], tol[1])
        for name, p_ in net.named_parameters():
            if not name.endswith("diffusion.diffusion_time"):
                chk("grad " + name, p_.grad, gold_gp[name], tol[2])
                continue
            # grad t_c = -sum_v w (L y) cancels: its fp32 floor is the upstream gradient's error (the input-gradient
            # bound) carried through the dot product's absolute size, on top of the parameter-gradient bound
            gold_t = gold_gp[name].numpy()
            err = np.abs(p_.grad.cpu().double().numpy() - gold_t)
            bound = tol[2] * np.abs(gold_t).max() + tol[1] * dots[int(name.split(".")[0].split("_")[1])]
            print("[measured] {} grad {} err/max|gold|={:.3e} err/bound={:.3e}".format(
                chk.label, name, err.max() / np.abs(gold_t).max(), (err / bound).max()))
            if not np.all(err <= bound):
                chk.misses.append("{}: err / bound {:.3g}".format(name, (err / bound).max()))
    finally:
        dn.set_engine("tc3x")
    chk.done()


@gpu
@pytest.mark.parametrize("engine", ["simt", "tc3x"])
@pytest.mark.parametrize("C_width", [64, 128])
def test_implicit_net_at_tensor_core_widths(cuda, engine, C_width):
    verts, faces = dn.synthetic.torus_mesh(30, 50, seed=6)
    _implicit_net_case(engine, C_width, [(verts, faces)], seed=C_width, label="c{}".format(C_width))


@gpu
@pytest.mark.parametrize("engine", ["simt", "tc3x"])
def test_implicit_net_on_a_stack_of_two_meshes(cuda, engine):
    meshes = [dn.synthetic.torus_mesh(30, 40, seed=1), dn.synthetic.torus_mesh(30, 40, seed=9)]
    _implicit_net_case(engine, 64, meshes, seed=5, label="stack2")


# ---------------------------------------------------------------------------------------------------------------
# 7. the bounds are sharp enough (CPU)
# ---------------------------------------------------------------------------------------------------------------
def _pcg(L, m, t, b, rtol):
    """Jacobi-PCG of one column in fp64, stopped at ||r|| <= rtol ||b|| (the kernel's recurrence, on the CPU)."""
    A = sp.diags(m) + t * L
    d = m + t * L.diagonal()
    x = np.zeros_like(b)
    r = b.copy()
    z = r / d
    p = z.copy()
    rz = r @ z
    while np.linalg.norm(r) > rtol * np.linalg.norm(b):
        q = A @ p
        a = rz / (p @ q)
        x += a * p
        r -= a * q
        z = r / d
        rz, rz_old = r @ z, rz
        p = z + rz / rz_old * p
    return x


# errors that stay below 100x the bound on every case, with their measured factor (worst perturbation / bound).  CG
# stopped at rtol = 1e-5 leaves a residual of at most 1e-5 ||b||, while the bound's fp32 store term alone is
# u || |A| |y| || >= u ||b||: no case can show it more than about 1e-5 / (2 rtol + u) = 125x
SENSITIVITY_EXCEPTIONS = {"rtol 1e-5": 92.7}


def test_bounds_reject_structural_errors():
    factors = {}
    for mesh, Cc in (("patch80", 32), ("torus1200", 48)):
        L, m = _mesh(mesh)
        x, _ = _data(L.shape[0], Cc, seed=3)
        t = _times(Cc, "edges")
        gold = Gold(L, m, x, t, lam=True)
        tc = _tc(t)

        # the gold rounded to fp32 is inside both bounds
        y32 = gold.y.astype(np.float32).astype(np.float64)
        res0, rb0, eb0 = gold.error_bound(gold.b, y32, gold.y)
        assert np.all(res0 <= rb0) and np.all(np.abs(y32 - gold.y).max(0) <= eb0)

        def factor(name, y_bad):
            res, rb = residual_bound(L, m, t, gold.b, np.asarray(y_bad, dtype=np.float32).astype(np.float64))
            factors[name] = max(factors.get(name, 0.0), float(np.max(res / rb)))

        # one column solved with its neighbour's time
        c = int(np.argmax(np.abs(np.diff(tc))))
        y = gold.y.copy()
        y[:, c] = sla.spsolve((sp.diags(m) + tc[c + 1] * L).tocsc(), gold.b[:, c])
        factor("neighbour's time", y)
        # one row's last L entry dropped (a rowptr off-by-one)
        Ld = L.copy()
        v = int(np.argmax(np.diff(L.indptr)))
        Ld.data[L.indptr[v + 1] - 1] = 0.0
        factor("row's last entry dropped", np.stack([sla.spsolve((sp.diags(m) + tc[k] * Ld).tocsc(), gold.b[:, k])
                                                     for k in range(Cc)], 1))
        # CG stopped at rtol = 1e-5
        factor("rtol 1e-5", np.stack([_pcg(L, m, tc[k], gold.b[:, k], 1e-5) for k in range(Cc)], 1))
        # b = x instead of M x
        factor("b = x", OI.implicit_diffusion(x / m[:, None], m, L, t))              # A^-1 x
    print("MEASURED sensitivity factors", {k: "{:.3g}".format(v) for k, v in factors.items()})
    for name, f in factors.items():
        if name in SENSITIVITY_EXCEPTIONS:
            assert f >= 0.5 * SENSITIVITY_EXCEPTIONS[name], (name, f)
        else:
            assert f >= 100.0, "{}: only {:.3g} x the bound".format(name, f)
