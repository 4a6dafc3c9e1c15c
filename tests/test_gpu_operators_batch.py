"""Operators of a whole list of small meshes in one launch sequence (geometry.compute_operators_batch, the batched
Laplacian and eigensolver kernels, get_all_operators(batch_misses=True)): every mesh against the fp64 numpy / scipy
oracle (oracle/dn_oracle_ops.py) with the per-mesh route's tolerances, bitwise against compute_operators where the two
run the same arithmetic, and the dn_eig_*_batched kernels against numpy fp64 on ragged batches.

Eigenvectors are compared through the projector onto the leading k' <= k of them, k' ending at a relative spectral gap
>= 1e-3 of the oracle's spectrum, as in test_gpu_operators.py."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle as O  # noqa: E402  (checker only)
import dn_oracle_ops as OO  # noqa: E402

import diffusion_net_b200 as dn  # noqa: E402
import diffusion_net_b200.eigen  # noqa: E402,F401  (dn.eigen: not imported at package level)

gpu = pytest.mark.gpu
S = dn.synthetic

# ragged V from 140 to 6000; one mesh narrower than the block (k < V < k + guard) and open patches (the poorly
# conditioned boundary case) in each list
BATCHES = {
    128: [lambda: S.torus_mesh(36, 50, seed=0), lambda: S.patch_mesh(20, 17, seed=1), lambda: S.icosphere_mesh(4, seed=2),
          lambda: S.torus_mesh(10, 14, seed=3), lambda: S.patch_mesh(55, 55, seed=3), lambda: S.icosphere_mesh(3, seed=5),
          lambda: S.torus_mesh(60, 100, seed=6), lambda: S.torus_mesh(41, 50, seed=7)],
    32: [lambda: S.torus_mesh(12, 16, seed=0), lambda: S.patch_mesh(6, 7, seed=1), lambda: S.icosphere_mesh(3, seed=2),
         lambda: S.patch_mesh(31, 23, seed=3), lambda: S.torus_mesh(36, 50, seed=4), lambda: S.icosphere_mesh(2, seed=5),
         lambda: S.torus_mesh(23, 29, seed=6), lambda: S.patch_mesh(12, 14, seed=4), lambda: S.torus_mesh(40, 50, seed=1)],
}


def _kprime(evals, k, rel_gap=1e-3):
    """Largest k' <= k such that evals[k'] - evals[k'-1] >= rel_gap * evals[k'] (evals holds more than k values)."""
    for kp in range(k, 0, -1):
        if evals[kp] - evals[kp - 1] >= rel_gap * abs(evals[kp]):
            return kp
    return 0


def _projector_err(phi_a, phi_b, mass):
    """max|P_a - P_b| / max|P_b| with P = Phi Phi^T M, explicit for V <= 4k; larger, applied to 16 seeded random
    vectors."""
    if phi_a.shape[0] <= 4096:
        Pa, Pb = (p @ (p.T * mass[None, :]) for p in (phi_a, phi_b))
        return O.rel_err(Pa, Pb)
    X = np.random.RandomState(0).randn(phi_a.shape[0], 16) * mass[:, None]
    return O.rel_err(phi_a @ (phi_a.T @ X), phi_b @ (phi_b.T @ X))


def _np(t):
    return t.detach().cpu().numpy()


def _coo_np(t):
    t = t.coalesce()
    i = _np(t.indices())
    return sp.csr_matrix((_np(t.values()).astype(np.float64), (i[0], i[1])), shape=tuple(t.shape))


def _check_against(out, gold, k, gold_evals_ext):
    """The checks of test_compute_operators_against_oracle: L pattern + values, mass, frames, evals, projector over
    k', M-orthonormality, gradX / gradY; same tolerances."""
    frames, mass, L, evals, evecs, gx, gy = out
    g_frames, g_mass, g_L, g_evals, g_evecs, g_gx, g_gy = gold
    Lm, gL = _coo_np(L), sp.csr_matrix(g_L)
    assert np.array_equal(Lm.indptr, gL.indptr) and np.array_equal(Lm.indices, gL.indices)
    assert abs(Lm - gL).max() <= 1e-6 * abs(gL).max()
    m = _np(mass).astype(np.float64)
    assert np.abs(m - g_mass).max() <= 1e-6 * np.abs(g_mass).max()
    assert O.rel_err(_np(frames), g_frames) <= 1e-6
    ev = _np(evals).astype(np.float64)
    assert np.all(np.diff(ev) >= 0)
    assert np.abs(ev - g_evals[:k]).max() <= 1e-5 * g_evals[k - 1]
    kp = _kprime(gold_evals_ext, k)
    assert kp > 0
    phi = _np(evecs).astype(np.float64)
    assert _projector_err(phi[:, :kp], g_evecs[:, :kp], g_mass) <= 1e-5
    assert np.abs(phi.T @ (phi * m[:, None]) - np.eye(k)).max() <= 1e-5
    for mine, g in ((gx, g_gx), (gy, g_gy)):
        M, G = _coo_np(mine), sp.csr_matrix(g)
        assert np.array_equal(M.indptr, G.indptr) and np.array_equal(M.indices, G.indices)
        assert abs(M - G).max() <= 1e-5 * abs(G).max()
    return kp


def _same(a, b):
    if a.is_sparse:
        return torch.equal(a.indices(), b.indices()) and torch.equal(a.values(), b.values())
    return torch.equal(a, b)


BITWISE = (0, 1, 2, 5, 6)       # frames, mass, L, gradX, gradY: the same arithmetic whatever the batch


def _same_operators(a, b):
    """Two results for one mesh from different batches: bitwise but for the eigenpairs, which share the batch's filter
    degree and so agree to the solver's tolerance (here: to fp32 rounding of the returned values)."""
    ea, eb = _np(a[3]).astype(np.float64), _np(b[3]).astype(np.float64)
    return all(_same(a[i], b[i]) for i in BITWISE) and np.abs(ea - eb).max() <= 1e-6 * eb[-1]


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    dn._lib.load()
    return torch.device("cuda")


_cache = {}


def _case(cuda, k):
    """meshes, oracle golds (with one eigenvalue more), the batched result and the per-mesh results of BATCHES[k]"""
    if k not in _cache:
        meshes = [make() for make in BATCHES[k]]
        golds = []
        for v, f in meshes:
            g = OO.compute_operators(v.numpy(), f.numpy(), k + 1)
            golds.append(((g[0].astype(np.float64), g[1], g[2], g[3][:k], g[4][:, :k], g[5], g[6]), g[3]))
        st = {}
        batched = dn.geometry.compute_operators_batch([v for v, _ in meshes], [f for _, f in meshes], k, device=cuda,
                                                      stats=st)
        single = [dn.geometry.compute_operators(v, f, k, device=cuda) for v, f in meshes]
        _cache[k] = (meshes, golds, batched, single, st)
    return _cache[k]


# ---------------------------------------------------------------------------------------------------------------
# host
# ---------------------------------------------------------------------------------------------------------------
def test_batch_groups_keep_order_and_respect_max_rows():
    groups = dn.geometry.batch_groups
    assert groups([], 100) == []
    assert groups([5, 5, 5], 100) == [(0, 3)]
    assert groups([60, 50, 40, 70, 10], 100) == [(0, 1), (1, 3), (3, 5)]
    assert groups([300, 20, 30], 100) == [(0, 1), (1, 3)]            # a mesh above the cap is a group of its own
    assert groups([20, 300, 30], 100) == [(0, 1), (1, 2), (2, 3)]
    rng = np.random.RandomState(0)
    Vs = list(rng.randint(1, 500, size=200))
    g = groups(Vs, 1000)
    assert [i for a, b in g for i in range(a, b)] == list(range(200))
    assert all(sum(Vs[a:b]) <= 1000 or b - a == 1 for a, b in g)
    assert all(sum(Vs[a:b + 1]) > 1000 for a, b in g[:-1])          # greedy: the next mesh did not fit


def test_batch_plan_matches_the_header_constants():
    hdr = open(os.path.join(ROOT, "include", "diffusion_net_b200.h")).read()
    assert int(re.search(r"#define DN_EIG_TILE_ROWS (\d+)", hdr).group(1)) == dn.eigen.TILE_ROWS
    assert int(re.search(r"#define DN_EIG_SLICE_ROWS (\d+)", hdr).group(1)) == dn.eigen.SLICE_ROWS


# ---------------------------------------------------------------------------------------------------------------
# 1, 2: every mesh against fp64 truth, and against compute_operators on that mesh alone
# ---------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("k", sorted(BATCHES))
def test_every_mesh_of_a_batch_against_oracle(cuda, k):
    meshes, golds, batched, single, st = _case(cuda, k)
    assert len(batched) == len(meshes)
    B = k + max(16, k // 4)
    assert st["eig"][0]["n_stacked"] == sum(v.shape[0] >= B for v, _ in meshes) < len(meshes)
    for out, (gold, ext) in zip(batched, golds):
        assert all(t.device.type == "cuda" and t.dtype == torch.float32 for t in out)
        _check_against(out, gold, k, ext)


@gpu
@pytest.mark.parametrize("k", sorted(BATCHES))
def test_batched_equals_per_mesh_where_it_must(cuda, k):
    meshes, golds, batched, single, _ = _case(cuda, k)
    for b, (out, one, (gold, ext)) in enumerate(zip(batched, single, golds)):
        for i in BITWISE:
            assert _same(out[i], one[i]), (b, i)
        # evals / evecs come from two different iterations; compared in fp64 (fp32 would hide the solver's tolerance)
    v64 = [(v.double(), f) for v, f in meshes]
    b64 = dn.geometry.compute_operators_batch([v for v, _ in v64], [f for _, f in v64], k, device=cuda)
    for (v, f), out, (gold, ext) in zip(v64, b64, golds):
        assert all(t.dtype == torch.float64 for t in out)
        one = dn.geometry.compute_operators(v, f, k, device=cuda)
        ea, eb = _np(out[3]), _np(one[3])
        assert np.abs(ea - eb).max() <= 1e-8 * eb[-1]
        kp = _kprime(ext, k)
        assert _projector_err(_np(out[4])[:, :kp], _np(one[4])[:, :kp], _np(one[1])) <= 1e-5
    # the prepared CSR registered against gradX / gradY drives the layers without a conversion
    gx, gy = batched[0][5], batched[0][6]
    assert (id(gx), id(gy)) in dn.ops._prep_cache


# ---------------------------------------------------------------------------------------------------------------
# 3: composition independence and determinism
# ---------------------------------------------------------------------------------------------------------------
@gpu
def test_result_does_not_depend_on_the_batch_and_is_deterministic(cuda):
    k = 32
    meshes, golds, batched, _, _ = _case(cuda, k)
    order = [6, 2, 4, 0]                                # other neighbours, other positions
    vl, fl = [meshes[i][0] for i in order], [meshes[i][1] for i in order]
    a = dn.geometry.compute_operators_batch(vl, fl, k, device=cuda)
    b = dn.geometry.compute_operators_batch(vl, fl, k, device=cuda)
    for j, i in enumerate(order):
        _check_against(a[j], golds[i][0], k, golds[i][1])
        assert all(_same(x, y) for x, y in zip(a[j], b[j]))        # the same batch twice: bitwise
        assert _same_operators(a[j], batched[i])


# ---------------------------------------------------------------------------------------------------------------
# 4: the batched kernels against numpy fp64
# ---------------------------------------------------------------------------------------------------------------
def _plan(Vs, cuda):
    return dn.eigen.BatchPlan(Vs, cuda)


RAGGED = [37, 1031, 64, 200, 2500, 7]                   # none a multiple of a tile but 64; 2500 spans three slices


@gpu
def test_batched_gram_rotate_residuals_against_numpy(cuda):
    lib = dn._lib.load()
    plan = _plan(RAGGED, cuda)
    rb, n, V = plan.row_begin, plan.n, plan.V
    m_, n_, ld = 70, 45, 80
    g = torch.Generator().manual_seed(0)
    X = torch.randn(V, ld, generator=g, dtype=torch.float64)
    Y = torch.randn(V, ld, generator=g, dtype=torch.float64)
    Xd, Yd = X.to(cuda), Y.to(cuda)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    active = torch.tensor([1, 1, 0, 1, 1, 1], dtype=torch.int32, device=cuda)
    ws = torch.empty(8 * plan.n_slices * m_ * n_, dtype=torch.uint8, device=cuda)
    out = torch.full((n, m_, n_), -7.0, dtype=torch.float64, device=cuda)
    gram = lambda: dn._lib.check(lib.dn_eig_gram_batched(Xd.data_ptr(), ld, Yd.data_ptr(), ld, C.byref(plan.struct), m_, n_,
                                                         active.data_ptr(), out.data_ptr(), ws.data_ptr(), ws.numel(), st),
                                 "gram")
    gram()
    first = out.clone()
    gram()
    assert torch.equal(out, first)
    for b in range(n):
        want = X[rb[b]:rb[b + 1], :m_].numpy().T @ Y[rb[b]:rb[b + 1], :n_].numpy()
        if b == 2:
            assert bool((out[b] == -7.0).all())
        else:
            assert np.abs(_np(out[b]) - want).max() <= 1e-13 * np.sqrt(RAGGED[b]) * max(np.abs(want).max(), 1.0)
    # a mesh alone gives the bits it gives inside the batch
    solo = _plan([RAGGED[4]], cuda)
    xs, ys = Xd[rb[4]:rb[5]].contiguous(), Yd[rb[4]:rb[5]].contiguous()
    o1 = torch.empty(1, m_, n_, dtype=torch.float64, device=cuda)
    dn._lib.check(lib.dn_eig_gram_batched(xs.data_ptr(), ld, ys.data_ptr(), ld, C.byref(solo.struct), m_, n_, None,
                                          o1.data_ptr(), ws.data_ptr(), ws.numel(), st), "gram")
    assert torch.equal(o1[0], out[4])
    # rotate: Z_b = beta Z_b + X_b C_b
    kd = 70
    Cm = torch.randn(n, kd, n_, generator=g, dtype=torch.float64)
    Z0 = torch.randn(V, ld, generator=g, dtype=torch.float64)
    for beta in (0.0, 1.0):
        Z = Z0.clone().to(cuda)
        dn._lib.check(lib.dn_eig_rotate_batched(Xd.data_ptr(), ld, Cm.to(cuda).data_ptr(), C.byref(plan.struct), kd, n_,
                                                beta, active.data_ptr(), Z.data_ptr(), ld, st), "rotate")
        Z = Z.cpu()
        assert torch.equal(Z[:, n_:], Z0[:, n_:])
        for b in range(n):
            r = slice(rb[b], rb[b + 1])
            if b == 2:
                assert torch.equal(Z[r], Z0[r])
                continue
            want = beta * Z0[r, :n_].numpy() + X[r, :kd].numpy() @ Cm[b].numpy()
            assert np.abs(Z[r, :n_].numpy() - want).max() <= 1e-13 * kd
    # residual norms with each mesh's own theta
    theta = torch.randn(n, n_, generator=g, dtype=torch.float64)
    res = torch.full((n, n_), -7.0, dtype=torch.float64, device=cuda)
    dn._lib.check(lib.dn_eig_residual_norms_batched(Xd.data_ptr(), ld, Yd.data_ptr(), ld, theta.to(cuda).data_ptr(),
                                                    C.byref(plan.struct), n_, active.data_ptr(), res.data_ptr(),
                                                    ws.data_ptr(), ws.numel(), st), "residual_norms")
    for b in range(n):
        r = slice(rb[b], rb[b + 1])
        want = np.linalg.norm(X[r, :n_].numpy() - theta[b].numpy()[None, :] * Y[r, :n_].numpy(), axis=0)
        if b == 2:
            assert bool((res[b] == -7.0).all())
        else:
            assert np.abs(_np(res[b]) - want).max() <= 1e-13 * want.max()


@gpu
def test_batched_filter_and_finalize_against_numpy(cuda):
    lib = dn._lib.load()
    k = 8
    meshes = [S.torus_mesh(7, 9, seed=0), S.patch_mesh(9, 11, seed=1), S.icosphere_mesh(2, seed=2), S.torus_mesh(13, 17, seed=3)]
    Vs = [int(v.shape[0]) for v, _ in meshes]           # 63, 99, 162, 221: mesh boundaries inside 8-row CTAs and tiles
    plan = _plan(Vs, cuda)
    rb, n, V = plan.row_begin, plan.n, plan.V
    lops = []
    for v, f in meshes:
        rowptr, colidx, lvals, mass, avals, adiag, bound = dn.geometry.mesh_laplacian(v.double().to(cuda), f.to(cuda))
        lops.append(dn.eigen.LaplaceOperator(int(v.shape[0]), rowptr, colidx, avals, adiag, mass, bound))
    s = dn.eigen._BatchSolver(lops, k, 40, 0)
    g = torch.Generator().manual_seed(1)
    Y, Yp = (torch.randn(V, 40, generator=g, dtype=torch.float64) for _ in range(2))
    coef = torch.randn(3, n, generator=g, dtype=torch.float64)
    s.set_active([1, 0, 1, 1])
    out = torch.full((V, 40), -7.0, dtype=torch.float64, device=cuda)
    s.filt(Y.to(cuda), Yp.to(cuda), out, coef.to(cuda))
    out = out.cpu()
    for b, op in enumerate(lops):
        r = slice(rb[b], rb[b + 1])
        if b == 1:
            assert bool((out[r] == -7.0).all())         # an inactive mesh's rows are not written
            continue
        A = sp.csr_matrix((_np(op.avals), _np(op.colidx), _np(op.rowptr)), shape=(op.V, op.V)) + sp.diags(_np(op.adiag))
        want = coef[0, b].item() * (A @ Y[r].numpy()) + coef[1, b].item() * Y[r].numpy() + coef[2, b].item() * Yp[r].numpy()
        assert np.abs(out[r].numpy() - want).max() <= 1e-13 * np.abs(want).max()
    # finalize: phi = M^-1/2 y of each mesh's own columns, largest-magnitude entry positive
    cols = torch.stack([torch.randperm(40, generator=g)[:k] for _ in range(n)]).to(torch.int32)
    ev = torch.empty(V, k, dtype=torch.float64, device=cuda)
    Yd = Y.to(cuda)
    dn._lib.check(lib.dn_eig_finalize_batched(Yd.data_ptr(), 40, cols.to(cuda).data_ptr(), k, s.mass.data_ptr(), s.bt,
                                              ev.data_ptr(), s.ws.data_ptr(), s.ws.numel(),
                                              C.c_void_p(torch.cuda.current_stream().cuda_stream)), "finalize")
    for b, op in enumerate(lops):
        r = slice(rb[b], rb[b + 1])
        phi = Y[r].numpy()[:, cols[b].numpy()] / np.sqrt(_np(op.mass))[:, None]
        top = np.abs(phi).argmax(axis=0)
        phi = phi * np.where(phi[top, np.arange(k)] < 0, -1.0, 1.0)[None, :]
        assert np.array_equal(_np(ev[r]), phi)


# ---------------------------------------------------------------------------------------------------------------
# 5: errors name the mesh; groups
# ---------------------------------------------------------------------------------------------------------------
@gpu
def test_errors_name_the_mesh_and_groups_do_not_change_results(cuda):
    k = 32
    meshes, _, batched, _, _ = _case(cuda, k)
    vl, fl = [v for v, _ in meshes], [f for _, f in meshes]
    tiny = S.patch_mesh(5, 6, seed=0)                   # V = 30 <= k
    with pytest.raises(ValueError, match=r"^mesh 2: failed to compute eigendecomp: k_eig = 32 is not below"):
        dn.geometry.compute_operators_batch(vl[:2] + [tiny[0]] + vl[2:], fl[:2] + [tiny[1]] + fl[2:], k, device=cuda)
    bad = vl[3].clone()
    bad[5, 0] = float("nan")
    with pytest.raises(RuntimeError, match=r"^mesh 3: NaN Laplace matrix"):
        dn.geometry.compute_operators_batch(vl[:3] + [bad] + vl[4:], fl, k, device=cuda)
    with pytest.raises(RuntimeError, match=r"^mesh 7: NaN"):    # ... counted in the caller's list, not in the group
        dn.geometry.compute_operators_batch(vl[:7] + [bad] + vl[8:], fl[:7] + [fl[3]] + fl[8:], k, device=cuda, max_rows=2500)
    off = fl[1].clone()
    off[0, 0] = vl[1].shape[0]
    with pytest.raises(ValueError, match=r"^mesh 1: faces index vertices outside"):
        dn.geometry.compute_operators_batch(vl, [fl[0], off] + fl[2:], k, device=cuda)
    with pytest.raises(NotImplementedError, match=r"^mesh 1: point clouds"):
        dn.geometry.compute_operators_batch(vl[:2], [fl[0], torch.zeros(0, 3, dtype=torch.int64)], k, device=cuda)
    with pytest.raises(RuntimeError, match="CUDA devices only"):
        dn.geometry.compute_operators_batch(vl[:2], fl[:2], k)
    st = {}
    grouped = dn.geometry.compute_operators_batch(vl, fl, k, device=cuda, max_rows=2500, stats=st)
    assert st["groups"] >= 3
    for a, b in zip(grouped, batched):
        assert _same_operators(a, b)
    # caller-supplied normals for some meshes only
    nrm = torch.zeros(vl[1].shape[0], 3)
    nrm[:, 1] = 1.0
    fr = dn.geometry.compute_operators_batch(vl[:3], fl[:3], 8, normals=[None, nrm, None], device=cuda)
    assert torch.equal(fr[1][0], dn.geometry.compute_operators(vl[1], fl[1], 8, normals=nrm, device=cuda)[0])
    assert torch.equal(fr[2][0], batched[2][0])


# ---------------------------------------------------------------------------------------------------------------
# 6: the cache
# ---------------------------------------------------------------------------------------------------------------
@gpu
def test_get_all_operators_batches_the_misses(cuda, tmp_path):
    k = 32
    meshes, _, batched, single, _ = _case(cuda, k)
    sel = [0, 2, 3, 5, 7]
    vl, fl = [meshes[i][0] for i in sel], [meshes[i][1] for i in sel]
    cache = str(tmp_path / "cache")
    geo = dn.geometry
    for j in (1, 3):                                    # two entries are there already, written by the per-mesh route
        geo.get_operators(vl[j], fl[j], k, cache, device=cuda, compute_missing=True)
    planted = {j: geo.find_cache_bucket(vl[j], fl[j], cache) for j in (1, 3)}
    for p in planted.values():
        t0 = os.path.getmtime(p)
        os.utime(p, (t0 - 100, t0 - 100))
    stamp = {j: os.path.getmtime(p) for j, p in planted.items()}
    first = geo.get_all_operators(vl, fl, k, cache, device=cuda, compute_missing=True, batch_misses=True)
    assert {j: os.path.getmtime(p) for j, p in planted.items()} == stamp          # hits are not recomputed
    want = sorted(os.path.basename(geo.find_cache_bucket(v, f, cache)) for v, f in zip(vl, fl))
    assert sorted(os.listdir(cache)) == want and len(set(want)) == len(sel)
    for j, i in enumerate(sel):                         # input order; misses are the batched route's tensors
        if j not in planted:
            assert _same_operators(tuple(first[t][j] for t in range(7)), batched[i])
    stamp = {f: os.path.getmtime(os.path.join(cache, f)) for f in os.listdir(cache)}
    second = geo.get_all_operators(vl, fl, k, cache, device=cuda, compute_missing=True, batch_misses=True)
    assert {f: os.path.getmtime(os.path.join(cache, f)) for f in os.listdir(cache)} == stamp     # all hits
    for t in range(7):
        for a, b in zip(first[t], second[t]):
            if a.is_sparse:
                assert torch.equal(a.coalesce().indices(), b.coalesce().indices())
                assert torch.equal(a.coalesce().values(), b.coalesce().values())
            else:
                assert torch.equal(a, b)
    # one written entry through the reader drives the net like the returned tuple
    j = 0
    loaded = geo.load_operators_npz(geo.find_cache_bucket(vl[j], fl[j], cache), device=cuda)
    torch.manual_seed(3)
    net = dn.DiffusionNet(C_in=3, C_out=4, C_width=32, N_block=2, dropout=False).to(cuda).eval()
    x = torch.randn(vl[j].shape[0], 3, generator=torch.Generator().manual_seed(1)).to(cuda)
    ys = []
    with torch.no_grad():
        for fr, mass, L, evals, evecs, gx, gy in (loaded, tuple(first[t][j] for t in range(7))):
            ys.append(net(x, mass, L=L, evals=evals, evecs=evecs, gradX=gx, gradY=gy))
    assert torch.equal(ys[0], ys[1])
    # without compute_missing a miss still raises; the default route is the per-mesh loop
    with pytest.raises(NotImplementedError):
        geo.get_all_operators([meshes[1][0]], [meshes[1][1]], k, cache, device=cuda, batch_misses=True)


# ---------------------------------------------------------------------------------------------------------------
# 7: straight into MeshBatch + forward_batch
# ---------------------------------------------------------------------------------------------------------------
@gpu
def test_batched_operators_drive_forward_batch(cuda):
    k = 128
    meshes, golds, batched, single, _ = _case(cuda, k)
    # a truncation (a multiple of 16, the fused batch kernels' K) that ends at a spectral gap of at least three meshes
    # wider than the block: there the net's output does not depend on the basis chosen inside a cluster
    wide = [i for i, (v, _) in enumerate(meshes) if v.shape[0] >= 160]
    kp, sel = next((kk, [i for i in wide if _kprime(golds[i][1][:kk + 1], kk) == kk]) for kk in range(112, 0, -16)
                   if sum(_kprime(golds[i][1][:kk + 1], kk) == kk for i in wide) >= 3)
    torch.manual_seed(3)
    net = dn.DiffusionNet(C_in=16, C_out=4, C_width=64, N_block=2, dropout=False)
    g = torch.Generator().manual_seed(9)
    with torch.no_grad():
        for name, prm in net.named_parameters():
            if name.endswith("diffusion_time"):
                prm.copy_(1e-3 + 0.05 * torch.rand(prm.shape, generator=g))
    params = {key: _np(v).astype(np.float64) for key, v in net.state_dict().items()}
    net = net.to(cuda).eval()
    xs = [torch.randn(meshes[i][0].shape[0], 16, generator=torch.Generator().manual_seed(i)) for i in sel]
    outs = {}
    engine = dn.get_engine()
    dn.set_engine("tc3x")
    try:
        for name, src in (("batched", batched), ("single", single)):
            items = [dict(mass=src[i][1], evals=src[i][3][:kp].contiguous(), evecs=src[i][4][:, :kp].contiguous(),
                          gradX=src[i][5], gradY=src[i][6]) for i in sel]
            with torch.no_grad():
                outs[name] = net.forward_batch(dn.MeshBatch(items), [x.to(cuda) for x in xs])
    finally:
        dn.set_engine(engine)
    for j, i in enumerate(sel):
        gd = golds[i][0]
        want = O.diffusion_net(xs[j].numpy().astype(np.float64), gd[1], gd[3][:kp], gd[4][:, :kp], sp.csr_matrix(gd[5]),
                               sp.csr_matrix(gd[6]), params, 2)
        assert O.rel_err(_np(outs["batched"][j]), want) <= 1e-5
        assert O.rel_err(_np(outs["batched"][j]), _np(outs["single"][j])) <= 1e-5
