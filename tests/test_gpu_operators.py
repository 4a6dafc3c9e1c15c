"""Operator construction on the GPU (geometry.compute_operators: frames, cotan Laplacian, mass, the Chebyshev-filtered
eigensolver, build_grad) against the cache entries the live reference wrote (tests/golden/op_cache*/) and against the
numpy/scipy oracle (oracle/dn_oracle_ops.py, the reference's exact eigsh call) at user sizes.

Eigenvectors are compared through the projector onto the leading k' <= k of them, k' ending at a relative spectral gap
>= 1e-3 of the oracle's spectrum: inside a (near-)degenerate cluster single eigenvectors are not comparable between
two solvers.  The oracle pins run on the CPU; everything else needs an H100."""
import glob
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from conftest import GOLDEN, ROOT

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle as O  # noqa: E402  (checker only)
import dn_oracle_ops as OO  # noqa: E402

import diffusion_net_b200 as dn  # noqa: E402

gpu = pytest.mark.gpu
FIXTURES = [(os.path.join(GOLDEN, "op_cache"), 16), (os.path.join(GOLDEN, "op_cache_patch"), 32)]


def _entry(d):
    return np.load(glob.glob(os.path.join(d, "*.npz"))[0], allow_pickle=True)


def _csc(z, p):
    return sp.csc_matrix((z[p + "_data"], z[p + "_indices"], z[p + "_indptr"]), shape=tuple(z[p + "_shape"]))


def _kprime(evals, k, rel_gap=1e-3):
    """Largest k' <= k such that evals[k'] - evals[k'-1] >= rel_gap * evals[k'] (evals holds more than k values)."""
    for kp in range(k, 0, -1):
        if evals[kp] - evals[kp - 1] >= rel_gap * abs(evals[kp]):
            return kp
    return 0


def _projector_err(phi_a, phi_b, mass):
    """max|P_a - P_b| / max|P_b| with P = Phi Phi^T M, explicit for V <= 4k; larger, applied to 16 seeded random
    vectors (the principal-angle sine would be dominated by the fp32 rounding of an M-orthonormal basis)."""
    if phi_a.shape[0] <= 4096:
        Pa, Pb = (p @ (p.T * mass[None, :]) for p in (phi_a, phi_b))
        return O.rel_err(Pa, Pb)
    X = np.random.RandomState(0).randn(phi_a.shape[0], 16) * mass[:, None]
    return O.rel_err(phi_a @ (phi_a.T @ X), phi_b @ (phi_b.T @ X))


# ---------------------------------------------------------------------------------------------------------------
# 1. oracle pin (CPU): the numpy restatement reproduces what the live reference wrote
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fixture", FIXTURES, ids=["torus12x16", "patch"])
def test_oracle_compute_operators_matches_reference_entry(fixture):
    d, k = fixture
    z = _entry(d)
    frames, mass, L, evals, evecs, gx, gy = OO.compute_operators(z["verts"], z["faces"], k)
    Lz = _csc(z, "L")
    assert abs(L - Lz).max() <= 1e-6 * abs(Lz).max()
    assert O.rel_err(mass, z["mass"]) <= 1e-6
    assert O.rel_err(frames, z["frames"]) <= 1e-6
    order = np.argsort(z["evals"], kind="stable")
    assert np.abs(evals - z["evals"][order]).max() <= 1e-5 * evals[-1]
    kp = _kprime(np.concatenate((evals, [np.inf])), k)
    assert _projector_err(evecs[:, :kp], z["evecs"][:, order][:, :kp].astype(np.float64), mass) <= 1e-5
    for mine, p in ((gx, "gradX"), (gy, "gradY")):
        G = _csc(z, p)
        assert abs(mine - G).max() <= 1e-5 * abs(G).max()


# ---------------------------------------------------------------------------------------------------------------
# build checks (CPU): the new kernels compile for sm_90a without spills
# ---------------------------------------------------------------------------------------------------------------
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.mark.skipif(shutil.which(NVCC) is None and not os.path.exists(NVCC), reason="nvcc not found")
@pytest.mark.parametrize("src", ["dn_eig.cu", "dn_geom.cu"])
def test_operator_kernels_do_not_spill(tmp_path, src):
    flags = [f for f in dn._lib.NVCC_FLAGS if f != "-shared"]
    cmd = [NVCC] + flags + ["-Xptxas", "-v", "-c", os.path.join(dn._lib._CSRC, src), "-o", str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [l for l in (r.stdout + r.stderr).splitlines() if "spill stores" in l]
    assert lines
    for l in lines:
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", l)
        assert m and m.group(1) == "0" and m.group(2) == "0", l


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    dn._lib.load()
    return torch.device("cuda")


def _np(t):
    return t.detach().cpu().numpy()


def _coo_np(t):
    t = t.coalesce()
    i = _np(t.indices())
    return sp.csr_matrix((_np(t.values()).astype(np.float64), (i[0], i[1])), shape=tuple(t.shape))


def _check_against(out, gold, k, gold_evals_ext, tol_pattern=True):
    """Section 2 of the checks: L pattern + values, mass, frames, evals, projector over k', gradX / gradY."""
    frames, mass, L, evals, evecs, gx, gy = out
    g_frames, g_mass, g_L, g_evals, g_evecs, g_gx, g_gy = gold
    Lm = _coo_np(L)
    gL = sp.csr_matrix(g_L)
    if tol_pattern:
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
    assert _projector_err(_np(evecs)[:, :kp].astype(np.float64), g_evecs[:, :kp], g_mass) <= 1e-5
    for mine, g in ((gx, g_gx), (gy, g_gy)):
        M, G = _coo_np(mine), sp.csr_matrix(g)
        assert np.array_equal(M.indptr, G.indptr) and np.array_equal(M.indices, G.indices)
        assert abs(M - G).max() <= 1e-5 * abs(G).max()
    return kp


@gpu
@pytest.mark.parametrize("fixture", FIXTURES, ids=["torus12x16", "patch"])
def test_compute_operators_matches_reference_entry(cuda, fixture):
    d, k = fixture
    z = _entry(d)
    verts, faces = torch.from_numpy(z["verts"]), torch.from_numpy(z["faces"])
    out = dn.geometry.compute_operators(verts, faces, k, device=cuda)
    assert all(t.device.type == "cuda" and t.dtype == torch.float32 for t in out)
    order = np.argsort(z["evals"], kind="stable")
    gold = (z["frames"].astype(np.float64), z["mass"].astype(np.float64), _csc(z, "L").astype(np.float64),
            z["evals"][order].astype(np.float64), z["evecs"][:, order].astype(np.float64), _csc(z, "gradX"),
            _csc(z, "gradY"))
    # the gap after the k-th pair comes from the oracle's spectrum one pair further
    ext = OO.compute_operators(z["verts"], z["faces"], k + 1)[3]
    _check_against(out, gold, k, ext)


def _oracle_case(verts, faces, k):
    v, f = verts.numpy(), faces.numpy()
    g = OO.compute_operators(v, f, k + 1)
    return (g[0].astype(np.float64), g[1], g[2], g[3][:k], g[4][:, :k], g[5], g[6]), g[3]


CASES = {
    "torus40x50_k128": (lambda: dn.synthetic.torus_mesh(40, 50, seed=1), 128),
    "icosphere_k64": (lambda: dn.synthetic.icosphere_mesh(4, seed=2), 64),
    "patch3k_k128": (lambda: dn.synthetic.patch_mesh(55, 55, seed=3), 128),
}


@gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_compute_operators_against_oracle(cuda, case):
    make, k = CASES[case]
    verts, faces = make()
    gold, ext = _oracle_case(verts, faces, k)
    out = dn.geometry.compute_operators(verts, faces, k, device=cuda)
    kp = _check_against(out, gold, k, ext)
    frames, mass, L, evals, evecs, gx, gy = out
    m = _np(mass).astype(np.float64)
    phi = _np(evecs).astype(np.float64)
    assert np.abs(phi.T @ (phi * m[:, None]) - np.eye(k)).max() <= 1e-5
    # residuals of the fp64 solution (fp32 rounding of phi alone exceeds the bound on fine meshes)
    out64 = dn.geometry.compute_operators(verts.double(), faces, k, device=cuda)
    phi64, lam64, m64 = _np(out64[4]), _np(out64[3]), _np(out64[1])
    Lg = sp.csr_matrix(gold[2])
    R = Lg @ phi64 + 1e-8 * phi64 - (phi64 * m64[:, None]) * lam64[None, :]
    assert np.all(np.linalg.norm(R, axis=0) <= 1e-5 * lam64[-1] * np.linalg.norm(phi64 * m64[:, None], axis=0))
    # basis-invariant consumers over k'
    hks = _np(dn.geometry.compute_hks_autoscale(evals[:kp].contiguous(), evecs[:, :kp].contiguous(), 16))
    g_hks = O.compute_hks(gold[3][:kp], gold[4][:, :kp], O.hks_autoscale_scales(16, np.float64))
    assert O.rel_err(hks, g_hks) <= 1e-5
    _net_parity(cuda, out, gold, kp)


def _net_parity(cuda, out, gold, kp):
    torch.manual_seed(3)
    net = dn.DiffusionNet(C_in=3, C_out=4, C_width=32, N_block=2, dropout=False)
    g = torch.Generator().manual_seed(9)
    with torch.no_grad():
        for name, prm in net.named_parameters():
            if name.endswith("diffusion_time"):
                prm.copy_(1e-3 + 0.05 * torch.rand(prm.shape, generator=g))
    params = {k: _np(v).astype(np.float64) for k, v in net.state_dict().items()}
    net = net.to(cuda).eval()
    frames, mass, L, evals, evecs, gx, gy = out
    x = torch.randn(mass.shape[0], 3, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        y = net(x.to(cuda), mass, L=L, evals=evals[:kp].contiguous(), evecs=evecs[:, :kp].contiguous(), gradX=gx,
                gradY=gy)
    g = gold
    want = O.diffusion_net(x.numpy().astype(np.float64), g[1], g[3][:kp], g[4][:, :kp], sp.csr_matrix(g[5]),
                           sp.csr_matrix(g[6]), params, 2)
    assert O.rel_err(_np(y), want) <= 1e-5


@gpu
def test_torus_20k_misses_no_eigenvalue(cuda):
    verts, faces = dn.synthetic.torus_mesh(100, 200, seed=0)
    k = 128
    gold, ext = _oracle_case(verts, faces, k)
    out = dn.geometry.compute_operators(verts, faces, k, device=cuda)
    kp = _check_against(out, gold, k, ext)
    assert kp >= 100


@gpu
def test_torus_200k_converges(cuda):
    verts, faces = dn.synthetic.torus_mesh(400, 500, seed=0)
    k = 128
    st = {}
    frames, mass, L, evals, evecs, gx, gy = dn.geometry.compute_operators(verts.double(), faces, k, device=cuda, stats=st)
    lam, phi, m = evals, evecs, mass
    assert bool((lam[1:] >= lam[:-1]).all())
    G = phi.T @ (phi * m[:, None])
    assert float((G - torch.eye(k, device=cuda, dtype=G.dtype)).abs().max()) <= 1e-5
    # against the fp64 Laplacian (the returned L is rounded to fp32 like the reference's, too coarse for this bound)
    v64, f64 = verts.double().to(cuda), faces.to(cuda)
    rowptr, colidx, lvals = dn.geometry.mesh_laplacian(v64, f64)[:3]
    L64 = torch.sparse_csr_tensor(rowptr.long(), colidx.long(), lvals, (verts.shape[0],) * 2)
    R = L64 @ phi + 1e-8 * phi - (phi * m[:, None]) * lam[None, :]
    lhs = R.norm(dim=0)
    rhs = 1e-5 * lam[-1] * (phi * m[:, None]).norm(dim=0)
    assert bool((lhs <= rhs).all()), (float((lhs / rhs).max()), st)


@gpu
def test_compute_operators_is_deterministic(cuda):
    verts, faces = dn.synthetic.icosphere_mesh(3, seed=5)
    a = dn.geometry.compute_operators(verts, faces, 48, device=cuda)
    b = dn.geometry.compute_operators(verts, faces, 48, device=cuda)
    for x, y in zip(a, b):
        if x.is_sparse:
            assert torch.equal(x.indices(), y.indices()) and torch.equal(x.values(), y.values())
        else:
            assert torch.equal(x, y)


@gpu
def test_cache_miss_writes_the_reference_bucket(cuda, tmp_path):
    z = _entry(FIXTURES[0][0])
    verts, faces = torch.from_numpy(z["verts"]), torch.from_numpy(z["faces"])
    cache = str(tmp_path / "cache")
    out = dn.geometry.get_operators(verts, faces, 16, cache, device=cuda, compute_missing=True)
    name = os.path.basename(glob.glob(os.path.join(FIXTURES[0][0], "*.npz"))[0])
    assert sorted(os.listdir(cache)) == [name]
    w = np.load(os.path.join(cache, name), allow_pickle=True)
    assert sorted(w.files) == sorted(z.files)
    for key in z.files:
        assert w[key].dtype == z[key].dtype and w[key].shape == z[key].shape, key
    assert np.array_equal(w["L_indptr"], z["L_indptr"]) and np.array_equal(w["L_indices"], z["L_indices"])
    assert np.array_equal(w["gradX_indptr"], z["gradX_indptr"]) and np.array_equal(w["gradX_indices"], z["gradX_indices"])
    hit = dn.geometry.get_operators(verts, faces, 16, cache, device=cuda)            # hit through the reader
    for a, b in zip(out, hit):
        if a.is_sparse:
            assert torch.equal(a.coalesce().indices(), b.coalesce().indices())
            assert torch.equal(a.coalesce().values(), b.coalesce().values())
        else:
            assert torch.equal(a, b)
    t0 = os.path.getmtime(os.path.join(cache, name))
    os.utime(os.path.join(cache, name), (t0 - 100, t0 - 100))
    dn.geometry.get_operators(verts, faces, 16, cache, device=cuda, overwrite_cache=True, compute_missing=True)
    assert os.listdir(cache) == [name] and os.path.getmtime(os.path.join(cache, name)) > t0 - 50
    dn.geometry.get_operators(verts, faces, 20, cache, device=cuda, compute_missing=True)   # more k_eig than cached
    assert os.listdir(cache) == [name] and int(np.load(os.path.join(cache, name))["k_eig"]) == 20
    # a planted entry under the same hash but for other vertices sends the write to bucket _1
    cache2 = str(tmp_path / "cache2")
    os.makedirs(cache2)
    planted = dict(np.load(os.path.join(cache, name), allow_pickle=True))
    planted["verts"] = planted["verts"] + 1.0
    np.savez(os.path.join(cache2, name), **planted)
    dn.geometry.get_operators(verts, faces, 16, cache2, device=cuda, compute_missing=True)
    assert sorted(os.listdir(cache2)) == [name, name.replace("_0.npz", "_1.npz")]


@gpu
def test_compute_operators_edge_cases(cuda):
    verts, faces = dn.synthetic.patch_mesh(12, 14, seed=4)
    out = dn.geometry.compute_operators(verts, faces, 0, device=cuda)
    assert out[3].shape == (0,) and out[4].shape == (verts.shape[0], 0)
    # caller-supplied normals replace the computed ones (geometry.py:157-160)
    nrm = torch.zeros(verts.shape[0], 3)
    nrm[:, 1] = 1.0
    fr = dn.geometry.compute_operators(verts, faces, 8, normals=nrm, device=cuda)[0]
    gold = OO.tangent_frames(verts.numpy(), faces.numpy(), normals=nrm.numpy())
    assert O.rel_err(_np(fr), gold) <= 1e-6
    out64 = dn.geometry.compute_operators(verts.double(), faces, 8, device=cuda)
    assert all(t.dtype == torch.float64 for t in out64)
    with pytest.raises(NotImplementedError):
        dn.geometry.compute_operators(verts, torch.zeros(0, 3, dtype=torch.int64), 8, device=cuda)
    with pytest.raises(RuntimeError, match="CUDA devices only"):
        dn.geometry.compute_operators(verts, faces, 8)
    bad = verts.clone()
    bad[3, 1] = float("nan")
    with pytest.raises(RuntimeError, match="NaN"):
        dn.geometry.compute_operators(bad, faces, 8, device=cuda)
    # get_all_operators passes normals[i] through
    outs = dn.geometry.get_all_operators([verts], [faces], 8, None, normals=[nrm], device=cuda, compute_missing=True)
    assert torch.equal(outs[0][0], fr)
