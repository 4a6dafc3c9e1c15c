"""CPU restatement (numpy/scipy) of the reference's operator construction for triangle meshes (geometry.py:101-392).

TEST INFRASTRUCTURE ONLY, like ``dn_oracle`` (whose ``build_grad`` / ``edge_tangent_vectors`` it uses): the gold that
``geometry.compute_operators`` is checked against at sizes where ``eigsh`` takes seconds.  Pinned by
``tests/test_gpu_operators.py`` against the cache entries the live reference wrote (``tests/golden/op_cache/`` and
``tests/golden/op_cache_patch/``, the latter from ``oracle/make_golden_ops.py``).  Citations are to
``/root/reference/src/diffusion_net/geometry.py``.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

try:
    from dn_oracle import build_grad, edge_tangent_vectors
except ImportError:                                                            # imported as oracle.dn_oracle_ops
    from .dn_oracle import build_grad, edge_tangent_vectors


def _normalize(x, divide_eps=1e-6):
    return x / (np.linalg.norm(x, axis=-1) + divide_eps)[..., None]                # geometry.py:38-48


def vertex_normals(verts, faces):
    """geometry.py:101-148 for meshes: unit face normals (in verts' dtype, :80-90) summed per vertex in fp64
    (np.add.at, :105-107) and normalised; NaN rows are wiggled with RandomState(777) and recomputed, rows still NaN get
    random normals from the same seed (:128-141).  Returned in verts' dtype (:144)."""
    def mesh_normals(v):
        c = v[faces]
        fn = _normalize(np.cross(c[:, 1] - c[:, 0], c[:, 2] - c[:, 0]))
        out = np.zeros(v.shape)
        for i in range(3):
            np.add.at(out, faces[:, i], fn)
        with np.errstate(invalid="ignore", divide="ignore"):
            return out / np.linalg.norm(out, axis=-1, keepdims=True)
    normals = mesh_normals(verts)
    bad = np.isnan(normals).any(axis=1, keepdims=True)
    if bad.any():
        scale = np.linalg.norm(np.amax(verts, axis=0) - np.amin(verts, axis=0)) * 1e-4
        wiggle = (np.random.RandomState(seed=777).rand(*verts.shape) - 0.5) * scale
        normals = mesh_normals(verts + bad * wiggle)
    bad = np.isnan(normals).any(axis=1)
    if bad.any():
        normals[bad, :] = (np.random.RandomState(seed=777).rand(*verts.shape) - 0.5)[bad, :]
        normals = normals / np.linalg.norm(normals, axis=-1)[:, np.newaxis]
    return normals.astype(verts.dtype)


def tangent_frames(verts, faces, normals=None):
    """geometry.py:151-177: rows (basisX, basisY, normal), in verts' dtype."""
    n = vertex_normals(verts, faces) if normals is None else np.asarray(normals, dtype=verts.dtype)
    e1 = np.array([1, 0, 0], dtype=verts.dtype)
    e2 = np.array([0, 1, 0], dtype=verts.dtype)
    bx = np.where((np.abs(n @ e1) < 0.9)[:, None], e1[None, :], e2[None, :])
    bx = bx - n * (bx * n).sum(-1, keepdims=True)
    bx = _normalize(bx)
    by = np.cross(n, bx)
    return np.stack((bx, by, n), axis=-2)


def compute_operators(verts, faces, k_eig, normals=None):
    """geometry.py:276-392 for triangle meshes in numpy/scipy: ``(frames, mass, L, evals, evecs, gradX, gradY)`` with
    L (scipy CSC), gradX / gradY (scipy CSR) in fp64, frames in verts' dtype.  The Laplacian / areas are the
    restatements of potpourri3d's in ``ref_import`` (the functions that produced the reference-written fixtures), and
    the eigenpairs come from the reference's exact call ``eigsh(L + eps I, k, M, sigma=eps)`` (:340-352), clipped at 0
    and sorted ascending."""
    import scipy.sparse.linalg as sla
    try:
        from ref_import import _cotan_laplacian, _vertex_areas
    except ImportError:                                                        # imported as oracle.dn_oracle
        from .ref_import import _cotan_laplacian, _vertex_areas
    verts, faces = np.asarray(verts), np.asarray(faces)
    eps = 1e-8                                                                 # :308
    v64 = verts.astype(np.float64)
    frames = tangent_frames(verts, faces, normals)                             # :312
    L = _cotan_laplacian(v64, faces, denom_eps=1e-10)                          # :322
    mass = _vertex_areas(v64, faces)                                           # :323
    mass += eps * np.mean(mass)                                                # :324
    if np.isnan(L.data).any():
        raise RuntimeError("NaN Laplace matrix")
    if np.isnan(mass).any():
        raise RuntimeError("NaN mass matrix")
    Lc = L.tocoo()                                                             # :332-334
    if k_eig > 0:
        evals, evecs = sla.eigsh((L + sp.identity(L.shape[0]) * eps).tocsc(), k=k_eig, M=sp.diags(mass), sigma=eps)
        evals = np.clip(evals, a_min=0.0, a_max=float("inf"))                  # :352
        order = np.argsort(evals, kind="stable")
        evals, evecs = evals[order], evecs[:, order]
    else:
        evals, evecs = np.zeros(0), np.zeros((verts.shape[0], 0))
    edges = np.stack((Lc.row, Lc.col), axis=0)                                 # :375
    G = build_grad(verts.shape[0], edges, edge_tangent_vectors(verts, frames, edges))
    return frames, mass, L, evals, evecs, G.real.tocsr(), G.imag.tocsr()


