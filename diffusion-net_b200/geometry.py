"""The pieces of the reference's ``geometry`` module that sit either side of the block: ``to_basis`` / ``from_basis``
(geometry.py:572-598), heat-kernel-signature features (geometry.py:600-633), the operator cache (geometry.py:426-568)
and operator construction for triangle meshes (geometry.py:101-392) -- all with the reference signatures, all running
the hand-written kernels.
Batched (B,V,*) or single-mesh (V,*) inputs, as the reference accepts."""
from __future__ import annotations

import hashlib
import os

import numpy as np
import torch

from . import _lib, ops


def to_basis(values, basis, massvec):
    """(B,V,D),(B,V,K),(B,V) -> (B,K,D): ``basis^T @ (values * massvec[...,None])`` (geometry.py:572-583).
    Differentiable in ``values`` like the reference's ``torch.matmul`` version (backward = ``from_basis`` with the mass
    as row scale); asking for gradients w.r.t. the operators raises."""
    if values.dim() == 2:
        return ops.to_basis(values, basis, massvec)
    return torch.stack([ops.to_basis(values[b], basis[b], massvec[b]) for b in range(values.shape[0])], 0)


def from_basis(values, basis):
    """(B,K,D),(B,V,K) -> (B,V,D): ``basis @ values`` (geometry.py:586-598, real branch).  Differentiable in ``values``
    (backward = ``to_basis`` without mass)."""
    if values.is_complex() or basis.is_complex():
        raise NotImplementedError("complex from_basis is dead code in the reference (utils.cmatmul does not exist)")
    if values.dim() == 2:
        return ops.from_basis(values, basis)
    return torch.stack([ops.from_basis(values[b], basis[b]) for b in range(values.shape[0])], 0)


# ------------------------------------------------------------------------------------------------
# heat kernel signatures (input features of every experiment that passes --input_features=hks)
# ------------------------------------------------------------------------------------------------
def compute_hks(evals, evecs, scales):
    """(K),(V,K),(S) -> (V,S) or batched (B,K),(B,V,K),(B,S) -> (B,V,S):
    ``sum_k exp(-evals[k]*scales[s]) * evecs[v,k]^2`` (geometry.py:600-628).  One streaming pass over ``evecs``;
    the reference materialises a (B,V,S,K) tensor."""
    if evals.dim() == 1:
        return ops.compute_hks_raw(evals, evecs, scales)
    return torch.stack([ops.compute_hks_raw(evals[b], evecs[b], scales[b]) for b in range(evals.shape[0])], 0)


def compute_hks_autoscale(evals, evecs, count):
    """geometry.py:630-633: ``count`` log-spaced scales in [1e-2, 1]."""
    scales = torch.logspace(-2, 0., steps=count, device=evals.device, dtype=evals.dtype)
    return compute_hks(evals, evecs, scales)


# ------------------------------------------------------------------------------------------------
# operator cache <-> device  (geometry.py:426-568; a miss is built by compute_operators on request)
# ------------------------------------------------------------------------------------------------
def hash_arrays(arrs):
    """utils.py:71-76 -- the cache file name is sha1(verts bytes, faces bytes)."""
    h = hashlib.sha1()
    for a in arrs:
        h.update(np.ascontiguousarray(a).view(np.uint8))
    return h.hexdigest()


def _to_np(t):
    return t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)


def _coo_from_csc(npz, prefix, device, dtype):
    """A scipy-CSC triple of the cache file as the coalesced COO tensor the reference returns (utils.py:50-55)."""
    indptr, indices = npz[prefix + "_indptr"], npz[prefix + "_indices"]
    n = int(npz[prefix + "_shape"][0])
    cols = torch.repeat_interleave(torch.arange(n), torch.as_tensor(np.diff(indptr).astype(np.int64)))
    idx = torch.stack((torch.as_tensor(indices.astype(np.int64)), cols), 0)
    val = torch.as_tensor(npz[prefix + "_data"].astype(np.float32))
    return torch.sparse_coo_tensor(idx, val, (n, n)).coalesce().to(device=device, dtype=dtype)


def load_operators_npz(path_or_npz, k_eig=None, device="cuda", dtype=torch.float32):
    """One cache entry (the ``np.savez`` of geometry.py:548-568) -> the reference's operator tuple
    ``(frames, mass, L, evals, evecs, gradX, gradY)`` resident on ``device``.

    gradX/gradY come back as the same coalesced COO tensors the reference returns, so they can be passed to the
    layers unchanged -- but their kernel-side form (shared-pattern int32 CSR + transposed CSR) is built here directly
    from the file's CSC arrays and registered against those tensors, so the first forward does no conversion."""
    npz = np.load(path_or_npz, allow_pickle=True) if isinstance(path_or_npz, (str, os.PathLike)) else path_or_npz
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("diffusion_net_b200 keeps operators on CUDA devices only (no CPU path); got {}".format(device))
    k_have = int(npz["k_eig"].item())
    k_eig = k_have if k_eig is None else int(k_eig)
    if k_eig > k_have:
        raise ValueError("cache entry holds {} eigenpairs, {} requested".format(k_have, k_eig))
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device=device, dtype=dtype)
    frames, mass = to(npz["frames"]), to(npz["mass"])
    evals, evecs = to(npz["evals"][:k_eig]), to(npz["evecs"][:, :k_eig])
    L = _coo_from_csc(npz, "L", device, dtype)
    V = int(npz["gradX_shape"][0])
    same = (np.array_equal(npz["gradX_indptr"], npz["gradY_indptr"])
            and np.array_equal(npz["gradX_indices"], npz["gradY_indices"]))
    if same and dtype == torch.float32:
        gops = ops.GradOperators.from_csc(V, npz["gradX_indptr"], npz["gradX_indices"], npz["gradX_data"],
                                          npz["gradY_data"], device)
        gradX, gradY = gops.to_sparse_coo()
        ops.register_prepared(gradX, gradY, gops)
    else:  # distinct patterns (never produced by geometry.py:381-382, but legal): generic path at first use
        gradX, gradY = _coo_from_csc(npz, "gradX", device, dtype), _coo_from_csc(npz, "gradY", device, dtype)
    return frames, mass, L, evals, evecs, gradX, gradY


def find_cached_operators(verts, faces, k_eig, op_cache_dir):
    """The cache probe of geometry.py:447-492: returns the opened npz of the matching entry or None."""
    verts_np, faces_np = _to_np(verts), _to_np(faces)
    key = hash_arrays((verts_np, faces_np))
    i = 0
    while True:
        path = os.path.join(op_cache_dir, "{}_{}.npz".format(key, i))
        try:
            npz = np.load(path, allow_pickle=True)
        except FileNotFoundError:
            return None
        if not (np.array_equal(verts_np, npz["verts"]) and np.array_equal(faces_np, npz["faces"])):
            i += 1                       # hash collision: next bucket (geometry.py:470-473)
            continue
        if int(npz["k_eig"].item()) < k_eig or "L_data" not in npz:
            return None                  # the reference would rebuild such an entry (geometry.py:482-490)
        return npz


def find_cache_bucket(verts, faces, op_cache_dir):
    """The file the reference's ``get_operators`` writes a freshly computed entry to (geometry.py:447-533): the first
    ``<sha1>_<i>.npz`` that is absent, unreadable or holds this very mesh (a stale entry -- too few eigenpairs, no
    ``L_data``, or ``overwrite_cache`` -- is rewritten in place); buckets holding other meshes are skipped."""
    verts_np, faces_np = _to_np(verts), _to_np(faces)
    key = hash_arrays((verts_np, faces_np))
    i = 0
    while True:
        path = os.path.join(op_cache_dir, "{}_{}.npz".format(key, i))
        try:
            npz = np.load(path, allow_pickle=True)
            same = np.array_equal(verts_np, npz["verts"]) and np.array_equal(faces_np, npz["faces"])
        except FileNotFoundError:
            return path
        except Exception:                # geometry.py:529-532: an unreadable entry is replaced
            return path
        if same:
            return path
        i += 1                           # hash collision (geometry.py:470-473)


def write_operators_npz(path, verts, faces, k_eig, operators, grad_ops):
    """The ``np.savez`` of geometry.py:539-568 for a tuple returned by ``compute_operators``: fp32 data, int32 index
    arrays, the sparse matrices as CSC.  L is exactly symmetric, so its CSC arrays are its CSR arrays; the CSC of
    gradX / gradY is the transposed device CSR of ``grad_ops`` (``dn_csr_transpose``)."""
    frames, mass, L, evals, evecs, gradX, gradY = operators
    f32 = np.float32
    np_ = lambda t: t.detach().cpu().numpy()
    V = int(mass.shape[0])
    Lc = L.coalesce()
    rows = np_(Lc.indices()[0])
    L_indptr = np.searchsorted(rows, np.arange(V + 1)).astype(np.int32)
    g = grad_ops
    _, rt, ct, vt = g.csr_t
    vt = np_(vt[:2 * g.nnz]).reshape(-1, 2)
    gx_ptr, gx_idx = np_(rt).astype(np.int32), np_(ct[:g.nnz]).astype(np.int32)
    shape = np.array((V, V), dtype=np.int64)
    np.savez(path, verts=_to_np(verts).astype(f32), frames=np_(frames).astype(f32), faces=_to_np(faces), k_eig=k_eig,
             mass=np_(mass).astype(f32), L_data=np_(Lc.values()).astype(f32), L_indices=np_(Lc.indices()[1]).astype(np.int32),
             L_indptr=L_indptr, L_shape=shape, evals=np_(evals).astype(f32), evecs=np_(evecs).astype(f32),
             gradX_data=vt[:, 0].astype(f32), gradX_indices=gx_idx, gradX_indptr=gx_ptr, gradX_shape=shape,
             gradY_data=vt[:, 1].astype(f32), gradY_indices=gx_idx, gradY_indptr=gx_ptr, gradY_shape=shape)


def get_operators(verts, faces, k_eig=128, op_cache_dir=None, normals=None, overwrite_cache=False, device=None,
                  compute_missing=False):
    """``geometry.get_operators`` (geometry.py:426): same arguments, same file naming, same returned tuple.  ``device``
    (extra) places the operators directly on a GPU; default = ``verts.device``.
    On a cache miss (or with ``overwrite_cache``) this raises unless ``compute_missing=True``; then the operators are
    built on the GPU by ``compute_operators`` and, with an ``op_cache_dir``, written to the bucket the reference would
    write (``find_cache_bucket``), in its file format.  The computed tuple is returned; the next call is a hit."""
    verts_np = _to_np(verts)
    if np.isnan(verts_np).any():
        raise RuntimeError("tried to construct operators from NaN verts")
    device = torch.device(device) if device is not None else verts.device
    npz = None
    if op_cache_dir is not None and not overwrite_cache:
        npz = find_cached_operators(verts, faces, k_eig, op_cache_dir)
    if npz is None:
        if not compute_missing:
            raise NotImplementedError(
                "no usable cache entry for this mesh in {!r}: populate the cache with the reference's get_operators(), "
                "or pass compute_missing=True to build the operators on the GPU".format(op_cache_dir))
        out, g = _compute_operators(verts, faces, k_eig, normals, device, None)
        if op_cache_dir is not None:
            os.makedirs(op_cache_dir, exist_ok=True)
            write_operators_npz(find_cache_bucket(verts, faces, op_cache_dir), verts, faces, k_eig, out, g)
        return out
    return load_operators_npz(npz, k_eig=k_eig, device=device, dtype=verts.dtype)


def get_all_operators(verts_list, faces_list, k_eig, op_cache_dir=None, normals=None, device=None,
                      compute_missing=False, batch_misses=False):
    """geometry.py:395-424: seven parallel lists; ``normals[i]`` goes with mesh i.
    ``batch_misses`` (extra, with ``compute_missing``): the meshes without a usable cache entry are built together by
    ``compute_operators_batch`` -- one launch sequence per group of small meshes instead of one eigensolve after the
    other -- and written to the same buckets in the same format; hits are read as without it."""
    if not (batch_misses and compute_missing):
        outs = [get_operators(v, f, k_eig, op_cache_dir, normals=None if normals is None else normals[i], device=device,
                              compute_missing=compute_missing)
                for i, (v, f) in enumerate(zip(verts_list, faces_list))]
        return tuple([o[i] for o in outs] for i in range(7))
    outs, misses = [None] * len(verts_list), []
    for i, (v, f) in enumerate(zip(verts_list, faces_list)):
        if np.isnan(_to_np(v)).any():
            raise RuntimeError("tried to construct operators from NaN verts")
        npz = find_cached_operators(v, f, k_eig, op_cache_dir) if op_cache_dir is not None else None
        if npz is None:
            misses.append(i)
        else:
            outs[i] = load_operators_npz(npz, k_eig=k_eig, device=torch.device(device) if device is not None else v.device,
                                         dtype=v.dtype)
    if misses:
        built = _compute_operators_batch([verts_list[i] for i in misses], [faces_list[i] for i in misses], k_eig,
                                         None if normals is None else [normals[i] for i in misses], device, None, None)
        for i, (out, g) in zip(misses, built):
            outs[i] = out
            if op_cache_dir is not None:
                os.makedirs(op_cache_dir, exist_ok=True)
                write_operators_npz(find_cache_bucket(verts_list[i], faces_list[i], op_cache_dir), verts_list[i],
                                    faces_list[i], k_eig, out, g)
    return tuple([o[i] for o in outs] for i in range(7))


# ------------------------------------------------------------------------------------------------
# operator construction for triangle meshes (geometry.py:276-392) on the GPU
# ------------------------------------------------------------------------------------------------
EPS = 1e-8          # geometry.py:308: mass shift (times the mean) and eigenproblem shift


def _vertex_normals(v64, f64, frames):
    """dn_vertex_frames on a mesh or a disjoint union of meshes: (V,3) fp64 vertex normals (NaN where a vertex has
    none) and whether any is NaN (one host read).  ``frames`` receives frames built from these unrounded normals, for
    ``_frames_from_normals`` to overwrite."""
    V, F = int(v64.shape[0]), int(f64.shape[0])
    dev = v64.device
    nrm = torch.empty(V, 3, dtype=torch.float64, device=dev)
    nbad = torch.zeros(1, dtype=torch.int32, device=dev)
    ws = torch.empty(12 * F + 8 * V + 1024, dtype=torch.uint8, device=dev)
    _lib.call("dn_vertex_frames", v64, f64, F, V, None, nrm, frames, nbad, ws, ws.numel(), ops._stream())
    return nrm, int(nbad.item()) > 0


def _frames_from_normals(normals, dtype, frames):
    """dn_vertex_frames from given (V,3) normals into ``frames`` (V,3,3) fp64; the normals are rounded to ``dtype``
    first, as the reference converts them (geometry.py:144)."""
    nbad = torch.zeros(1, dtype=torch.int32, device=frames.device)
    _lib.call("dn_vertex_frames", None, None, 0, int(frames.shape[0]),
              normals.to(device=frames.device, dtype=dtype).to(torch.float64).contiguous(), None, frames, nbad, None, 0,
              ops._stream())
    return frames


def _vertex_frames(v64, f64, normals, dtype, verts):
    """geometry.py:101-177 for meshes: (V,3,3) fp64 frames from dn_vertex_frames, with the reference's remedy for NaN
    normals (geometry.py:128-141: wiggle the bad vertices with RandomState(777) and recompute; if still NaN, random
    normals from the same seed).  Normals are rounded to ``dtype`` before the frames are built, as the reference
    converts them (geometry.py:144)."""
    dev = v64.device
    frames = torch.empty(int(v64.shape[0]), 3, 3, dtype=torch.float64, device=dev)
    if normals is None:
        normals, any_bad = _vertex_normals(v64, f64, frames)
        if any_bad:
            verts_np = _to_np(verts)
            bad = torch.isnan(normals).any(dim=1, keepdim=True).cpu().numpy()
            bbox = np.amax(verts_np, axis=0) - np.amin(verts_np, axis=0)
            wiggle = (np.random.RandomState(seed=777).rand(*verts_np.shape) - 0.5) * (np.linalg.norm(bbox) * 1e-4)
            wiggled = torch.from_numpy(np.ascontiguousarray(verts_np + bad * wiggle, dtype=np.float64)).to(dev)
            normals, any_bad = _vertex_normals(wiggled, f64, frames)
            if any_bad:
                bad = torch.isnan(normals).any(dim=1).cpu().numpy()
                rnd = (np.random.RandomState(seed=777).rand(*verts_np.shape) - 0.5)[bad, :]
                rnd = rnd / np.linalg.norm(rnd, axis=-1)[:, None]
                normals[torch.from_numpy(bad).to(dev)] = torch.from_numpy(rnd).to(dev)
    return _frames_from_normals(normals, dtype, frames)


def mesh_laplacian(v64, f64, eps=EPS, row_begin=None, first=0):
    """dn_mesh_laplacian: ``(rowptr, colidx, L_vals, mass, A_vals, A_diag, bound)`` on the device (fp64 values, int32
    indices), the reference's cotan Laplacian and lumped mass (geometry.py:322-329) and the operator the eigensolver
    runs on.  Raises the reference's RuntimeError on a NaN Laplacian or mass (geometry.py:326-329).

    With ``row_begin`` (the n + 1 row offsets, an int32 device tensor, of the n meshes whose disjoint union v64 / f64
    hold): dn_mesh_laplacian_batched, which gives each mesh its own mass shift and bound.  ``bound`` is then a numpy
    array of n, an eighth value holds the offsets ``rowptr[row_begin]`` of the meshes' entries (numpy int64), and the
    NaN errors name their mesh, counted from ``first``."""
    V, F = int(v64.shape[0]), int(f64.shape[0])
    n = 1 if row_begin is None else int(row_begin.numel()) - 1
    dev = v64.device
    cap = max(6 * F + V, 1)
    rowptr = torch.empty(V + 1, dtype=torch.int32, device=dev)
    colidx = torch.empty(cap, dtype=torch.int32, device=dev)
    lvals = torch.empty(cap, dtype=torch.float64, device=dev)
    avals = torch.empty(cap, dtype=torch.float64, device=dev)
    mass = torch.empty(V, dtype=torch.float64, device=dev)
    adiag = torch.empty(V, dtype=torch.float64, device=dev)
    bound = torch.empty(n, dtype=torch.float64, device=dev)
    nan = torch.empty(n, 2, dtype=torch.int32, device=dev)
    ws = torch.empty(120 * F + 12 * V + 2048, dtype=torch.uint8, device=dev)
    out = (rowptr, colidx, lvals, mass, avals, adiag, bound, nan, ws, ws.numel(), ops._stream())
    if row_begin is None:
        _lib.call("dn_mesh_laplacian", v64, f64, F, V, eps, *out)
        ends = rowptr[-1:]
    else:
        _lib.call("dn_mesh_laplacian_batched", v64, f64, F, V, n, row_begin, eps, *out)
        ends = rowptr[row_begin.long()]
    del ws, out
    host = torch.cat((bound, nan.flatten().double(), ends.double())).cpu().numpy()      # one read of all three
    bound_h, nan_h, nzb = host[:n], host[n:3 * n].reshape(n, 2), host[3 * n:].astype(np.int64)
    for b in range(n):
        mesh = "" if row_begin is None else "mesh {}: ".format(first + b)
        if nan_h[b, 0]:
            raise RuntimeError(mesh + "NaN Laplace matrix")
        if nan_h[b, 1]:
            raise RuntimeError(mesh + "NaN mass matrix")
    nnz = int(nzb[-1])
    csr = (rowptr, colidx[:nnz], lvals[:nnz], mass, avals[:nnz], adiag)
    return csr + (float(bound_h[0]),) if row_begin is None else csr + (bound_h, nzb)


def compute_operators(verts, faces, k_eig, normals=None, device=None, stats=None):
    """``geometry.compute_operators`` (geometry.py:276-392) for triangle meshes, on the GPU: returns
    ``(frames, mass, L, evals, evecs, gradX, gradY)`` resident on ``device`` (default ``verts.device``), each in the
    dtype of ``verts``; L, gradX and gradY are coalesced COO tensors, and (for fp32) gradX / gradY are registered
    against their prepared CSR so the first forward does no conversion.

    Frames, Laplacian, mass and the eigenpairs are computed in fp64 by the library's kernels (``eigen`` has the
    solver: the k_eig lowest pairs of ``(L + 1e-8 I, M)``, the problem of the reference's ``eigsh(..., sigma=1e-8)``,
    ascending, clipped at 0, sign-fixed so that each eigenvector's largest-magnitude entry is positive).  L is rounded
    to fp32 on the way out as the reference's ``sparse_np_to_torch`` does.  gradX / gradY come from ``dn_build_grad``,
    which is fp32: for fp64 ``verts`` they are still fp32-grade.  Deterministic: two calls give bitwise-equal results.

    Raises RuntimeError for a CPU device or a NaN Laplacian / mass, NotImplementedError for a point cloud (empty
    ``faces``), ValueError for faces outside [0, V), ValueError("failed to compute eigendecomp ...") if the
    eigensolver does not converge or k_eig >= V (the reference's ``eigsh`` refuses k >= V and, after its retries,
    raises that error).  ``stats``
    (dict, optional) receives per-stage times in ms and the solver's counters."""
    return _compute_operators(verts, faces, k_eig, normals, device, stats)[0]


def _compute_operators(verts, faces, k_eig, normals, device, stats):
    """compute_operators, also returning the ``ops.GradOperators`` of (gradX, gradY)."""
    from . import eigen
    device = torch.device(device) if device is not None else verts.device
    if device.type != "cuda":
        raise RuntimeError("diffusion_net_b200 keeps operators on CUDA devices only (no CPU path); got {}".format(device))
    if faces.numel() == 0:
        raise NotImplementedError("point clouds need robust_laplacian.point_cloud_laplacian and a KNN graph; only "
                                  "triangle meshes are supported")
    dtype = verts.dtype
    with torch.cuda.device(device):
        ev = []
        mark = lambda: ev.append(torch.cuda.Event(enable_timing=True)) or ev[-1].record()
        mark()
        v64 = torch.as_tensor(verts).detach().to(device=device, dtype=torch.float64).contiguous()
        f64 = torch.as_tensor(faces).detach().to(device=device, dtype=torch.int64).reshape(-1, 3).contiguous()
        V = int(v64.shape[0])
        if int(f64.min()) < 0 or int(f64.max()) >= V:
            raise ValueError("faces index vertices outside [0, {})".format(V))
        frames = _vertex_frames(v64, f64, normals, dtype, verts)
        mark()
        rowptr, colidx, lvals, mass, avals, adiag, bound = mesh_laplacian(v64, f64)
        mark()
        op = eigen.LaplaceOperator(V, rowptr, colidx, avals, adiag, mass, bound)
        est = {} if stats is not None else None
        evals, evecs = eigen.lowest_eigenpairs(op, int(k_eig), stats=est)
        mark()
        rows = torch.repeat_interleave(torch.arange(V, device=device), (rowptr[1:] - rowptr[:-1]).long(),
                                       output_size=int(colidx.numel()))
        idx = torch.stack((rows, colidx.long()), 0)
        g = build_grad_operators(v64.to(torch.float32), frames.to(torch.float32), idx)
        mark()
        if dtype == torch.float32:
            gradX, gradY = g.to_sparse_coo()
            ops.register_prepared(gradX, gradY, g)
        else:
            gradX, gradY = (t.to(dtype) for t in g.to_sparse_coo())
        L = torch.sparse_coo_tensor(idx, lvals.to(torch.float32).to(dtype), (V, V), is_coalesced=True)
        out = (frames.to(dtype), mass.to(dtype), L, evals.to(dtype), evecs.to(dtype), gradX, gradY)
        if stats is not None:
            torch.cuda.synchronize(device)
            ms = [a.elapsed_time(b) for a, b in zip(ev[:-1], ev[1:])]
            stats.update(frames_ms=ms[0], laplacian_ms=ms[1], eig_ms=ms[2], build_grad_ms=ms[3], **est)
    return out, g


# ------------------------------------------------------------------------------------------------
# the same for a dataset of small meshes: one launch sequence per group of meshes
# ------------------------------------------------------------------------------------------------
def batch_groups(n_rows, max_rows):
    """Consecutive index ranges ``[(i0, i1), ...]`` covering ``range(len(n_rows))`` in order: each group takes meshes
    while its vertex total stays within ``max_rows`` (a single mesh above ``max_rows`` is a group of its own)."""
    groups, i0, total = [], 0, 0
    for i, v in enumerate(n_rows):
        if i > i0 and total + v > max_rows:
            groups.append((i0, i))
            i0, total = i, 0
        total += v
    if len(n_rows) > i0:
        groups.append((i0, len(n_rows)))
    return groups


def compute_operators_batch(verts_list, faces_list, k_eig, normals=None, device=None, max_rows=None, stats=None):
    """``compute_operators`` for a list of triangle meshes (a dataset of small meshes, a few hundred to some ten
    thousand vertices each): a list of its seven-tuples, in order, same dtypes and placement, gradX / gradY registered
    against their prepared CSR.  The meshes of a group are laid out as one disjoint union: frames, Laplacian + mass and
    ``build_grad`` run once on the union (``dn_mesh_laplacian_batched``; the frame and gradient kernels are per vertex
    and work on a union as they are), and ``eigen.lowest_eigenpairs_batch`` iterates all meshes together.

    frames, mass, L, gradX and gradY of every mesh are bitwise what ``compute_operators`` returns for it alone; evals /
    evecs come from a different iteration (no locking, one filter degree for the meshes of a group) and agree to the
    solver's tolerance, with it and between two different lists.  Two calls on the same list give bitwise-equal results.

    ``normals`` is a list (entries may be None).  All meshes share one dtype.  ``max_rows`` caps the vertex total of a
    group (default: what fits a third of the free device memory, at five V x B fp64 blocks, the eigenvectors and the
    Laplacian's workspace per vertex); a longer list is processed group by group.  Errors are ``compute_operators``'
    own, prefixed with ``mesh {i}: ``.  ``stats`` (dict, optional) receives the stage times in ms summed over the
    groups (``laplacian_ms`` includes the upload and the face range check, ``split_ms`` is the cutting of the union
    into per-mesh tensors), the number of groups and the solver's counters per group (``eig``)."""
    return [o for o, _ in _compute_operators_batch(verts_list, faces_list, k_eig, normals, device, max_rows, stats)]


def _compute_operators_batch(verts_list, faces_list, k_eig, normals, device, max_rows, stats):
    """compute_operators_batch, returning (tuple, ops.GradOperators) per mesh."""
    n = len(verts_list)
    if n == 0:
        return []
    device = torch.device(device) if device is not None else verts_list[0].device
    if device.type != "cuda":
        raise RuntimeError("diffusion_net_b200 keeps operators on CUDA devices only (no CPU path); got {}".format(device))
    dtype = verts_list[0].dtype
    for i, (v, f) in enumerate(zip(verts_list, faces_list)):
        if f.numel() == 0:
            raise NotImplementedError("mesh {}: point clouds need robust_laplacian.point_cloud_laplacian and a KNN graph; "
                                      "only triangle meshes are supported".format(i))
        if v.dtype != dtype:
            raise ValueError("mesh {}: the meshes of one call share a dtype ({} after {})".format(i, v.dtype, dtype))
    k_eig = int(k_eig)
    Vs = [int(v.shape[0]) for v in verts_list]
    if max_rows is None:
        from . import eigen
        B = eigen.block_size(None, k_eig)
        with torch.cuda.device(device):
            max_rows = max(torch.cuda.mem_get_info()[0] // 3 // (5 * 8 * B + 8 * k_eig + 2048), 1)
    out = []
    groups = batch_groups(Vs, int(max_rows))
    if stats is not None:
        stats.update(groups=len(groups), frames_ms=0.0, laplacian_ms=0.0, eig_ms=0.0, build_grad_ms=0.0, split_ms=0.0, eig=[])
    with torch.cuda.device(device):
        for i0, i1 in groups:
            out += _compute_group(verts_list[i0:i1], faces_list[i0:i1], k_eig,
                                  [None] * (i1 - i0) if normals is None else list(normals[i0:i1]), device, dtype, i0, stats)
    return out


def _compute_group(verts_list, faces_list, k_eig, normals, device, dtype, first, stats):
    from . import eigen
    n = len(verts_list)
    ev = []
    mark = lambda: ev.append(torch.cuda.Event(enable_timing=True)) or ev[-1].record()
    mark()
    Vs = [int(v.shape[0]) for v in verts_list]
    rb = np.concatenate(([0], np.cumsum(Vs)))
    V = int(rb[-1])
    v64s = [torch.as_tensor(v).detach().to(device=device, dtype=torch.float64).contiguous() for v in verts_list]
    f64s = [torch.as_tensor(f).detach().to(device=device, dtype=torch.int64).reshape(-1, 3) for f in faces_list]
    lohi = torch.stack([torch.stack(torch.aminmax(f)) for f in f64s]).cpu().numpy()      # one read for the range check
    for b in range(n):
        if lohi[b, 0] < 0 or lohi[b, 1] >= Vs[b]:
            raise ValueError("mesh {}: faces index vertices outside [0, {})".format(first + b, Vs[b]))
    v64 = torch.cat(v64s)
    f64 = torch.cat([f + int(rb[b]) for b, f in enumerate(f64s)]).contiguous()
    row_begin = torch.from_numpy(rb.astype(np.int32)).to(device)
    # Laplacian + mass of the union, (mass shift, bound, NaN flags) per mesh
    rowptr, colidx, lvals, mass, avals, adiag, bound_h, nzb = mesh_laplacian(v64, f64, row_begin=row_begin, first=first)
    nnz = int(nzb[-1])
    mark()
    # frames of the union; a mesh with a NaN normal takes compute_operators' own route (its remedy is a host step)
    frames = torch.empty(V, 3, 3, dtype=torch.float64, device=device)
    nrm, any_bad = _vertex_normals(v64, f64, frames)
    redo = []
    if any_bad:
        bad_rows = torch.isnan(nrm).any(dim=1).cpu().numpy()
        redo = [b for b in range(n) if normals[b] is None and bad_rows[rb[b]:rb[b + 1]].any()]
    for b, nb in enumerate(normals):
        if nb is not None:
            nrm[rb[b]:rb[b + 1]] = nb.to(device=device, dtype=torch.float64)
    _frames_from_normals(nrm, dtype, frames)
    for b in redo:
        frames[rb[b]:rb[b + 1]] = _vertex_frames(v64s[b], f64s[b].contiguous(), None, dtype, verts_list[b])
    mark()
    # per-mesh views of the union's CSR with local indices, and the eigenpairs
    rows = torch.repeat_interleave(torch.arange(V, device=device), (rowptr[1:] - rowptr[:-1]).long(), output_size=nnz)
    off = torch.repeat_interleave(row_begin[:-1].long(), torch.from_numpy(np.diff(nzb)).to(device), output_size=nnz)
    col_local = (colidx.long() - off).to(torch.int32)
    lops = []
    for b in range(n):
        r0, r1, p0, p1 = int(rb[b]), int(rb[b + 1]), int(nzb[b]), int(nzb[b + 1])
        lops.append(eigen.LaplaceOperator(Vs[b], rowptr[r0:r1 + 1] - p0, col_local[p0:p1], avals[p0:p1], adiag[r0:r1],
                                          mass[r0:r1], bound_h[b]))
    est = {} if stats is not None else None
    pairs = eigen.lowest_eigenpairs_batch(lops, k_eig, stats=est, first=first)
    mark()
    # build_grad on the union's pattern (one entry more than L's in the row of a vertex no face references)
    g = build_grad_operators(v64.to(torch.float32), frames.to(torch.float32), torch.stack((rows, colidx.long()), 0))
    _, grp, gci, gvals = g.csr
    gnzb = grp[row_begin.long()].cpu().numpy().astype(np.int64)
    goff = torch.repeat_interleave(row_begin[:-1].long(), torch.from_numpy(np.diff(gnzb)).to(device), output_size=g.nnz)
    gcol_local = (gci[:g.nnz].long() - goff).to(torch.int32)
    gv = gvals[:2 * g.nnz].view(-1, 2)
    mark()
    out = []
    lvals32 = lvals.to(torch.float32).to(dtype)
    rows_local = rows - off
    for b in range(n):
        r0, r1, p0, p1 = int(rb[b]), int(rb[b + 1]), int(nzb[b]), int(nzb[b + 1])
        q0, q1 = int(gnzb[b]), int(gnzb[b + 1])
        gb = ops.GradOperators.from_csr(Vs[b], grp[r0:r1 + 1] - q0, gcol_local[q0:q1], gv[q0:q1].clone())
        if dtype == torch.float32:
            gradX, gradY = gb.to_sparse_coo()
            ops.register_prepared(gradX, gradY, gb)
        else:
            gradX, gradY = (t.to(dtype) for t in gb.to_sparse_coo())
        idx = torch.stack((rows_local[p0:p1], col_local[p0:p1].long()), 0)
        L = torch.sparse_coo_tensor(idx, lvals32[p0:p1].clone(), (Vs[b], Vs[b]), is_coalesced=True)
        evals, evecs = pairs[b]
        out.append(((frames[r0:r1].to(dtype), mass[r0:r1].to(dtype), L, evals.to(dtype), evecs.to(dtype), gradX, gradY), gb))
    mark()
    if stats is not None:
        torch.cuda.synchronize(device)
        ms = [a.elapsed_time(b) for a, b in zip(ev[:-1], ev[1:])]
        for key, t in zip(("laplacian_ms", "frames_ms", "eig_ms", "build_grad_ms", "split_ms"), ms):
            stats[key] += t
        stats["eig"].append(est)
    return out


# ------------------------------------------------------------------------------------------------
# operator construction, per-vertex part (SURVEY.md 8f-4): the reference's pure-Python build_grad loop on the device
# ------------------------------------------------------------------------------------------------
def edge_tangent_vectors(verts, frames, edges):
    """Reference geometry.py:198-207 (plain torch ops, any device): (E,2) tangent-plane coordinates of every edge."""
    edge_vecs = verts[edges[1, :], :] - verts[edges[0, :], :]
    basisX = frames[edges[0, :], 0, :]
    basisY = frames[edges[0, :], 1, :]
    return torch.stack(((edge_vecs * basisX).sum(-1), (edge_vecs * basisY).sum(-1)), dim=-1)


def _check_edges(edges, V, edge_tangent):
    """The reference's loop raises IndexError on a tail outside [0, V) and reads one tangent row per edge: refuse bad
    ``edges`` / ``edge_tangent`` on the host instead of letting the kernels drop or over-read them (one host sync)."""
    if edges.dim() != 2 or edges.shape[0] != 2:
        raise ValueError("edges must have shape (2, E), got {}".format(tuple(edges.shape)))
    E = int(edges.shape[1])
    if E > 0:
        lo, hi = (int(x) for x in torch.aminmax(edges))
        if lo < 0 or hi >= V:
            raise IndexError("edges index vertices outside [0, {}): min {}, max {}".format(V, lo, hi))
    if edge_tangent is not None and tuple(edge_tangent.shape) != (E, 2):
        raise ValueError("edge_tangent must have shape ({}, 2), got {}".format(E, tuple(edge_tangent.shape)))


def build_grad_operators(verts, frames, edges, edge_tangent=None):
    """``edge_tangent_vectors`` + ``build_grad`` (reference geometry.py:198-273) on the GPU, straight into the prepared
    shared-pattern CSR the layers consume: returns ``ops.GradOperators`` standing for the (gradX, gradY) pair
    (``.to_sparse_coo()`` gives the two coalesced COO tensors the reference returns).  ``edges``: (2,E) integer tensor
    as in the reference (for meshes: the Laplacian's sparsity pattern, geometry.py:374-376).  Two host syncs (the edge
    range check and the entry count); fp64 2x2 solves like numpy; 1e-6-grade agreement with the reference
    (tests/test_gpu_parity.py).  Raises IndexError for edges outside [0, V), ValueError for an ``edge_tangent`` that is
    not (E, 2)."""
    V = int(verts.shape[0])
    _check_edges(edges, V, edge_tangent)
    ops._require_cuda(verts)
    dev = verts.device
    edges = edges.to(device=dev, dtype=torch.int64).contiguous()
    E = int(edges.shape[1])
    verts = verts.to(torch.float32).contiguous()
    frames = frames.to(device=dev, dtype=torch.float32).contiguous()
    et = None if edge_tangent is None else edge_tangent.to(device=dev, dtype=torch.float32).contiguous()
    rowptr = torch.empty(V + 1, dtype=torch.int32, device=dev)
    colidx = torch.empty(max(E + V, 1), dtype=torch.int32, device=dev)
    vals = torch.empty(max(E + V, 1), 2, dtype=torch.float32, device=dev)
    ws = torch.empty(max(4 * V, 4), dtype=torch.uint8, device=dev)
    with ops._on(verts):
        _lib.call("dn_build_grad", verts, frames, et, edges, E, V, rowptr, colidx, vals, ws, ws.numel(), ops._stream())
    nnz = int(rowptr[-1].item()) if V > 0 else 0
    return ops.GradOperators.from_csr(V, rowptr, colidx[:max(nnz, 1)] if nnz else colidx[:0], vals[:nnz])


def build_grad(verts, edges, edge_tangent_vectors):
    """Drop-in for the reference's ``build_grad`` (geometry.py:209-273): numpy / torch in, scipy complex CSC (V,V) out,
    computed by ``dn_build_grad`` on the current CUDA device instead of the per-vertex Python loop.  Raises IndexError
    for edges outside [0, V), ValueError for tangent vectors that are not (E, 2)."""
    import scipy.sparse
    V = int(verts.shape[0])
    as_t = lambda a: a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))
    edges, edge_tangent_vectors = as_t(edges), as_t(edge_tangent_vectors)
    _check_edges(edges, V, edge_tangent_vectors)
    dev = torch.device("cuda", torch.cuda.current_device())
    g = build_grad_operators(torch.empty(V, 3, device=dev), torch.empty(V, 3, 3, device=dev),
                             edges.to(device=dev, dtype=torch.int64),
                             edge_tangent=edge_tangent_vectors.to(device=dev, dtype=torch.float32))
    rowptr, colidx, vals = g.to_host_csr()
    vals = np.asarray(vals, dtype=np.float64)
    data = vals[:, 0] + 1j * vals[:, 1]
    return scipy.sparse.csr_matrix((data, np.asarray(colidx), np.asarray(rowptr)), shape=(V, V)).tocsc()
