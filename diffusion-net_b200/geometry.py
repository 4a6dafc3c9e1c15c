"""The pieces of the reference's ``geometry`` module that sit either side of the block: ``to_basis`` / ``from_basis``
(geometry.py:572-598), heat-kernel-signature features (geometry.py:600-633) and the READ side of the operator
cache (geometry.py:426-519) -- all with the reference signatures, all running the hand-written kernels.
Batched (B,V,*) or single-mesh (V,*) inputs, as the reference accepts."""
from __future__ import annotations

import hashlib
import os

import numpy as np
import torch

from . import ops


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
# operator cache -> device  (the read side of geometry.py:426-519; construction itself is out of scope)
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


def get_operators(verts, faces, k_eig=128, op_cache_dir=None, normals=None, overwrite_cache=False, device=None):
    """``geometry.get_operators`` (geometry.py:426) for a POPULATED cache: same arguments, same file naming, same
    returned tuple.  ``device`` (extra) places the operators directly on a GPU; default = ``verts.device``.
    Building operators (robust-laplacian / eigsh / build_grad, geometry.py:275-393) is out of this framework's
    scope (SURVEY.md 8f item 4): a cache miss raises instead of computing."""
    verts_np = _to_np(verts)
    if np.isnan(verts_np).any():
        raise RuntimeError("tried to construct operators from NaN verts")
    device = torch.device(device) if device is not None else verts.device
    npz = None
    if op_cache_dir is not None and not overwrite_cache:
        npz = find_cached_operators(verts, faces, k_eig, op_cache_dir)
    if npz is None:
        raise NotImplementedError(
            "no usable cache entry for this mesh in {!r}: operator construction is outside the CUDA hot path -- "
            "populate the cache with the reference's get_operators()".format(op_cache_dir))
    return load_operators_npz(npz, k_eig=k_eig, device=device, dtype=verts.dtype)


def get_all_operators(verts_list, faces_list, k_eig, op_cache_dir=None, normals=None, device=None):
    """geometry.py:395-424: seven parallel lists."""
    outs = [get_operators(v, f, k_eig, op_cache_dir, device=device) for v, f in zip(verts_list, faces_list)]
    return tuple([o[i] for o in outs] for i in range(7))


# ------------------------------------------------------------------------------------------------
# operator construction, per-vertex part (SURVEY.md 8f-4): the reference's pure-Python build_grad loop on the device
# ------------------------------------------------------------------------------------------------
def edge_tangent_vectors(verts, frames, edges):
    """Reference geometry.py:198-207 (plain torch ops, any device): (E,2) tangent-plane coordinates of every edge."""
    edge_vecs = verts[edges[1, :], :] - verts[edges[0, :], :]
    basisX = frames[edges[0, :], 0, :]
    basisY = frames[edges[0, :], 1, :]
    return torch.stack(((edge_vecs * basisX).sum(-1), (edge_vecs * basisY).sum(-1)), dim=-1)


def build_grad_operators(verts, frames, edges, edge_tangent=None):
    """``edge_tangent_vectors`` + ``build_grad`` (reference geometry.py:198-273) on the GPU, straight into the prepared
    shared-pattern CSR the layers consume: returns ``ops.GradOperators`` standing for the (gradX, gradY) pair
    (``.to_sparse_coo()`` gives the two coalesced COO tensors the reference returns).  ``edges``: (2,E) integer tensor
    as in the reference (for meshes: the Laplacian's sparsity pattern, geometry.py:374-376).  One host sync (the entry
    count); fp64 2x2 solves like numpy; 1e-6-grade agreement with the reference (tests/test_gpu_parity.py)."""
    import ctypes as C
    from . import _lib
    ops._require_cuda(verts)
    dev = verts.device
    V = int(verts.shape[0])
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
        _lib.check(_lib.load().dn_build_grad(verts.data_ptr(), frames.data_ptr(), et.data_ptr() if et is not None else None,
                                             edges.data_ptr(), E, V, rowptr.data_ptr(), colidx.data_ptr(), vals.data_ptr(),
                                             ws.data_ptr(), ws.numel(), ops._stream()), "dn_build_grad")
    nnz = int(rowptr[-1].item()) if V > 0 else 0
    return ops.GradOperators.from_csr(V, rowptr, colidx[:max(nnz, 1)] if nnz else colidx[:0], vals[:nnz])


def build_grad(verts, edges, edge_tangent_vectors):
    """Drop-in for the reference's ``build_grad`` (geometry.py:209-273): numpy / torch in, scipy complex CSC (V,V) out,
    computed by ``dn_build_grad`` on the current CUDA device instead of the per-vertex Python loop."""
    import scipy.sparse
    dev = torch.device("cuda", torch.cuda.current_device())
    V = int(verts.shape[0])
    as_t = lambda a, dt: (a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))).to(device=dev, dtype=dt)
    g = build_grad_operators(torch.empty(V, 3, device=dev), torch.empty(V, 3, 3, device=dev), as_t(edges, torch.int64),
                             edge_tangent=as_t(edge_tangent_vectors, torch.float32))
    rowptr, colidx, vals = g.to_host_csr()
    vals = np.asarray(vals, dtype=np.float64)
    data = vals[:, 0] + 1j * vals[:, 1]
    return scipy.sparse.csr_matrix((data, np.asarray(colidx), np.asarray(rowptr)), shape=(V, V)).tocsc()
