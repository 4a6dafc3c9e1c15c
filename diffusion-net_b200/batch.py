"""Batches of independent meshes as ONE vertex range (BASELINE config 4: 32 small meshes; SURVEY.md 8e).

The reference runs a batch as a Python loop over meshes (layers.py:217-222).  ``MeshBatch`` lays the meshes out
back to back (every start rounded up to a 128-row tile), builds one block-diagonal shared-pattern CSR with
batch-global column indices and the small device tables of ``dn_mesh_batch`` (include/diffusion_net_b200.h), so that
``DiffusionNet.forward_batch`` runs every stage of every block as ONE launch over all meshes
(``dn_block_fwd_batched``): grouped split-V to_basis, one packed spectral multiplier per mesh, a from_basis chain that
picks its weights per tile, and the per-vertex stages (gather, MiniMLP, first/last linear) over the whole range.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib, ops


class MeshBatch:
    """``items``: dicts with mass (V), evals (K), evecs (V,K), gradX, gradY (sparse COO (V,V) or a prepared
    ``ops.GradOperators`` under 'gradX') -- the reference's operator tuple per mesh -- and optionally faces (F,3) /
    edges (E,2) for ``DiffusionNet.forward_batch`` with outputs_at 'faces' / 'edges'.  Build once, reuse every step.

    For nets with diffusion_method='implicit_dense', every item also carries 'L' (sparse COO (V,V) as get_operators
    returns it, or a prepared ``ops.LaplacianCSR``); the batch then holds one block-diagonal Laplacian CSR in its layout
    (``lap``, built on first use, so a spectral net never pays for it; None when the items carry no L;
    ``has_laplacian`` tells which without building it).  Such items may leave out 'evals' / 'evecs' (k_eig = 0): the batch then
    has K = 0 and serves implicit nets only."""

    def __init__(self, items, device=None):
        lib = _lib.load()
        self.n_meshes = B = len(items)
        if B < 1:
            raise ValueError("MeshBatch needs at least one mesh")
        dev = torch.device(device) if device is not None else items[0]["mass"].device
        if dev.type != "cuda":
            raise RuntimeError("diffusion_net_b200 runs on CUDA tensors only (no CPU fallback)")
        self.device = dev
        self.n_rows = [int(it["mass"].shape[0]) for it in items]
        n_eig = lambda it: (int(it["evals"].shape[0]) if it.get("evals") is not None else 0,
                            int(it["evecs"].shape[1]) if it.get("evecs") is not None else 0)
        K = n_eig(items[0])[0]
        if any(n_eig(it) != (K, K) for it in items):
            raise ValueError("every mesh of a batch needs the same number of eigenpairs")
        has_lap = [it.get("L") is not None for it in items]
        if any(has_lap) and not all(has_lap):
            raise ValueError("MeshBatch: 'L' must be given for every item or for none")
        if K == 0 and not all(has_lap):
            raise ValueError("MeshBatch: items without eigenpairs need the Laplacian 'L' (implicit diffusion)")
        self.K = K
        n_rows = np.asarray(self.n_rows, dtype=np.int32)
        row_begin = np.zeros(B + 1, dtype=np.int32)
        tiles_max = int(sum((v + 127) // 128 for v in self.n_rows))
        tile_mesh = np.zeros(max(tiles_max, 1), dtype=np.int32)
        tb_rows = np.zeros(2 * 1024, dtype=np.int32)
        cta_begin = np.zeros(B + 1, dtype=np.int32)
        sm = C.c_int(0)
        cc = C.c_int(0)
        smem = C.c_int64(0)
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        _lib.check(lib.dn_device_query(idx, C.byref(sm), C.byref(cc), C.byref(smem)), "dn_device_query")
        n_ctas = lib.dn_mesh_batch_plan(B, n_rows.ctypes.data, int(sm.value), row_begin.ctypes.data, tile_mesh.ctypes.data,
                                        tb_rows.ctypes.data, cta_begin.ctypes.data)
        if n_ctas < 0:
            _lib.check(n_ctas, "dn_mesh_batch_plan")
        self.row_begin = [int(v) for v in row_begin]
        self.V = V = self.row_begin[-1]
        f32 = dict(dtype=torch.float32, device=dev)
        self.mass = torch.zeros(V, **f32)
        self.evecs = torch.zeros(V, K, **f32)
        self.evals = torch.empty(B, K, **f32)
        rp = [np.zeros(1, dtype=np.int64)]
        cols, vals = [], []
        nnz = 0
        for b, it in enumerate(items):
            r0, n = self.row_begin[b], self.n_rows[b]
            self.mass[r0:r0 + n] = it["mass"].to(**f32)
            if K:
                self.evecs[r0:r0 + n] = it["evecs"].to(**f32)
                self.evals[b] = it["evals"].to(**f32)
            g = it["gradX"]
            if not isinstance(g, ops.GradOperators):
                g = ops.prepare_operators(it["gradX"].to(dev), it["gradY"].to(dev))
            rowptr, colidx, gv = g.to_host_csr()
            rowptr = np.asarray(rowptr, dtype=np.int64)
            pad = (self.row_begin[b + 1] - r0) - n
            rp.append(rowptr[1:] + nnz)
            if pad:
                rp.append(np.full(pad, rowptr[-1] + nnz, dtype=np.int64))
            cols.append(np.asarray(colidx, dtype=np.int64) + r0)
            vals.append(np.asarray(gv, dtype=np.float32).reshape(-1, 2))
            nnz += int(rowptr[-1])
        rowptr = torch.from_numpy(np.concatenate(rp).astype(np.int32)).to(dev)
        colidx = torch.from_numpy(np.concatenate(cols).astype(np.int32)).to(dev)
        vals_xy = torch.from_numpy(np.concatenate(vals)).to(dev)
        self.gops = ops.GradOperators.from_csr(V, rowptr, colidx, vals_xy)
        self._tile_mesh = torch.from_numpy(tile_mesh[:max(V // 128, 1)].copy()).to(dev)
        self._tb_rows = torch.from_numpy(tb_rows[:2 * n_ctas].copy()).to(dev)
        self._cta_begin = torch.from_numpy(cta_begin).to(dev)
        self.desc = _lib.dn_mesh_batch(B, n_ctas, self._tile_mesh.data_ptr(), self._tb_rows.data_ptr(),
                                       self._cta_begin.data_ptr())
        # rows [begin, end) of every mesh, for the implicit solve, and the block-diagonal Laplacian
        rows = np.stack([row_begin[:-1], row_begin[:-1] + n_rows], 1).astype(np.int32)
        self._mesh_rows = torch.from_numpy(rows.reshape(-1).copy()).to(dev)
        self.has_laplacian = all(has_lap)
        self._laps = [it["L"] for it in items] if self.has_laplacian else None
        self._lap = None
        # one row segment per mesh, for the mass-weighted mean of outputs_at 'global_mean' (ops.global_mean_pool)
        self.segments = ops.Segments(self.row_begin[:-1], self.n_rows, V, dev)
        # elements for outputs_at 'faces' / 'edges', vertex ids offset to batch rows (None unless every item has them)
        self.faces, self.edges, self._elem_counts = None, None, {}
        for name in ("faces", "edges"):
            if all(it.get(name) is not None for it in items):
                els = [torch.as_tensor(it[name]).to(device=dev, dtype=torch.int64) for it in items]
                setattr(self, name, torch.cat([e + r0 for e, r0 in zip(els, self.row_begin)], 0))
                self._elem_counts[name] = [int(e.shape[0]) for e in els]

    @property
    def lap(self):
        """The batch's block-diagonal ops.LaplacianCSR (built once, on first use), or None without L."""
        if self._lap is None and self._laps is not None:
            self._lap = self._block_laplacian(self._laps, self.device)
            self._laps = None
        return self._lap

    def _block_laplacian(self, Ls, dev):
        """One ops.LaplacianCSR over the batch layout: mesh b's CSR with its columns offset to its rows, padding rows
        empty (the per-mesh CSRs are built or taken as prepared, then laid out on the host once)."""
        rp = [np.zeros(1, dtype=np.int64)]
        cols, vals = [], []
        nnz = 0
        for b, L in enumerate(Ls):
            lap = L if isinstance(L, ops.LaplacianCSR) else ops.prepare_laplacian(L.to(dev))
            r0, n = self.row_begin[b], self.n_rows[b]
            if not isinstance(lap, ops.LaplacianCSR) or lap.V != n:
                raise ValueError("MeshBatch: mesh {} has {} vertices but its L is not a ({}, {}) Laplacian".format(
                    b, n, n, n))
            _, rowptr, colidx, cv = lap.csr
            rowptr = rowptr.cpu().numpy().astype(np.int64)
            rp.append(rowptr[1:] + nnz)
            pad = (self.row_begin[b + 1] - r0) - n
            if pad:
                rp.append(np.full(pad, rowptr[-1] + nnz, dtype=np.int64))
            cols.append(colidx[:lap.nnz].cpu().numpy().astype(np.int64) + r0)
            vals.append(cv[:2 * lap.nnz].cpu().numpy().reshape(-1, 2))
            nnz += lap.nnz
        if nnz >= 2 ** 31:
            raise ValueError("MeshBatch: the batch Laplacian has {} entries, more than int32 indices hold".format(nnz))
        return ops.LaplacianCSR.from_csr(self.V, torch.from_numpy(np.concatenate(rp).astype(np.int32)).to(dev),
                                         torch.from_numpy(np.concatenate(cols).astype(np.int32)).to(dev),
                                         torch.from_numpy(np.concatenate(vals).astype(np.float32)).to(dev))

    def elem_counts(self, name):
        """Number of 'faces' or 'edges' of every mesh (the split of the batch's element outputs)."""
        return self._elem_counts[name]

    def pack(self, xs):
        """List of per-mesh (V_b, C) features -> one (V, C) tensor in the batch layout (padding rows zero).
        Differentiable: gradients reach every x_b."""
        Cc = xs[0].shape[-1]
        out = torch.zeros(self.V, Cc, dtype=torch.float32, device=self.device)
        for b, x in enumerate(xs):
            out[self.row_begin[b]:self.row_begin[b] + self.n_rows[b]] = x
        return out

    def unpack(self, y):
        return [y[self.row_begin[b]:self.row_begin[b] + self.n_rows[b]] for b in range(self.n_meshes)]


def block_forward_batched_raw(batch, x_in, time, A_re, A_im, weights, biases, with_features, head=None):
    """dn_block_fwd_ex with a batch descriptor: one DiffusionNetBlock (eval) over every mesh of ``batch`` (x_in in the batch
    layout).  ``head``: see ops.block_forward_raw."""
    x_in = ops._f32c(x_in)
    if x_in.shape[0] != batch.V:
        raise ValueError("x_in is not in this batch's layout ({} rows, expected {})".format(x_in.shape[0], batch.V))
    return ops.block_forward_raw(x_in, batch.mass, batch.evals, batch.evecs, batch.gops, time, A_re, A_im, weights, biases,
                                 with_features, head=head, batch_desc=batch.desc)
