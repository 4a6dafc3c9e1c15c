"""Batches of independent meshes as ONE vertex range (BASELINE config 4: 32 small meshes; SURVEY.md 8e).

The reference runs a batch as a Python loop over meshes (layers.py:217-222).  ``MeshBatch`` lays the meshes out
back to back (every start rounded up to a 128-row tile), builds one block-diagonal shared-pattern CSR with
batch-global column indices and the small device tables of ``dn_mesh_batch`` (include/diffusion_net_b200.h), so that
``DiffusionNet.forward_batch`` runs every stage of every block as ONE launch over all meshes
(``dn_block_fwd_batched``): grouped split-V to_basis, one packed spectral multiplier per mesh, a from_basis chain that
picks its weights per tile, and the per-vertex stages (gather, MiniMLP, first/last linear) over the whole range.

``MeshDataset`` keeps a whole dataset's operators on the device, back to back without padding, and assembles any batch
of its meshes (a shuffled training step) with one ``dn_batch_gather`` launch: the layout is planned on the host from the
meshes' sizes, its tables go up in one pinned copy, and nothing is read back.  ``MeshBatch(items)`` is the dataset of
``items`` gathered in order.
"""
from __future__ import annotations

import ctypes as C
import operator
import types

import numpy as np
import torch

from . import _lib, ops

# ranges of a gather table (dn_batch_gather): per batch mesh, (src_begin, dst_begin, n, n_dst) in units of
R_ROWS, R_MESH, R_PTR, R_ENT, R_FACES, R_EDGES = range(6)   # rows, meshes, row pointers, CSR entries, faces, edges
N_RANGES = 6
# a BatchSlot holding elements adds: the corners' offset and padding row (the mesh's first row), and the vertex ->
# element CSR entries of faces and edges
R_CORNER_OFF, R_FACES_CSR, R_EDGES_CSR = range(6, 9)
N_SLOT_RANGES = 9
ELEMENT_KINDS = (("faces", R_FACES, R_FACES_CSR), ("edges", R_EDGES, R_EDGES_CSR))
_INT32_LIMIT = 2 ** 31


def _check_items(items, device):
    """MeshBatch's checks of the item dicts, before anything is copied or launched: (device, rows of every mesh, K,
    whether the items carry L).  Every per-mesh array must have its mesh's row count, as the mesh's rows in the
    concatenated dataset are placed by its mass alone."""
    if len(items) < 1:
        raise ValueError("MeshBatch needs at least one mesh")
    dev = torch.device(device) if device is not None else items[0]["mass"].device
    if dev.type != "cuda":
        raise RuntimeError("diffusion_net_b200 runs on CUDA tensors only (no CPU fallback)")
    for b, it in enumerate(items):
        if it["mass"].dim() != 1:
            raise ValueError("MeshBatch: mesh {}'s mass must be 1-D (V,), got shape {}".format(
                b, tuple(it["mass"].shape)))
    n_rows = [int(it["mass"].shape[0]) for it in items]
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
    for b, (it, n) in enumerate(zip(items, n_rows)):
        if K and (tuple(it["evals"].shape) != (K,) or tuple(it["evecs"].shape) != (n, K)):
            raise ValueError("MeshBatch: mesh {} has {} vertices and {} eigenpairs but evals of shape {} and evecs of "
                             "shape {}".format(b, n, K, tuple(it["evals"].shape), tuple(it["evecs"].shape)))
        g = it["gradX"]
        gV = (g.V, g.V) if isinstance(g, ops.GradOperators) else tuple(g.shape)
        if gV != (n, n) or (not isinstance(g, ops.GradOperators) and tuple(it["gradY"].shape) != (n, n)):
            raise ValueError("MeshBatch: mesh {} has {} vertices but gradient operators of shape {}".format(b, n, gV))
    return dev, n_rows, K, all(has_lap)


def _sm_count(dev):
    sm, cc, smem = C.c_int(0), C.c_int(0), C.c_int64(0)
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    _lib.call("dn_device_query", idx, C.byref(sm), C.byref(cc), C.byref(smem))
    return int(sm.value)


def plan_rows(n_rows, sm_count):
    """dn_mesh_batch_plan (host): (row_begin [B + 1], tile_mesh [max(V / 128, 1)], tb_rows [2 n_ctas],
    cta_begin [B + 1], n_ctas) as int32 arrays.  More than 1024 meshes, or a padded total of 2^31 - 256 rows or more,
    raise RuntimeError (unsupported) before anything is allocated."""
    n_rows = np.asarray(n_rows, dtype=np.int64)
    B = len(n_rows)
    padded = (n_rows + 127) // 128 * 128
    if B < 1 or (n_rows < 0).any():
        _lib.check(_lib.ERR_INVALID_ARGUMENT, "dn_mesh_batch_plan")
    if int(padded.sum()) >= _INT32_LIMIT - 256:
        _lib.check(_lib.ERR_UNSUPPORTED, "dn_mesh_batch_plan")
    row_begin = np.zeros(B + 1, dtype=np.int32)
    tile_mesh = np.zeros(max(int(padded.sum()) // 128, 1), dtype=np.int32)
    tb_rows = np.zeros(2 * 1024, dtype=np.int32)
    cta_begin = np.zeros(B + 1, dtype=np.int32)
    n32 = n_rows.astype(np.int32)
    n_ctas = _lib.load().dn_mesh_batch_plan(B, n32.ctypes.data, int(sm_count), row_begin.ctypes.data,
                                            tile_mesh.ctypes.data, tb_rows.ctypes.data, cta_begin.ctypes.data)
    if n_ctas < 0:
        _lib.check(n_ctas, "dn_mesh_batch_plan")
    return row_begin, tile_mesh, tb_rows[:2 * n_ctas].copy(), cta_begin, int(n_ctas)


def _starts(counts):
    """Exclusive prefix sum (int64): where each mesh's units begin in the concatenation."""
    out = np.zeros(len(counts) + 1, dtype=np.int64)
    np.cumsum(counts, out=out[1:])
    return out


def gather_table(ids, n_rows, row_begin, n_ent, n_faces=None, n_edges=None):
    """The (B, N_RANGES, 4) int64 table of dn_batch_gather for batch mesh b = dataset mesh ids[b], from sizes only:
    the dataset's meshes have n_rows rows, n_ent CSR entries (gradient or Laplacian) and n_faces / n_edges elements
    (None: not gathered), back to back; the batch's rows begin at row_begin (plan_rows).  A dataset row-pointer array
    holds n_rows + 1 entries per mesh; the batch writes every mesh's padded rows, and the last mesh also row V."""
    ids = np.asarray(ids, dtype=np.int64)
    n_rows = np.asarray(n_rows, dtype=np.int64)
    B = len(ids)
    rb = np.asarray(row_begin, dtype=np.int64)
    nb, pad = n_rows[ids], rb[1:] - rb[:-1]
    src_row = _starts(n_rows)[ids]
    last = np.zeros(B, dtype=np.int64)
    last[-1] = 1
    t = np.zeros((B, N_RANGES, 4), dtype=np.int64)
    t[:, R_ROWS] = np.stack([src_row, rb[:-1], nb, pad], 1)
    t[:, R_MESH] = np.stack([ids, np.arange(B), np.ones(B, np.int64), np.ones(B, np.int64)], 1)
    t[:, R_PTR] = np.stack([src_row + ids, rb[:-1], nb + 1, pad + last], 1)
    for r, cnt in ((R_ENT, n_ent), (R_FACES, n_faces), (R_EDGES, n_edges)):
        if cnt is not None:
            cnt = np.asarray(cnt, dtype=np.int64)
            c = cnt[ids]
            t[:, r] = np.stack([_starts(cnt)[ids], _starts(c)[:-1], c, c], 1)
    return t


def _int32_entries(t, what):
    nnz = int(t[:, R_ENT, 2].sum())
    if nnz >= _INT32_LIMIT:
        raise ValueError("MeshBatch: the batch {} has {} entries, more than int32 indices hold".format(what, nnz))
    return nnz


def batch_tables(ids, n_rows, n_ent, n_faces=None, n_edges=None, sm_count=132, plan=None):
    """Everything ``MeshDataset.batch`` builds on the host, from the dataset meshes' sizes only (no tensor, no GPU):
    the dn_mesh_batch plan, the per-mesh row ranges of the implicit solve, the global-mean segments and the gather
    table.  A batch that int32 indices cannot address is refused here (RuntimeError for rows, as dn_mesh_batch_plan
    refuses them; ValueError for gradient entries).  ``plan``: plan_rows' result for these meshes, when the caller
    already has it."""
    ids = np.asarray(ids, dtype=np.int64)
    nb = np.asarray(n_rows, dtype=np.int64)[ids]
    row_begin, tile_mesh, tb_rows, cta_begin, n_ctas = plan if plan is not None else plan_rows(nb, sm_count)
    V = int(row_begin[-1])
    table = gather_table(ids, n_rows, row_begin, n_ent, n_faces, n_edges)
    nnz = _int32_entries(table, "gradient operators")
    seg_begin = row_begin[:-1].copy()
    seg_rows = nb.astype(np.int32)
    return dict(row_begin=row_begin, V=V, n_ctas=n_ctas, tile_mesh=tile_mesh[:max(V // 128, 1)].copy(),
                tb_rows=tb_rows, cta_begin=cta_begin,
                mesh_rows=np.stack([seg_begin, seg_begin + seg_rows], 1).reshape(-1).astype(np.int32),
                seg_begin=seg_begin, seg_rows=seg_rows,
                tile_seg=np.asarray(ops.Segments.tile_table(seg_begin, seg_rows, V), dtype=np.int32).reshape(-1),
                table=table, nnz=nnz)


def _upload(arrays, dev):
    """Device copies of host int32 / int64 arrays through ONE pinned buffer and ONE non-blocking copy."""
    offs, total = [], 0
    for a in arrays:
        offs.append(total)
        total += (a.nbytes + 15) // 16 * 16
    host = torch.empty(max(total, 16), dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    for a, o in zip(arrays, offs):
        hv[o:o + a.nbytes] = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    d = host.to(dev, non_blocking=True)
    tdt = {np.dtype(np.int32): torch.int32, np.dtype(np.int64): torch.int64}
    return [d[o:o + a.nbytes].view(tdt[a.dtype]).view(a.shape) for a, o in zip(arrays, offs)]


def _part(src, dst, op, width, rng, table_host, offset_range=0):
    return _lib.dn_gather_part(src.data_ptr(), dst.data_ptr(), op, int(width), rng, offset_range,
                               int(table_host[:, rng, 3].max()))


def _gather(parts, table, n_meshes, dev):
    """One dn_batch_gather launch; parts whose batch array is empty are left out (no launch when none is left)."""
    parts = [p for p, dst in parts if dst.numel() > 0 and p.width > 0]
    if not parts:
        return
    arr = (_lib.dn_gather_part * len(parts))(*parts)
    with torch.cuda.device(dev):
        _lib.call("dn_batch_gather", arr, len(parts), table, N_RANGES, n_meshes, ops._stream())


class _DatasetLaplacian:
    """The dataset's per-mesh Laplacians, concatenated on first use (a spectral net never pays for them): local CSRs
    back to back, every mesh's row pointers (V_b + 1 entries) kept."""

    def __init__(self, Ls, n_rows, dev):
        self._Ls, self.n_rows, self.device = Ls, n_rows, dev
        self.arrays = None

    def get(self):
        if self.arrays is None and self._Ls is not None:
            laps = []
            for b, (L, n) in enumerate(zip(self._Ls, self.n_rows)):
                lap = L if isinstance(L, ops.LaplacianCSR) else ops.prepare_laplacian(L.to(self.device))
                if not isinstance(lap, ops.LaplacianCSR) or lap.V != n:
                    raise ValueError("MeshBatch: mesh {} has {} vertices but its L is not a ({}, {}) Laplacian".format(
                        b, n, n, n))
                laps.append(lap)
            self.arrays = (torch.cat([l.csr[1] for l in laps]), torch.cat([l.csr[2][:l.nnz] for l in laps]),
                           torch.cat([l.csr[3][:2 * l.nnz] for l in laps]), [l.nnz for l in laps])
            self._Ls = None
        return self.arrays


class MeshDataset:
    """A dataset of meshes resident on the device, from which any batch is assembled on the GPU.

    ``items``: the item dicts ``MeshBatch`` takes (mass, evals / evecs, gradX / gradY or a prepared
    ``ops.GradOperators`` under 'gradX', optionally L (sparse or ``ops.LaplacianCSR``), faces, edges), checked as
    ``MeshBatch`` checks them.  Everything is concatenated once on the device with device-to-device copies, without
    padding (int64 offsets: a dataset may hold more than 2^31 rows or entries; only a batch must fit int32), and the
    per-mesh sizes and offsets stay on the host (``n_meshes``, ``n_rows``, ``row_begin``, ``K``).  The caller may drop
    the per-mesh tensors afterwards; Laplacians given as sparse L are kept until first used.

    ``batch(ids)`` returns the ``MeshBatch`` of the meshes ``ids`` (repeats allowed) with one kernel launch, no host
    synchronisation and no device-to-host transfer, so a shuffled training loop queues each step's batch behind the
    previous step's work::

        ds = MeshDataset(items)
        for ids in torch.randperm(len(items), generator=g).split(32):
            b = ds.batch(ids.tolist())
            losses, _ = net.forward_batch_global_nll(b, ds.pack(features, b), labels[ids])
    """

    def __init__(self, items, device=None):
        dev, n_rows, K, has_lap = _check_items(items, device)
        self._build(items, dev, n_rows, K, has_lap, _sm_count(dev))

    def _build(self, items, dev, n_rows, K, has_lap, sm):
        """The concatenation, from what _check_items returned for ``items`` and the device's SM count."""
        self.device, self.n_meshes, self.n_rows, self.K = dev, len(items), n_rows, K
        self.row_begin = [int(v) for v in _starts(n_rows)]
        self.V = self.row_begin[-1]
        self._sm = sm
        f32 = dict(dtype=torch.float32, device=dev)
        self.mass = torch.cat([it["mass"].to(**f32) for it in items])
        self.evecs = torch.cat([it["evecs"].to(**f32) for it in items]) if K else torch.zeros(self.V, 0, **f32)
        self.evals = torch.stack([it["evals"].to(**f32) for it in items]) if K else torch.zeros(self.n_meshes, 0, **f32)
        grads = [it["gradX"] if isinstance(it["gradX"], ops.GradOperators) else
                 ops.prepare_operators(it["gradX"].to(dev), it["gradY"].to(dev)) for it in items]
        self._grad_nnz = [g.nnz for g in grads]
        self._grad = (torch.cat([g.csr[1] for g in grads]), torch.cat([g.csr[2][:g.nnz] for g in grads]),
                      torch.cat([g.csr[3][:2 * g.nnz] for g in grads]))
        self._elems = {}
        for name in ("faces", "edges"):
            if all(it.get(name) is not None for it in items):
                els = [torch.as_tensor(it[name]).to(device=dev, dtype=torch.int64) for it in items]
                self._elems[name] = (torch.cat(els, 0), [int(e.shape[0]) for e in els])
        self.has_laplacian = has_lap
        self._lap = _DatasetLaplacian([it["L"] for it in items] if has_lap else None, n_rows, dev)

    def __len__(self):
        return self.n_meshes

    def _ids(self, ids):
        if torch.is_tensor(ids):
            if ids.device.type != "cpu":
                raise ValueError("MeshDataset.batch: ids must be a host list or a CPU tensor, got a tensor on {}: the "
                                 "batch layout is planned on the host from the meshes' sizes".format(ids.device))
            if ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool or ids.dim() > 1:
                raise TypeError("MeshDataset.batch: ids must be integers, got a {} tensor of shape {}".format(
                    ids.dtype, tuple(ids.shape)))
            ids = ids.tolist()
        ids = [operator.index(i) for i in ids]
        if not ids:
            raise ValueError("MeshDataset.batch needs at least one mesh id")
        bad = [i for i in ids if not 0 <= i < self.n_meshes]
        if bad:
            raise IndexError("MeshDataset.batch: mesh id {} is outside the dataset's {} meshes".format(bad[0],
                                                                                                     self.n_meshes))
        return ids

    def batch(self, ids):
        """The ``MeshBatch`` of dataset meshes ``ids`` (a host list or a CPU int tensor; repeats allowed), bitwise
        what ``MeshBatch([items[i] for i in ids])`` builds.  One kernel launch; no host synchronisation."""
        ids = self._ids(ids)
        mb = MeshBatch.__new__(MeshBatch)
        mb._gather_from(self, ids)
        return mb

    def pack(self, t, batch, rotations=None):
        """A per-vertex tensor in the dataset layout (V_total,) or (V_total, C), float32 (features such as HKS or xyz)
        or int64 (labels), in ``batch``'s layout with zero padding rows: one launch, no host synchronisation.  Data
        only: a tensor that requires grad is refused (per-mesh lists still go through ``MeshBatch.pack``).

        ``rotations``: (batch.n_meshes, 3, 3) float32 (``random_rotations``) for float32 (V_total, 3) data such as
        vertex positions: every batch mesh's rows are multiplied by its matrix, ``x_b @ R_b`` as the reference's
        ``random_rotate_points`` does, by one more launch (``rotate_rows``)."""
        if getattr(batch, "_source", None) is not self._lap:
            raise ValueError("MeshDataset.pack: the batch was not drawn from this dataset")
        self._check_pack(t, "MeshDataset.pack")
        _check_rotated(t, rotations, batch, "MeshDataset.pack")
        t = t.contiguous()
        out = torch.empty((batch.V,) + tuple(t.shape[1:]), dtype=t.dtype, device=batch.device)
        width = (t.shape[1] if t.dim() == 2 else 1) * (2 if t.dtype == torch.int64 else 1)
        _gather([(_part(t, out, _lib.GATHER_COPY, width, R_ROWS, batch._table_host), out)], batch._table,
                batch.n_meshes, batch.device)
        if rotations is not None:
            _rotate(out, batch, rotations, out)
        return out

    def slot(self, n_meshes, max_rows=None, max_entries=None, elements=(), max_elements=None):
        """A ``BatchSlot`` of ``n_meshes`` meshes of this dataset: a batch whose buffers never move, refilled on the
        device from any mesh ids, so that a shuffled training step can be captured in one CUDA graph.  Its default
        capacity holds any ``n_meshes`` distinct meshes; ``max_rows`` / ``max_entries`` set it instead.
        ``elements``: 'faces', 'edges' or both (a sequence), for outputs_at 'faces' / 'edges' training: the slot then
        also holds those elements of the batch (the dataset's items must carry them), with ``max_elements`` (an int
        for every kind, or a dict by kind) setting their capacity; a slot sized for repeated ids by ``max_rows`` needs
        ``max_elements`` too."""
        return BatchSlot(self, n_meshes, max_rows, max_entries, elements, max_elements)

    def _check_pack(self, t, what, n=None):
        n = self.V if n is None else n
        if not torch.is_tensor(t) or t.dim() not in (1, 2) or t.shape[0] != n or \
                t.dtype not in (torch.float32, torch.int64):
            raise ValueError("{0}: expected a float32 or int64 tensor of shape ({1},) or ({1}, C) in the dataset layout, "
                             "got {2}".format(what, n, (tuple(t.shape), t.dtype) if torch.is_tensor(t)
                                              else type(t)))
        if t.requires_grad:
            raise ValueError("{} gathers data; got a tensor that requires grad (pack per-mesh tensors with "
                             "MeshBatch.pack to differentiate through the layout)".format(what))
        ops._require_cuda(t)
        if t.device != self.device:
            raise ValueError("{}: the tensor is on {}, the dataset on {}".format(what, t.device, self.device))

    def _slot_tables(self):
        """What every slot reads, built on first slot creation: the per-mesh size table on the device (rows, first row,
        gradient entries, first entry), and every mesh's transposed gradient CSR back to back in the forward CSR's
        layout (the transpose of a block-diagonal matrix is the block diagonal of the transposes, so a slot gathers it
        like the forward CSR and never transposes)."""
        if getattr(self, "_slot_data", None) is None:
            rowptr, colidx, vals = self._grad
            parts, ent0 = [], 0
            for i, (r0, n, nnz) in enumerate(zip(self.row_begin, self.n_rows, self._grad_nnz)):
                g = ops.GradOperators.from_csr(n, rowptr[r0 + i:r0 + i + n + 1], colidx[ent0:ent0 + nnz],
                                               vals[2 * ent0:2 * (ent0 + nnz)].view(-1, 2))
                _, rt, ct, vt = g.csr_t
                parts.append((rt, ct[:nnz], vt[:2 * nnz]))
                ent0 += nnz
            grad_t = tuple(torch.cat(p) for p in zip(*parts))
            sizes = np.stack([np.asarray(self.n_rows, np.int64), np.asarray(self.row_begin[:-1], np.int64),
                              np.asarray(self._grad_nnz, np.int64), _starts(self._grad_nnz)[:-1]], 1)
            self._slot_data = (torch.from_numpy(sizes).to(self.device), grad_t)
        return self._slot_data

    def _slot_element_tables(self, names):
        """What a slot holding the element kinds ``names`` reads besides _slot_tables': the size table with the columns
        dn_mesh_batch_plan_device_elements reads (_slot_tables' four, then (elements, first element) per kind), and
        per kind every mesh's vertex -> element CSR (ops.element_csr of its own elements: n_rows + 1 row pointers and
        k mesh-local element indices per element) back to back like the elements, so a slot gathers it and never
        sorts.  Each kind's CSR is built once, on the first slot that asks for that kind."""
        if getattr(self, "_slot_elem", None) is None:
            self._slot_elem = {}
        for name in names:
            if name not in self._slot_elem:
                els, counts = self._elems[name]
                self._check_elements(name, els, counts)
                rowptrs, entries, e0 = [], [], 0
                for n, cnt in zip(self.n_rows, counts):
                    rowptr, ent = ops.element_csr(els[e0:e0 + cnt], n)
                    rowptrs.append(rowptr)
                    entries.append(ent)
                    e0 += cnt
                self._slot_elem[name] = (torch.cat(rowptrs), torch.cat(entries))
        sizes = self._slot_tables()[0]
        cols = [sizes] + [torch.from_numpy(np.stack([np.asarray(self._elems[n][1], np.int64),
                                                     _starts(self._elems[n][1])[:-1]], 1)).to(self.device)
                          for n in names]
        return torch.cat(cols, 1).contiguous(), {n: self._slot_elem[n] for n in names}

    def _check_elements(self, name, els, counts):
        """Every corner of every mesh's elements names one of the mesh's vertices (one device-to-host read): a slot
        gathers and sorts them on the device, where an index out of range would read past its rows."""
        if els.shape[0] == 0:
            return
        dev = els.device
        mesh = torch.repeat_interleave(torch.arange(self.n_meshes, device=dev), torch.tensor(counts, device=dev))
        n = torch.tensor(self.n_rows, dtype=torch.int64, device=dev)[mesh]
        bad = ((els < 0) | (els >= n[:, None])).any(dim=1)
        if bool(bad.any()):
            e = int(bad.nonzero()[0, 0])
            m = int(mesh[e])
            raise ValueError("MeshDataset.slot: {} {} of mesh {} has a corner outside the mesh's {} vertices".format(
                name[:-1], e - int(_starts(counts)[m]), m, self.n_rows[m]))


class MeshBatch:
    """``items``: dicts with mass (V), evals (K), evecs (V,K), gradX, gradY (sparse COO (V,V) or a prepared
    ``ops.GradOperators`` under 'gradX') -- the reference's operator tuple per mesh -- and optionally faces (F,3) /
    edges (E,2) for ``DiffusionNet.forward_batch`` with outputs_at 'faces' / 'edges'.  Build once, reuse every step;
    for a different set of meshes every step, draw the batches from a ``MeshDataset``.

    For nets with diffusion_method='implicit_dense', every item also carries 'L' (sparse COO (V,V) as get_operators
    returns it, or a prepared ``ops.LaplacianCSR``); the batch then holds one block-diagonal Laplacian CSR in its layout
    (``lap``, built on first use, so a spectral net never pays for it; None when the items carry no L;
    ``has_laplacian`` tells which without building it).  Such items may leave out 'evals' / 'evecs' (k_eig = 0): the batch then
    has K = 0 and serves implicit nets only.

    ``MeshBatch(items)`` is ``MeshDataset(items).batch(range(len(items)))``: the layout is planned (and a batch too
    large for it refused) before anything is copied."""

    def __init__(self, items, device=None):
        dev, n_rows, K, has_lap = _check_items(items, device)
        sm = _sm_count(dev)
        plan = plan_rows(n_rows, sm)        # more than 1024 meshes or int32 rows: refused before anything is copied
        ds = MeshDataset.__new__(MeshDataset)
        ds._build(items, dev, n_rows, K, has_lap, sm)
        self._gather_from(ds, list(range(len(items))), plan)
        self._private_source = True         # nothing else draws from this dataset: lap may drop it once built

    def _gather_from(self, ds, ids, plan=None):
        dev = ds.device
        n_faces, n_edges = (ds._elems[k][1] if k in ds._elems else None for k in ("faces", "edges"))
        t = batch_tables(ids, ds.n_rows, ds._grad_nnz, n_faces, n_edges, ds._sm, plan)
        self.n_meshes = B = len(ids)
        self.device, self.K = dev, ds.K
        self.n_rows = [ds.n_rows[i] for i in ids]
        self.row_begin = [int(v) for v in t["row_begin"]]
        self.V = V = t["V"]
        self._table_host = tab = t["table"]
        (self._table, self._tile_mesh, self._tb_rows, self._cta_begin, self._mesh_rows, seg_begin, seg_rows,
         tile_seg) = _upload([tab, t["tile_mesh"], t["tb_rows"], t["cta_begin"], t["mesh_rows"], t["seg_begin"],
                              t["seg_rows"], t["tile_seg"]], dev)
        f32, i32 = dict(dtype=torch.float32, device=dev), dict(dtype=torch.int32, device=dev)
        self.mass = torch.empty(V, **f32)
        self.evecs = torch.empty(V, ds.K, **f32)
        self.evals = torch.empty(B, ds.K, **f32)
        rowptr, colidx = torch.empty(V + 1, **i32), torch.empty(t["nnz"], **i32)
        vals_xy = torch.empty(t["nnz"], 2, **f32)
        g_rowptr, g_colidx, g_vals = ds._grad
        COPY, ADD32, ADD64 = _lib.GATHER_COPY, _lib.GATHER_ADD_I32, _lib.GATHER_ADD_I64
        parts = [(_part(ds.mass, self.mass, COPY, 1, R_ROWS, tab), self.mass),
                 (_part(ds.evecs, self.evecs, COPY, ds.K, R_ROWS, tab), self.evecs),
                 (_part(ds.evals, self.evals, COPY, ds.K, R_MESH, tab), self.evals),
                 (_part(g_rowptr, rowptr, ADD32, 1, R_PTR, tab, R_ENT), rowptr),
                 (_part(g_colidx, colidx, ADD32, 1, R_ENT, tab, R_ROWS), colidx),
                 (_part(g_vals, vals_xy, COPY, 2, R_ENT, tab), vals_xy)]
        # elements for outputs_at 'faces' / 'edges', vertex ids offset to batch rows (None unless every item has them)
        self.faces, self.edges, self._elem_counts = None, None, {}
        for name, rng in (("faces", R_FACES), ("edges", R_EDGES)):
            if name in ds._elems:
                src, counts = ds._elems[name]
                out = torch.empty((int(tab[:, rng, 2].sum()),) + tuple(src.shape[1:]), dtype=torch.int64, device=dev)
                parts.append((_part(src, out, ADD64, int(np.prod(src.shape[1:])), rng, tab, R_ROWS), out))
                setattr(self, name, out)
                self._elem_counts[name] = [counts[i] for i in ids]
        _gather(parts, self._table, B, dev)
        self.gops = ops.GradOperators.from_csr(V, rowptr, colidx, vals_xy)
        self.desc = _lib.dn_mesh_batch(B, t["n_ctas"], self._tile_mesh.data_ptr(), self._tb_rows.data_ptr(),
                                       self._cta_begin.data_ptr())
        # one row segment per mesh, for the mass-weighted mean of outputs_at 'global_mean' (ops.global_mean_pool)
        self.segments = ops.Segments.wrap(V, seg_begin, seg_rows, tile_seg)
        self.has_laplacian = ds.has_laplacian
        self._source, self._ids, self._lap, self._private_source = ds._lap, ids, None, False

    @property
    def lap(self):
        """The batch's block-diagonal ops.LaplacianCSR (built once, on first use, by a second dn_batch_gather), or
        None without L."""
        if self._lap is None and self.has_laplacian:
            l_rowptr, l_colidx, l_vals, l_nnz = self._source.get()
            tab = gather_table(self._ids, self._source.n_rows, self.row_begin, l_nnz)
            nnz = _int32_entries(tab, "Laplacian")
            table, = _upload([tab], self.device)
            i32 = dict(dtype=torch.int32, device=self.device)
            rowptr, colidx = torch.empty(self.V + 1, **i32), torch.empty(nnz, **i32)
            vals = torch.empty(nnz, 2, dtype=torch.float32, device=self.device)
            _gather([(_part(l_rowptr, rowptr, _lib.GATHER_ADD_I32, 1, R_PTR, tab, R_ENT), rowptr),
                     (_part(l_colidx, colidx, _lib.GATHER_ADD_I32, 1, R_ENT, tab, R_ROWS), colidx),
                     (_part(l_vals, vals, _lib.GATHER_COPY, 2, R_ENT, tab), vals)], table, self.n_meshes, self.device)
            self._lap = ops.LaplacianCSR.from_csr(self.V, rowptr, colidx, vals)
            if self._private_source:        # MeshBatch(items): its dataset's Laplacian copy is not needed any more
                self._source = None
        return self._lap

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


def slot_capacity(n_rows, n_ent, n_meshes, sm_count):
    """(V_cap, entry_cap, n_tb_ctas) of a slot that holds any ``n_meshes`` distinct meshes of a dataset whose meshes
    have ``n_rows`` rows and ``n_ent`` gradient entries: the sum of the n_meshes largest padded row counts (at least one
    tile), the sum of the n_meshes largest entry counts (taken on their own: they may be other meshes'), and the
    to_basis grid min(1024, sm_count + n_meshes).

    The grid bound: dn_mesh_batch_plan gives mesh b want_b = round(chunks_b sm / total) CTAs, raised to 1, lowered to
    chunks_b, lowered to 1 near the 1024 budget, then lowered again to ceil(chunks_b / per).  Rounding adds at most 1/2
    and raising to 1 makes a value below 1/2 into 1, so want_b <= chunks_b sm / total + 1 and the batch uses at most
    sum_b (chunks_b sm / total + 1) = sm + n_meshes CTAs, and never more than 1024."""
    padded = sorted(((int(n) + 127) // 128 * 128 for n in n_rows), reverse=True)
    v_cap = max(sum(padded[:n_meshes]), 128)
    e_cap = sum(sorted((int(e) for e in n_ent), reverse=True)[:n_meshes])
    return v_cap, e_cap, min(1024, int(sm_count) + n_meshes)


def slot_element_capacity(n_elems, n_meshes):
    """The element capacity of a slot that holds any ``n_meshes`` distinct meshes whose meshes have ``n_elems``
    elements of one kind: the sum of the n_meshes largest counts, each padded to a 128-element tile (at least one
    tile), as slot_capacity sizes the rows."""
    padded = sorted(((int(n) + 127) // 128 * 128 for n in n_elems), reverse=True)
    return max(sum(padded[:n_meshes]), 128)


_ST_BAD_ID, _ST_OVER_CAPACITY = 1, 2


class BatchSlot:
    """A batch of ``n_meshes`` meshes of a ``MeshDataset`` whose device buffers never move: ``fill(ids)`` rewrites
    their contents from any mesh ids with a fixed launch sequence (a device planner, ``dn_mesh_batch_plan_device``, and
    one ``dn_batch_gather``) that reads nothing back and allocates nothing, so a shuffled training step, fill
    included, can be captured in one CUDA graph (``graphs.GraphedTrainStep``) and replayed with new ids::

        slot = ds.slot(32)
        ids = torch.zeros(32, dtype=torch.int64, device="cuda")
        def step(net, ids):
            slot.fill(ids)
            return net.forward_batch_global_nll(slot, slot.pack(X), slot.take(Y), label_smoothing=0.2)[0].sum()
        g = dn.graphs.GraphedTrainStep(net, step, (ids,))
        for chunk in torch.randperm(len(ds), device="cuda").split(32):   # a short last chunk needs its own slot
            if len(chunk) == 32:
                ids.copy_(chunk); g.zero_grads(net); g.replay(); opt.step()

    The reference's loop (one mesh per step, ``batch_size=None``) is ``ds.slot(1)`` with one graph.

    Fixed for the slot's life: ``n_meshes``, ``V`` (the row capacity V_cap), the gradient entry capacity, the to_basis
    grid and so every workspace size (``slot_capacity``).  A filled slot is ``ds.batch(ids)``'s layout on the batch's
    rows, bitwise, and the rows past them up to V are padding of the last mesh (mass, evecs and features 0, no
    gradient entries, tiles of the last mesh, outside every global-mean segment).  The to_basis CTAs past the batch's
    own get empty row ranges that no mesh reduces.  The backward's transposed gradient CSR is gathered from per-mesh
    transposes the dataset builds once.

    A fill from host ids checks them first (``MeshDataset.batch``'s errors, and a ValueError for a batch past the
    capacity, possible with repeats).  Device ids are checked on the device: an id outside the dataset or a batch past
    the capacity reads nothing through the ids and plans every mesh empty, so the step computes NaN for every loss
    (0 / 0 means) and NaN parameter gradients, and sets a sticky status that ``check()`` reads.

    Elements: a slot made with ``elements='faces'`` (and / or 'edges', which the dataset's items must carry) holds them
    too, in an element layout of fixed capacity (``element_capacity[name]``: by default the sum of the n_meshes largest
    element counts, each padded to 128, so any n_meshes distinct meshes fit; ``max_elements`` sets it, and a slot
    sized for repeated ids needs it as much as ``max_rows``) planned and gathered by the same two launches.  A slot
    made without ``elements`` holds none, whatever the items carry, and plans and gathers exactly what it did before
    elements existed.  Every mesh's elements
    begin on a 128-element tile; ``faces`` / ``edges`` are int64 (capacity, k) with vertex ids in slot rows, each
    padding element's corners the first row of its mesh (row 0 past the batch), so every corner names a row.
    ``element_segments[name]`` is one ``ops.Segments`` per mesh over the element layout and ``element_csr(name)`` the
    vertex -> element CSR of the real elements (ops.element_csr's format, gathered from per-mesh CSRs the dataset
    builds once): no vertex's entries reach a padding element.  ``pack_elements(t, name)`` brings per-element data
    (labels) into the element layout.  A batch whose elements exceed the capacity is over capacity like one whose rows
    do.

    Spectral nets on ``forward_batch_global_nll``, on ``forward_batch_nll`` with per-vertex labels in the batch layout
    (``pack``), and for outputs_at 'faces' / 'edges' on ``forward_batch_nll`` with labels in the element layout
    (``pack_elements``).  A slot keeps no host copy of its layout: ``n_rows``, ``row_begin``, ``unpack``,
    ``elem_counts``, ``forward_batch`` and implicit nets raise NotImplementedError."""

    element_capacity = types.MappingProxyType({})     # element kind -> capacity (read-only); none unless asked for

    def __init__(self, ds, n_meshes, max_rows=None, max_entries=None, elements=(), max_elements=None):
        n_meshes = operator.index(n_meshes)
        if n_meshes < 1:
            raise ValueError("MeshDataset.slot needs at least one mesh")
        if n_meshes > 1024:
            _lib.check(_lib.ERR_UNSUPPORTED, "MeshDataset.slot ({} meshes; at most 1024)".format(n_meshes))
        if ds.K == 0:
            raise ValueError("MeshDataset.slot: the dataset has no eigenpairs (k_eig = 0); a slot serves spectral nets")
        v_cap, e_cap, n_ctas = slot_capacity(ds.n_rows, ds._grad_nnz, n_meshes, ds._sm)
        if max_rows is not None:
            v_cap = max((operator.index(max_rows) + 127) // 128 * 128, 128)
        if max_entries is not None:
            e_cap = operator.index(max_entries)
        if v_cap >= _INT32_LIMIT - 256:
            _lib.check(_lib.ERR_UNSUPPORTED, "MeshDataset.slot ({} rows)".format(v_cap))
        if e_cap >= _INT32_LIMIT or e_cap < 0:
            raise ValueError("MeshBatch: the batch gradient operators have {} entries, more than int32 indices "
                             "hold".format(e_cap))
        names = (elements,) if isinstance(elements, str) else tuple(elements or ())
        for name in names:
            if name not in ("faces", "edges") or names.count(name) > 1:
                raise ValueError("MeshDataset.slot: elements are 'faces' and / or 'edges', each once; got {!r}".format(
                    elements))
            if name not in ds._elems:
                raise ValueError("MeshDataset.slot: elements={!r}, but the dataset's items carry no '{}'".format(
                    elements, name))
        if max_elements is not None and not names:
            raise ValueError("MeshDataset.slot: max_elements sizes the elements the slot holds; pass elements= too")
        if isinstance(max_elements, dict) and set(max_elements) - set(names):
            raise ValueError("MeshDataset.slot: max_elements names {} the slot does not hold ({})".format(
                sorted(set(max_elements) - set(names)), list(names)))
        kinds = [(name, rng, csr_rng) for name, rng, csr_rng in ELEMENT_KINDS if name in names]
        capacity = {}
        for name, _, _ in kinds:
            cap = slot_element_capacity(ds._elems[name][1], n_meshes)
            m = max_elements.get(name) if isinstance(max_elements, dict) else max_elements
            if m is not None:
                cap = max((operator.index(m) + 127) // 128 * 128, 128)
            if cap * int(ds._elems[name][0].shape[1]) >= _INT32_LIMIT:
                raise ValueError("MeshDataset.slot: {} {} have more corners than int32 indices hold".format(cap, name))
            capacity[name] = cap
        self.element_capacity = types.MappingProxyType(capacity)      # element kind -> capacity, fixed
        sizes, (g_rowptr_t, g_colidx_t, g_vals_t) = ds._slot_tables()
        elem_csr = {}
        if kinds:
            sizes, elem_csr = ds._slot_element_tables([name for name, _, _ in kinds])
        self._ds, self._sizes = ds, sizes
        self.device, self.K, self.n_meshes, self.V = ds.device, ds.K, n_meshes, v_cap
        self.entry_capacity = e_cap
        B, dev = n_meshes, ds.device
        # tail pieces no longer than the dataset's largest mesh: every gather grid is sized like ds.batch's
        pad_max = max(max((n + 127) // 128 * 128 for n in ds.n_rows), 128)
        self._tail = max(pad_max, -(-v_cap // (128 * B)) * 128)
        i32, i64, f32 = (dict(dtype=t, device=dev) for t in (torch.int32, torch.int64, torch.float32))
        self.ids = torch.zeros(B, **i64)
        self.status = torch.zeros(3, **i64)
        n_tiles = v_cap // 128
        (self._row_begin, self._tile_mesh, self._tb_rows, self._cta_begin, seg_begin, seg_rows, tile_seg) = (
            torch.zeros(n, **i32) for n in (B + 1, n_tiles, 2 * n_ctas, B + 1, B, B, n_tiles))
        self._static = {}
        self._n_ranges = N_SLOT_RANGES if kinds else N_RANGES
        self._table = torch.zeros(2 * B, self._n_ranges, 4, **i64)
        self._plan = _lib.dn_slot_plan(*(t.data_ptr() for t in (
            self._row_begin, self._tile_mesh, self._tb_rows, self._cta_begin, seg_begin, seg_rows, tile_seg,
            self._table, self.status)))
        self._n_ctas = n_ctas
        self.mass = torch.zeros(v_cap, **f32)
        self.evecs = torch.zeros(v_cap, ds.K, **f32)
        self.evals = torch.zeros(B, ds.K, **f32)
        rowptr, rowptr_t = torch.zeros(v_cap + 1, **i32), torch.zeros(v_cap + 1, **i32)
        colidx, colidx_t = torch.zeros(e_cap, **i32), torch.zeros(e_cap, **i32)
        vals, vals_t = torch.zeros(e_cap, 2, **f32), torch.zeros(e_cap, 2, **f32)
        g_rowptr, g_colidx, g_vals = ds._grad
        ent_max = max(ds._grad_nnz)
        COPY, ADD32 = _lib.GATHER_COPY, _lib.GATHER_ADD_I32
        part = lambda src, dst, op, width, rng, n, off=0: (_lib.dn_gather_part(src.data_ptr(), dst.data_ptr(), op,
                                                                                width, rng, off, n), dst)
        parts = [part(ds.mass, self.mass, COPY, 1, R_ROWS, self._tail),
                 part(ds.evecs, self.evecs, COPY, ds.K, R_ROWS, self._tail),
                 part(ds.evals, self.evals, COPY, ds.K, R_MESH, 1)]
        for (r_src, c_src, v_src), (r_dst, c_dst, v_dst) in (((g_rowptr, g_colidx, g_vals), (rowptr, colidx, vals)),
                                                              ((g_rowptr_t, g_colidx_t, g_vals_t),
                                                               (rowptr_t, colidx_t, vals_t))):
            parts += [part(r_src, r_dst, ADD32, 1, R_PTR, self._tail + 1, R_ENT),
                      part(c_src, c_dst, ADD32, 1, R_ENT, ent_max, R_ROWS),
                      part(v_src, v_dst, COPY, 2, R_ENT, ent_max)]
        # elements: corners offset by (and padded with) the mesh's first row, the CSR's row pointers placed like the
        # gradient CSR's and offset to the mesh's first CSR entry, its entries offset to the mesh's first element
        ADD64 = _lib.GATHER_ADD_I64
        self.faces = self.edges = None
        self.element_segments, self._elem_csr, self._elem_tail, self._elem_begin, kind_structs = {}, {}, {}, {}, []
        for name, rng, csr_rng in kinds:
            src, counts = ds._elems[name]
            cap, k = self.element_capacity[name], int(src.shape[1])
            pad_max = max(max((c + 127) // 128 * 128 for c in counts), 128)
            tail = self._elem_tail[name] = max(pad_max, -(-cap // (128 * B)) * 128)
            els = torch.zeros(cap, k, **i64)            # row 0 until the first fill: every corner names a row
            e_rowptr, e_ent = torch.zeros(v_cap + 1, **i32), torch.zeros(cap * k, **i32)
            begin, count, e_tile_seg = (torch.zeros(n, **i32) for n in (B + 1, B, cap // 128))
            src_rowptr, src_ent = elem_csr[name]
            if src.numel():
                parts += [part(src, els, ADD64, k, rng, tail, R_CORNER_OFF),
                          part(src_ent, e_ent, ADD32, 1, csr_rng, k * max(counts), rng)]
            parts.append(part(src_rowptr, e_rowptr, ADD32, 1, R_PTR, self._tail + 1, csr_rng))
            setattr(self, name, els)
            self._elem_csr[name] = (e_rowptr, e_ent)
            self.element_segments[name] = ops.Segments.wrap(cap, begin[:B], count, e_tile_seg)
            kind_structs.append(_lib.dn_slot_elements(cap, tail, k, rng, csr_rng, begin.data_ptr(), count.data_ptr(),
                                                      e_tile_seg.data_ptr()))
            self._elem_begin[name] = begin
        self._kinds = (_lib.dn_slot_elements * max(len(kind_structs), 1))(*kind_structs)
        self._n_kinds = len(kind_structs)
        parts = [p for p, dst in parts if dst.numel() > 0]
        self._parts = (_lib.dn_gather_part * len(parts))(*parts)
        self.gops = ops.GradOperators.from_csr(v_cap, rowptr, colidx, vals)
        self.gops._csr_t = (_lib.dn_csr(rowptr_t.data_ptr(), colidx_t.data_ptr(), vals_t.data_ptr(), e_cap),
                            rowptr_t, colidx_t, vals_t)
        self.desc = _lib.dn_mesh_batch(B, n_ctas, self._tile_mesh.data_ptr(), self._tb_rows.data_ptr(),
                                       self._cta_begin.data_ptr())
        self.segments = ops.Segments.wrap(v_cap, seg_begin, seg_rows, tile_seg)
        self.has_laplacian, self.lap = False, None
        self._mesh_ids = self._table[:B, R_MESH, 0]     # the filled ids; 0 for an invalid fill

    def fill(self, ids):
        """Plan and gather the batch of dataset meshes ``ids``: a CUDA int64 tensor of n_meshes ids (checked on the
        device), or a host list / CPU tensor (checked here first).  Two library launches whatever n_meshes is, no
        host synchronisation, no allocation (host ids: one pinned upload).  Returns the slot."""
        if torch.is_tensor(ids) and ids.device.type != "cpu":
            if ids.dtype != torch.int64 or tuple(ids.shape) != (self.n_meshes,) or ids.device != self.device:
                raise ValueError("BatchSlot.fill: device ids must be an int64 tensor of shape ({},) on {}, got {} of "
                                 "shape {} on {}".format(self.n_meshes, self.device, ids.dtype, tuple(ids.shape),
                                                         ids.device))
            if ids.data_ptr() != self.ids.data_ptr():
                self.ids.copy_(ids)
        else:
            ids = self._ds._ids(ids)
            if len(ids) != self.n_meshes:
                raise ValueError("BatchSlot.fill: {} ids for a slot of {} meshes".format(len(ids), self.n_meshes))
            ds = self._ds
            rows = sum((ds.n_rows[i] + 127) // 128 * 128 for i in ids)
            ents = sum(ds._grad_nnz[i] for i in ids)
            elems = {name: sum((ds._elems[name][1][i] + 127) // 128 * 128 for i in ids)
                     for name in self.element_capacity}
            if rows > self.V or ents > self.entry_capacity or \
                    any(e > self.element_capacity[name] for name, e in elems.items()):
                raise ValueError("BatchSlot.fill: the batch needs {}, more than the slot's capacity of {}".format(
                    self._amounts(rows, ents, elems), self._capacity_text()))
            self.ids.copy_(torch.tensor(ids, dtype=torch.int64).pin_memory(), non_blocking=True)
        with torch.cuda.device(self.device):
            st = ops._stream()
            _lib.call("dn_mesh_batch_plan_device_elements", self.ids, self.n_meshes, self._sizes,
                      int(self._sizes.shape[1]), self._ds.n_meshes, self._ds._sm, self.V, self.entry_capacity,
                      self._n_ctas, self._tail, self._n_ranges, C.byref(self._plan), self._kinds, self._n_kinds,
                      R_CORNER_OFF, st)
            if len(self._parts):
                _lib.call("dn_batch_gather", self._parts, len(self._parts), self._table, self._n_ranges,
                          2 * self.n_meshes, st)
        return self

    @staticmethod
    def _amounts(rows, ents, elems):
        words = ["{} rows".format(rows), "{} gradient entries".format(ents)]
        words += ["{} {}".format(e, name) for name, e in elems.items()]
        return ", ".join(words[:-1]) + " and " + words[-1]

    def _capacity_text(self):
        return self._amounts(self.V, self.entry_capacity, self.element_capacity)

    def check(self):
        """Raise if a fill since the last check had invalid device ids (IndexError) or exceeded the capacity
        (ValueError), naming the first offending position, and clear the status.  One device-to-host read."""
        kind, pos, bad = self.status.tolist()
        if kind:
            self.status.zero_()
        if kind == _ST_BAD_ID:
            raise IndexError("BatchSlot.fill: mesh id {} at position {} is outside the dataset's {} meshes".format(
                bad, pos, self._ds.n_meshes))
        if kind == _ST_OVER_CAPACITY:
            raise ValueError("BatchSlot.fill: the batch exceeds the slot's capacity of {} at position {}".format(
                self._capacity_text(), pos))

    def _static_out(self, what, src, shape):
        key = (what, src.data_ptr(), src.dtype, tuple(src.shape))
        out = self._static.get(key)
        if out is None:
            out = self._static[key] = torch.zeros(shape, dtype=src.dtype, device=self.device)
        return out

    def pack(self, t, rotations=None):
        """A dataset-layout float32 or int64 per-vertex tensor (V_total,) / (V_total, C) in the slot's layout, padding
        rows 0: one launch into a buffer that is the same tensor on every call with the same ``t``.  ``rotations``:
        (n_meshes, 3, 3) float32, one matrix per slot mesh, for float32 (V_total, 3) data, as in ``MeshDataset.pack``
        (one more launch; the rotated rows go to a buffer of their own, so ``pack(t)`` and ``pack(t, rotations=R)``
        do not overwrite each other)."""
        if isinstance(t, (list, tuple)):
            raise NotImplementedError("BatchSlot.pack takes one tensor in the dataset layout; per-mesh lists need the "
                                      "host layout of a MeshBatch")
        self._ds._check_pack(t, "BatchSlot.pack")
        _check_rotated(t, rotations, self, "BatchSlot.pack")
        out = self._static_out("pack" if rotations is None else "pack_rotated", t, (self.V,) + tuple(t.shape[1:]))
        t = t.contiguous()
        width = (t.shape[1] if t.dim() == 2 else 1) * (2 if t.dtype == torch.int64 else 1)
        if width:
            part = _lib.dn_gather_part(t.data_ptr(), out.data_ptr(), _lib.GATHER_COPY, width, R_ROWS, 0, self._tail)
            with torch.cuda.device(self.device):
                _lib.call("dn_batch_gather", C.byref(part), 1, self._table, self._n_ranges, 2 * self.n_meshes,
                          ops._stream())
        if rotations is not None:
            _rotate(out, self, rotations, out)
        return out

    def _element_kind(self, name, what):
        if name not in self.element_capacity:
            raise ValueError("BatchSlot.{}: the slot holds no {!r}: it holds {} (the elements every item of the "
                             "dataset carries)".format(what, name, sorted(self.element_capacity) or "none"))
        return dict((n, r) for n, r, _ in ELEMENT_KINDS)[name]

    def pack_elements(self, t, name):
        """A per-element float32 or int64 tensor (E_total,) / (E_total, C) in the dataset's element layout of kind
        ``name`` ('faces' or 'edges': every mesh's elements back to back, as its items list them), in the slot's
        element layout, padding elements 0: one launch into a buffer that is the same tensor on every call with the
        same ``t``.  Labels for forward_batch_nll of a 'faces' / 'edges' net."""
        rng = self._element_kind(name, "pack_elements")
        self._ds._check_pack(t, "BatchSlot.pack_elements", self._ds._elems[name][0].shape[0])
        out = self._static_out("pack_" + name, t, (self.element_capacity[name],) + tuple(t.shape[1:]))
        t = t.contiguous()
        width = (t.shape[1] if t.dim() == 2 else 1) * (2 if t.dtype == torch.int64 else 1)
        if width and t.numel():
            part = _lib.dn_gather_part(t.data_ptr(), out.data_ptr(), _lib.GATHER_COPY, width, rng, 0,
                                       self._elem_tail[name])
            with torch.cuda.device(self.device):
                _lib.call("dn_batch_gather", C.byref(part), 1, self._table, self._n_ranges, 2 * self.n_meshes,
                          ops._stream())
        return out

    def element_csr(self, name):
        """(rowptr int32 (V + 1), entries int32): the vertex -> element CSR of the filled batch's real elements of
        kind ``name``, in ops.element_csr's format on the slot's rows and element layout (ops.element_mean's ``csr``).
        Gathered at every fill into the same buffers."""
        self._element_kind(name, "element_csr")
        return self._elem_csr[name]

    def take(self, per_mesh):
        """``per_mesh[ids]`` (a per-mesh tensor of the dataset, e.g. whole-shape labels) into a buffer that is the same
        tensor on every call with the same ``per_mesh``."""
        if not torch.is_tensor(per_mesh) or per_mesh.dim() < 1 or per_mesh.shape[0] != self._ds.n_meshes or \
                per_mesh.device != self.device:
            raise ValueError("BatchSlot.take: expected a tensor of {} rows (one per dataset mesh) on {}, got {}".format(
                self._ds.n_meshes, self.device, (tuple(per_mesh.shape), per_mesh.device) if torch.is_tensor(per_mesh)
                else type(per_mesh)))
        out = self._static_out("take", per_mesh, (self.n_meshes,) + tuple(per_mesh.shape[1:]))
        torch.index_select(per_mesh, 0, self._mesh_ids, out=out)
        return out

    def _no_host_layout(self, what):
        raise NotImplementedError("BatchSlot.{}: a slot keeps no host copy of its layout (it is planned on the device "
                                  "at every fill); use ds.batch(ids) for per-mesh lists".format(what))

    @property
    def n_rows(self):
        self._no_host_layout("n_rows")

    @property
    def row_begin(self):
        self._no_host_layout("row_begin")

    def unpack(self, y):
        self._no_host_layout("unpack")

    def elem_counts(self, name):
        self._no_host_layout("elem_counts")


# ------------------------------------------------------------------------------------------------
# random rotations (the reference's xyz augmentation), per mesh of a batch or slot
# ------------------------------------------------------------------------------------------------
def rotation_from_uniforms(u, axis=None):
    """(n, 3, 3) float64 rotations from uniforms in [0, 1), with the reference's constructions (utils.py):
    ``axis=None``: u (n, 3), ``random_rotation_matrix`` (Graphics Gems III: a rotation by 2 pi u0 about z, then the
    Householder-type map (V V^T - I) with V from 2 pi u1 and 2 u2), uniform over SO(3);
    ``axis='y'``: u (n,) or (n, 1), ``random_rotate_points_y``'s rotation by 2 pi u about y.
    Torch ops only, on u's device."""
    u = u.to(torch.float64)
    two_pi = 2.0 * np.pi
    if axis == 'y':
        a = u.reshape(-1) * two_pi
        c, s = torch.cos(a), torch.sin(a)
        o, z = torch.ones_like(a), torch.zeros_like(a)
        return torch.stack([c, z, s, z, o, z, -s, z, c], -1).view(-1, 3, 3)
    if axis is not None:
        raise ValueError("rotation axis must be None (uniform over SO(3)) or 'y', got {!r}".format(axis))
    if u.dim() != 2 or u.shape[1] != 3:
        raise ValueError("rotation_from_uniforms: expected (n, 3) uniforms, got {}".format(tuple(u.shape)))
    theta, phi, z = u[:, 0] * two_pi, u[:, 1] * two_pi, u[:, 2] * 2.0
    r = torch.sqrt(z)
    V = torch.stack([torch.sin(phi) * r, torch.cos(phi) * r, torch.sqrt(2.0 - z)], -1)
    st, ct = torch.sin(theta), torch.cos(theta)
    o, zero = torch.ones_like(st), torch.zeros_like(st)
    Rz = torch.stack([ct, st, zero, -st, ct, zero, zero, zero, o], -1).view(-1, 3, 3)
    H = V.unsqueeze(-1) * V.unsqueeze(-2) - torch.eye(3, dtype=torch.float64, device=u.device)
    return (H.unsqueeze(-1) * Rz.unsqueeze(-3)).sum(-2)          # (V V^T - I) Rz


def random_rotations(n, axis=None, generator=None, device="cuda"):
    """(n, 3, 3) float32 random rotations, one per mesh, for ``pack(..., rotations=)``: the distributions of the
    reference's ``random_rotate_points`` (``axis=None``, uniform over SO(3) from 3 uniforms) and
    ``random_rotate_points_y`` (``axis='y'``, a uniform angle about y).  The same distributions, not the same random
    stream: the uniforms come from ``torch.rand`` on ``device`` (with ``generator`` if given) and the matrices are
    built with torch ops there (``rotation_from_uniforms``), so a step captured in a CUDA graph draws new rotations
    at every replay."""
    k = 1 if axis == 'y' else 3
    u = torch.rand(int(n), k, generator=generator, device=device, dtype=torch.float64)
    return rotation_from_uniforms(u, axis).to(torch.float32)


def _check_rotated(t, rotations, batch, what):
    if rotations is None:
        return
    if t.dtype != torch.float32 or t.dim() != 2 or t.shape[1] != 3:
        raise ValueError("{}: rotations apply to float32 (V_total, 3) data, got {} of shape {}".format(
            what, t.dtype, tuple(t.shape)))
    if not torch.is_tensor(rotations) or tuple(rotations.shape) != (batch.n_meshes, 3, 3) or \
            rotations.dtype != torch.float32 or rotations.device != batch.device:
        raise ValueError("{}: rotations must be a float32 ({}, 3, 3) tensor on {}, got {}".format(
            what, batch.n_meshes, batch.device, (tuple(rotations.shape), rotations.dtype, rotations.device)
            if torch.is_tensor(rotations) else type(rotations)))
    if rotations.requires_grad:
        raise ValueError("{}: rotations are data; got a tensor that requires grad".format(what))


def _rotate(x, batch, R, out):
    with torch.cuda.device(batch.device):
        _lib.call("dn_rotate_rows", x, batch.V, R.contiguous(), batch.n_meshes, batch._tile_mesh, out, ops._stream())
    return out


def rotate_rows(x, batch, rotations):
    """(V, 3) float32 rows ``x`` in the layout of ``batch`` (a ``MeshBatch`` or ``BatchSlot``) rotated per mesh:
    ``x_b @ R_b`` on the rows of mesh b (``dn_rotate_rows``, one launch; the mesh of a row comes from the layout's
    tile table, so no host layout is needed).  Padding rows, 0 in ``x``, stay 0.  Data only (no autograd)."""
    ops._require_cuda(x)
    if x.dtype != torch.float32 or tuple(x.shape) != (batch.V, 3):
        raise ValueError("rotate_rows: expected float32 ({}, 3) rows in the batch layout, got {} of shape {}".format(
            batch.V, x.dtype, tuple(x.shape)))
    _check_rotated(x, rotations, batch, "rotate_rows")
    if x.requires_grad:
        raise ValueError("rotate_rows rotates data; got rows that require grad")
    return _rotate(x.contiguous(), batch, rotations, torch.empty_like(x))


def block_forward_batched_raw(batch, x_in, time, A_re, A_im, weights, biases, with_features, head=None):
    """dn_block_fwd_ex with a batch descriptor: one DiffusionNetBlock (eval) over every mesh of ``batch`` (x_in in the batch
    layout).  ``head``: see ops.block_forward_raw."""
    x_in = ops._f32c(x_in)
    if x_in.shape[0] != batch.V:
        raise ValueError("x_in is not in this batch's layout ({} rows, expected {})".format(x_in.shape[0], batch.V))
    return ops.block_forward_raw(x_in, batch.mass, batch.evals, batch.evecs, batch.gops, time, A_re, A_im, weights, biases,
                                 with_features, head=head, batch_desc=batch.desc)
