"""MeshDataset: a device-resident dataset from which any batch of meshes is gathered on the GPU in one launch
(dn_batch_gather), and MeshBatch(items), which is now that dataset gathered in order.

MeshBatch itself uses the gather, so the layout gold here is the host concatenation MeshBatch used to do, restated in
numpy: every mesh start rounded up to a 128-row tile, zero padding rows, empty padding CSR rows, columns offset by the
mesh's row start, dn_mesh_batch_plan's CTA split.  The CPU tests check the size-only table builder against it (with a
numpy emulation of the kernel's two routines); the GPU tests compare every array of ds.batch(ids) and of
MeshBatch(items[ids]) with it bitwise, then the training routes, a shuffled run, the no-synchronisation contract and the
refusals."""
import copy
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle as O  # noqa: E402  (checker only)

import diffusion_net_b200 as dn  # noqa: E402
from diffusion_net_b200 import batch as B  # noqa: E402

gpu = pytest.mark.gpu
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
MAX_CTAS = 1024


# ---- the parent's host layout, restated ---------------------------------------------------------------------------
def _plan_gold(n_rows, sm):
    """dn_mesh_batch_plan restated: row_begin, tile_mesh (max(V / 128, 1)), tb_rows (2 n_ctas), cta_begin, n_ctas."""
    nb = len(n_rows)
    row_begin = [0]
    for v in n_rows:
        row_begin.append(row_begin[-1] + (v + 127) // 128 * 128)
    V = row_begin[-1]
    tile_mesh = np.zeros(max(V // 128, 1), np.int32)
    for b in range(nb):
        tile_mesh[row_begin[b] // 128:row_begin[b + 1] // 128] = b
    chunks = [(v + 15) // 16 for v in n_rows]
    total = sum(chunks)
    tb, cta_begin = [], []
    for b, c in enumerate(chunks):
        want = max((c * sm + total // 2) // total if total > 0 else 1, 1)
        if want > c > 0:
            want = c
        if len(tb) + want + (nb - 1 - b) > MAX_CTAS:
            want = 1
        cta_begin.append(len(tb))
        per = -(-c // want) if c > 0 else 0
        if per > 0:
            want = -(-c // per)
        end = row_begin[b] + n_rows[b]
        for k in range(want):
            rb = row_begin[b] + k * per * 16
            tb.append((min(rb, end), min(rb + per * 16, end)))
    cta_begin.append(len(tb))
    return (np.asarray(row_begin, np.int32), tile_mesh, np.asarray(tb, np.int32).reshape(-1),
            np.asarray(cta_begin, np.int32), len(tb))


def _csr_gold(csrs, row_begin, n_rows):
    """Block-diagonal CSR of per-mesh (rowptr, colidx, vals (nnz, 2)): padding rows empty, columns + the mesh's start."""
    rp, cols, vals, nnz = [np.zeros(1, np.int64)], [], [], 0
    for (rowptr, colidx, v), r0, n, r1 in zip(csrs, row_begin[:-1], n_rows, row_begin[1:]):
        rp.append(rowptr[1:] + nnz)
        rp.append(np.full(r1 - r0 - n, rowptr[-1] + nnz, np.int64))
        cols.append(colidx.astype(np.int64) + r0)
        vals.append(v.reshape(-1, 2))
        nnz += int(rowptr[-1])
    return (np.concatenate(rp).astype(np.int32), np.concatenate(cols).astype(np.int32),
            np.concatenate(vals).astype(np.float32))


def _layout_gold(meshes, ids, sm):
    """Every array and table of the batch of host meshes ``meshes[ids]`` as the host concatenation built it."""
    ms = [meshes[i] for i in ids]
    n_rows = [m["V"] for m in ms]
    row_begin, tile_mesh, tb_rows, cta_begin, n_ctas = _plan_gold(n_rows, sm)
    V, K = int(row_begin[-1]), ms[0]["K"]
    out = dict(row_begin=row_begin, V=V, n_ctas=n_ctas, tile_mesh=tile_mesh, tb_rows=tb_rows, cta_begin=cta_begin)
    out["mesh_rows"] = np.stack([row_begin[:-1], row_begin[:-1] + np.asarray(n_rows)], 1).reshape(-1).astype(np.int32)
    tile_seg = np.full((V + 127) // 128, -1, np.int32)
    for b, (r0, n) in enumerate(zip(row_begin[:-1], n_rows)):
        tile_seg[r0 // 128:(r0 + n + 127) // 128] = b
    out["seg"] = (row_begin[:-1].copy(), np.asarray(n_rows, np.int32), tile_seg)
    out["mass"] = np.zeros(V, np.float32)
    out["evecs"] = np.zeros((V, K), np.float32)
    out["evals"] = np.zeros((len(ids), K), np.float32)
    for b, (m, r0) in enumerate(zip(ms, row_begin)):
        out["mass"][r0:r0 + m["V"]] = m["mass"]
        if K:
            out["evecs"][r0:r0 + m["V"]] = m["evecs"]
            out["evals"][b] = m["evals"]
    out["grad"] = _csr_gold([m["grad"] for m in ms], row_begin, n_rows)
    out["lap"] = _csr_gold([m["lap"] for m in ms], row_begin, n_rows) if ms[0]["lap"] is not None else None
    for name in ("faces", "edges"):
        out[name] = np.concatenate([m[name] + r0 for m, r0 in zip(ms, row_begin)], 0)
    return out


# ---- synthetic meshes ------------------------------------------------------------------------------------------------
def _coo(V, rs, deg_hi=8, empty=()):
    deg = rs.randint(1, deg_hi, V)
    deg[list(empty)] = 0
    rows = np.repeat(np.arange(V), deg)
    return torch.from_numpy(np.stack([rows, rs.randint(0, V, rows.size)]))


def _mesh(V, K, seed, lap=True, empty=(), no_grad_entries=False):
    """A mesh item (CUDA tensors) and its host arrays: random values on random patterns (the layout does not care
    what they mean), gradient rows ``empty`` without entries, or no gradient entries at all."""
    rs = np.random.RandomState(seed)
    g = torch.Generator().manual_seed(seed)
    idx = _coo(V, rs, empty=empty) if not no_grad_entries else torch.zeros(2, 0, dtype=torch.int64)
    gX = torch.sparse_coo_tensor(idx, torch.randn(idx.shape[1], generator=g), (V, V)).coalesce()
    gY = torch.sparse_coo_tensor(gX.indices(), torch.randn(gX.indices().shape[1], generator=g), (V, V)).coalesce()
    item = dict(mass=(torch.rand(V, generator=g, dtype=torch.float64) + 0.5).cuda(), gradX=gX.cuda(), gradY=gY.cuda(),
                faces=torch.from_numpy(rs.randint(0, V, (2 * V + 1, 3))),
                edges=torch.from_numpy(rs.randint(0, V, (3 * V, 2))))
    if K:
        item["evals"] = torch.rand(K, generator=g).cuda()
        item["evecs"] = torch.randn(V, K, generator=g).cuda()
    if lap:
        li = _coo(V, rs)
        item["L"] = torch.sparse_coo_tensor(li, torch.randn(li.shape[1], generator=g), (V, V)).coalesce().cuda()

    def csr(A, Bm=None):
        i = A.indices().cpu().numpy()
        rowptr = np.zeros(V + 1, np.int64)
        np.add.at(rowptr, i[0] + 1, 1)
        vb = Bm.values().cpu().numpy() if Bm is not None else np.zeros(i.shape[1], np.float32)
        return np.cumsum(rowptr), i[1], np.stack([A.values().cpu().numpy(), vb], 1).astype(np.float32)

    host = dict(V=V, K=K, mass=item["mass"].float().cpu().numpy(), grad=csr(gX, gY),
                lap=csr(item["L"]) if lap else None, faces=item["faces"].numpy(), edges=item["edges"].numpy())
    if K:
        host["evals"], host["evecs"] = item["evals"].cpu().numpy(), item["evecs"].cpu().numpy()
    return item, host


def _prepared(item):
    """The same item with prepared operators (GradOperators under 'gradX', a LaplacianCSR under 'L')."""
    out = dict(item)
    out["gradX"] = dn.ops.GradOperators(item["gradX"], item["gradY"])
    out.pop("gradY")
    if "L" in item:
        out["L"] = dn.ops.LaplacianCSR(item["L"])
    return out


RAGGED = [1, 127, 128, 129, 3000, 40, 200]


def _meshes(sizes, K, lap=True, seed=0):
    out = []
    for i, V in enumerate(sizes):
        empty = range(0, V, 3) if i == 5 else ()              # a mesh with empty gradient rows
        out.append(_mesh(V, K, seed + i, lap=lap, empty=empty, no_grad_entries=(i == 6)))
    return [o[0] for o in out], [o[1] for o in out]


ID_SETS = [list(range(len(RAGGED))), [6, 4, 4, 1, 0, 2, 2, 5, 3, 4], list(reversed(range(len(RAGGED)))), [4]]


# ---- CPU: the size-only table builder -------------------------------------------------------------------------------
def _emulate(src, n_dst, op, width, rng, table, off_rng=0):
    """dn_batch_gather's routines on the host: per batch mesh, units [0, min(n, n_dst)) copied (op 'copy') or plus the
    mesh's offset (op 'add'), the rest of [0, n_dst) padding (0, or offset + count)."""
    dst = np.full(n_dst * width, -7, dtype=src.dtype)
    for b in range(table.shape[0]):
        s0, d0, n, nd = (int(v) for v in table[b, rng])
        k = min(n, nd) * width
        if op == "copy":
            seg, pad = src[s0 * width:s0 * width + k], 0
        else:
            off = table[b, off_rng, 1]
            seg, pad = src[s0 * width:s0 * width + k] + off, off + table[b, off_rng, 2]
        dst[d0 * width:d0 * width + k] = seg
        dst[d0 * width + k:(d0 + nd) * width] = pad
    return dst


def _dataset_host(meshes):
    cat = lambda f: np.concatenate([f(m) for m in meshes])
    return dict(mass=cat(lambda m: m["mass"]), evecs=cat(lambda m: m["evecs"].reshape(-1)),
                evals=cat(lambda m: m["evals"]), rowptr=cat(lambda m: m["grad"][0].astype(np.int32)),
                colidx=cat(lambda m: m["grad"][1].astype(np.int32)), vals=cat(lambda m: m["grad"][2].reshape(-1)),
                faces=cat(lambda m: m["faces"].reshape(-1)), edges=cat(lambda m: m["edges"].reshape(-1)))


def _host_meshes(sizes, K, seed=0):
    """Host-only meshes with the same structure as _mesh (no torch sparse, no GPU)."""
    out = []
    for i, V in enumerate(sizes):
        rs = np.random.RandomState(seed + i)
        deg = rs.randint(0, 8, V)
        rowptr = np.concatenate([[0], np.cumsum(deg)])
        nnz = int(rowptr[-1])
        out.append(dict(V=V, K=K, mass=rs.rand(V).astype(np.float32), evals=rs.rand(K).astype(np.float32),
                        evecs=rs.randn(V, K).astype(np.float32),
                        grad=(rowptr, rs.randint(0, V, nnz), rs.randn(nnz, 2).astype(np.float32)), lap=None,
                        faces=rs.randint(0, V, (2 * V + 1, 3)), edges=rs.randint(0, V, (V, 2))))
    return out


@pytest.mark.parametrize("ids", ID_SETS)
def test_batch_tables_against_the_host_layout(ids):
    """batch_tables (sizes only) gives the host layout's tables, and its gather table, applied by a numpy emulation of
    the kernel's two routines to the concatenated dataset, gives every array of the host layout."""
    K, sm = 4, 132
    meshes = _host_meshes(RAGGED, K)
    sizes = dict(n_rows=[m["V"] for m in meshes], n_ent=[int(m["grad"][0][-1]) for m in meshes],
                 n_faces=[len(m["faces"]) for m in meshes], n_edges=[len(m["edges"]) for m in meshes])
    t = B.batch_tables(ids, sm_count=sm, **sizes)
    gold = _layout_gold(meshes, ids, sm)
    for k in ("row_begin", "tile_mesh", "tb_rows", "cta_begin", "mesh_rows"):
        assert t[k].dtype == np.int32 and np.array_equal(t[k], gold[k]), k
    assert t["V"] == gold["V"] and t["n_ctas"] == gold["n_ctas"]
    for got, want in zip((t["seg_begin"], t["seg_rows"], t["tile_seg"]), gold["seg"]):
        assert np.array_equal(got, want)
    ds, tab, V, nb = _dataset_host(meshes), t["table"], gold["V"], len(ids)
    F, E = len(gold["faces"]), len(gold["edges"])
    assert np.array_equal(_emulate(ds["mass"], V, "copy", 1, B.R_ROWS, tab), gold["mass"])
    assert np.array_equal(_emulate(ds["evecs"], V, "copy", K, B.R_ROWS, tab), gold["evecs"].reshape(-1))
    assert np.array_equal(_emulate(ds["evals"], nb, "copy", K, B.R_MESH, tab), gold["evals"].reshape(-1))
    rowptr, colidx, vals = gold["grad"]
    assert np.array_equal(_emulate(ds["rowptr"], V + 1, "add", 1, B.R_PTR, tab, B.R_ENT), rowptr)
    assert np.array_equal(_emulate(ds["colidx"], t["nnz"], "add", 1, B.R_ENT, tab, B.R_ROWS), colidx)
    assert np.array_equal(_emulate(ds["vals"], t["nnz"], "copy", 2, B.R_ENT, tab), vals.reshape(-1))
    assert np.array_equal(_emulate(ds["faces"], F, "add", 3, B.R_FACES, tab, B.R_ROWS), gold["faces"].reshape(-1))
    assert np.array_equal(_emulate(ds["edges"], E, "add", 2, B.R_EDGES, tab, B.R_ROWS), gold["edges"].reshape(-1))


def test_batch_tables_refuse_what_int32_cannot_index():
    """A batch past int32 is refused from the sizes alone: rows (as dn_mesh_batch_plan refuses them, 'unsupported'),
    gradient entries, and more than 1024 meshes.  A dataset may be larger: only the batch counts."""
    big = 2 ** 30
    with pytest.raises(RuntimeError, match="unsupported"):
        B.batch_tables([0, 1], n_rows=[big, big], n_ent=[1, 1])
    B.batch_tables([0], n_rows=[big, big], n_ent=[1, 1])                      # one of them fits
    with pytest.raises(ValueError, match="more than int32"):
        B.batch_tables([0, 1], n_rows=[10, 10], n_ent=[big, big])
    t = B.batch_tables([1, 2], n_rows=[10, 10, 10], n_ent=[2 ** 33, big - 1, big])
    assert t["table"][0, B.R_ENT, 0] == 2 ** 33                                # int64 dataset offsets
    with pytest.raises(RuntimeError, match="unsupported"):
        B.batch_tables([0] * 1025, n_rows=[3], n_ent=[3])


def test_gather_kernel_does_not_spill(tmp_path):
    if shutil.which(NVCC) is None and not os.path.exists(NVCC):
        pytest.skip("needs nvcc")
    flags = [f for f in dn._lib.NVCC_FLAGS if f != "-shared"]
    cmd = [NVCC] + flags + ["-Xptxas", "-v", "-c", os.path.join(dn._lib._CSRC, "dn_batch_gather.cu"), "-o",
                            str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [l for l in (r.stdout + r.stderr).splitlines() if "spill stores" in l]
    assert len(lines) == 1
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", lines[0])
    assert m and m.groups() == ("0", "0", "0"), lines[0]


# ---- GPU: every array bitwise against the host layout ---------------------------------------------------------------
@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    dn._lib.load()
    yield torch.device("cuda")
    dn.set_engine("tc3x")


def _launches():
    return dn._lib.load().dn_kernel_launch_count()


def _bits(t):
    a = t.detach().cpu().numpy()
    return a.view(np.int32) if a.dtype == np.float32 else a


def _same(t, want):
    a, w = _bits(t), np.ascontiguousarray(want)
    w = w.view(np.int32) if w.dtype == np.float32 else w
    return a.shape == w.shape and a.dtype == w.dtype and np.array_equal(a, w)


def _check_layout(mb, gold):
    assert mb.row_begin == [int(v) for v in gold["row_begin"]] and mb.V == gold["V"]
    assert mb.desc.n_tb_ctas == gold["n_ctas"] and mb.desc.n_meshes == len(mb.n_rows)
    for name, got in (("tile_mesh", mb._tile_mesh), ("tb_rows", mb._tb_rows), ("cta_begin", mb._cta_begin),
                      ("mesh_rows", mb._mesh_rows)):
        assert _same(got, gold[name]), name
    for got, want in zip((mb.segments.begin, mb.segments.rows, mb.segments.tile_seg), gold["seg"]):
        assert _same(got, want)
    assert mb.segments.n_seg == mb.n_meshes and mb.segments.V == mb.V
    for name in ("mass", "evecs", "evals", "faces", "edges"):
        assert _same(getattr(mb, name), gold[name]), name
    for ops_, want in ((mb.gops, gold["grad"]), (mb.lap, gold["lap"])):
        if want is None:
            assert ops_ is None
            continue
        _, rowptr, colidx, vals = ops_.csr
        nnz = ops_.nnz
        assert nnz == len(want[1]) and ops_.V == mb.V
        assert _same(rowptr, want[0]) and _same(colidx[:nnz], want[1]) and _same(vals[:2 * nnz].view(-1, 2), want[2])


@gpu
@pytest.mark.parametrize("prepared", [False, True])
def test_batch_layout_against_the_host_layout(cuda, prepared):
    """Ragged sizes (V = 1, 127, 128, 129, 3000, a mesh with empty gradient rows, one with no gradient entries), ids
    with repeats, reversed and a single mesh, faces and edges, items as raw COO and as prepared operators: every array
    and table of ds.batch(ids) and of MeshBatch(items[ids]) is bitwise the host layout."""
    items, host = _meshes(RAGGED, 16)
    if prepared:
        items = [_prepared(it) for it in items]
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    ds = dn.MeshDataset(items)
    assert ds.n_meshes == len(items) and ds.n_rows == RAGGED and ds.K == 16 and ds.V == sum(RAGGED)
    for ids in ID_SETS:
        gold = _layout_gold(host, ids, sm)
        for mb in (ds.batch(ids), dn.MeshBatch([items[i] for i in ids])):
            _check_layout(mb, gold)
            assert mb.elem_counts("faces") == [len(host[i]["faces"]) for i in ids]
            assert mb.elem_counts("edges") == [len(host[i]["edges"]) for i in ids]
            assert mb.n_rows == [RAGGED[i] for i in ids] and mb.K == 16 and mb.has_laplacian


@gpu
def test_implicit_only_dataset_layout(cuda):
    """K = 0 with L: no eigenpairs in the layout, the Laplacian gathered on first use (one more launch)."""
    items, host = _meshes(RAGGED, 0)
    for it in items:
        dn.ops.prepare_laplacian(it["L"])                     # memoised: the first use below only gathers
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    ds = dn.MeshDataset(items)
    ids = ID_SETS[1]
    mb = ds.batch(ids)
    assert mb._lap is None                                    # not built before first use
    torch.cuda.synchronize()
    l0 = _launches()
    lap = mb.lap
    assert _launches() - l0 == 1 and mb.lap is lap
    _check_layout(mb, _layout_gold(host, ids, sm))
    assert mb.K == 0 and mb.evecs.shape == (mb.V, 0) and mb.evals.shape == (len(ids), 0)


@gpu
def test_laplacian_shape_error_is_raised_at_first_use(cuda):
    items, _ = _meshes([40, 50], 4)
    items[1]["L"] = items[0]["L"]
    mb = dn.MeshBatch(items)
    with pytest.raises(ValueError, match="mesh 1 has 50 vertices but its L is not a \\(50, 50\\) Laplacian"):
        mb.lap
    ds = dn.MeshDataset(items)
    b = ds.batch([0])
    with pytest.raises(ValueError, match="mesh 1 has 50 vertices"):
        b.lap


# ---- GPU: the routes, bitwise against MeshBatch -----------------------------------------------------------------------
SHAPES = [(12, 11), (36, 50), (8, 10), (16, 8), (20, 13)]


def _net_meshes(K, seed=0, lap=False):
    out = []
    for i, (n, m) in enumerate(SHAPES):
        mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=seed + i, device="cuda")
        _, faces = dn.synthetic.torus_mesh(n, m, seed=seed + i)
        it = dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY, faces=faces.cuda())
        if lap:
            Ls = (L + L.t()).coalesce()                           # any symmetric pattern; made SPD below
            d = torch.sparse_coo_tensor(torch.arange(n * m).repeat(2, 1), torch.full((n * m,), 20.0), L.shape)
            it["L"] = (Ls.abs() + d.cuda()).coalesce()
        out.append(it)
    return out


def _spectral_net(C_out=5, outputs_at="vertices", seed=0):
    torch.manual_seed(seed)
    net = dn.DiffusionNet(C_in=16, C_out=C_out, C_width=64, N_block=2, dropout=False,
                          outputs_at=outputs_at).cuda().train()
    with torch.no_grad():
        for n_, p_ in net.named_parameters():
            if n_.endswith("diffusion_time"):
                p_.uniform_(1e-3, 0.3)
    return net


def _features(ds, C_in=16, C_out=5, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(ds.V, C_in, generator=g).cuda(), torch.randint(0, C_out, (ds.V,), generator=g).cuda()


def _run(net, fn):
    """(outputs, parameter gradients, input gradient) of fn(net, x_requires_grad)."""
    net.zero_grad(set_to_none=True)
    out, x = fn(net)
    out = out if isinstance(out, (list, tuple)) else [out]
    sum(o.float().sum() for o in out if o.is_floating_point()).backward()
    return [o.detach().clone() for o in out], {n_: p_.grad.clone() for n_, p_ in net.named_parameters()}, x.grad.clone()


def _assert_bitwise(a, b):
    (oa, ga, xa), (ob, gb, xb) = a, b
    assert len(oa) == len(ob) and all(torch.equal(u, v) for u, v in zip(oa, ob))
    assert all(torch.equal(ga[k], gb[k]) for k in ga), [k for k in ga if not torch.equal(ga[k], gb[k])]
    assert torch.equal(xa, xb)


@gpu
@pytest.mark.parametrize("engine", ["tc3x", "bf16"])
def test_routes_bitwise_equal_to_meshbatch(cuda, engine):
    """forward_batch (inference and autograd), forward_batch_nll (vertices, faces), forward_batch_global_nll and an
    implicit net's forward_batch on ds.batch(ids) and on MeshBatch(items[ids]): outputs, parameter and input
    gradients bitwise equal."""
    dn.set_engine(engine)
    try:
        items = _net_meshes(64, lap=True)
        ds = dn.MeshDataset(items)
        ids = [3, 1, 1, 4, 0]
        X, Y = _features(ds)
        batches = (ds.batch(ids), dn.MeshBatch([items[i] for i in ids]))
        xs = [ds.pack(X, batches[0])] * 2                      # the layouts are equal (test_batch_layout_...)
        labels = [batches[0].unpack(ds.pack(Y, batches[0]))] * 2

        def per_route(make_net, call):
            res = []
            for b, x0, lab in zip(batches, xs, labels):
                net = make_net()
                res.append(_run(net, lambda n_: call(n_, b, x0.clone().requires_grad_(True), lab)))
            _assert_bitwise(*res)

        def fwd(n_, b, x, lab):
            return n_.forward_batch(b, x), x
        per_route(lambda: _spectral_net(), fwd)
        with torch.no_grad():
            outs = [_spectral_net().eval().forward_batch(b, x) for b, x in zip(batches, xs)]
        assert all(torch.equal(u, v) for u, v in zip(*outs))

        def nll(n_, b, x, lab):
            return n_.forward_batch_nll(b, x, lab)[0], x
        per_route(lambda: _spectral_net(), nll)

        def nll_faces(n_, b, x, lab):
            g = torch.Generator().manual_seed(3)
            fl = [torch.randint(0, 5, (c,), generator=g).cuda() for c in b.elem_counts("faces")]
            return n_.forward_batch_nll(b, x, fl)[0], x
        per_route(lambda: _spectral_net(outputs_at="faces"), nll_faces)

        def global_nll(n_, b, x, lab):
            return n_.forward_batch_global_nll(b, x, torch.tensor([i % 4 for i in ids]).cuda(),
                                               label_smoothing=0.1)[0], x
        per_route(lambda: _spectral_net(C_out=4, outputs_at="global_mean"), global_nll)

        def implicit_net():
            torch.manual_seed(1)
            net = dn.DiffusionNet(C_in=16, C_out=5, C_width=32, N_block=2, dropout=False,
                                  diffusion_method="implicit_dense").cuda().train()
            with torch.no_grad():
                for n_, p_ in net.named_parameters():
                    if n_.endswith("diffusion_time"):
                        p_.uniform_(1e-3, 0.05)
            return net
        per_route(implicit_net, fwd)
    finally:
        dn.set_engine("tc3x")


@gpu
def test_shuffled_run_against_the_per_mesh_loop(cuda):
    """Several SGD steps over ds.batch of a shuffled permutation; at every step the batch route's gradients match the
    per-mesh loop's over the same meshes from the same parameters (test_gpu_batch_train's tc3x bound)."""
    dn.set_engine("tc3x")
    items = _net_meshes(64, seed=10)
    ds = dn.MeshDataset(items)
    X, Y = _features(ds, seed=1)
    net = _spectral_net(seed=2)
    opt = torch.optim.SGD(net.parameters(), lr=1e-2)
    g = torch.Generator().manual_seed(5)
    steps = 0
    for epoch in range(2):
        for ids in torch.randperm(len(items), generator=g).split(2):
            ids = ids.tolist()
            b = ds.batch(ids)
            ref = copy.deepcopy(net)
            ref.zero_grad(set_to_none=True)
            loss_ref = 0
            for i in ids:
                r0, n = ds.row_begin[i], ds.n_rows[i]
                it = items[i]
                loss_ref = loss_ref + ref.forward_nll(X[r0:r0 + n], it["mass"], evals=it["evals"], evecs=it["evecs"],
                                                      gradX=it["gradX"], gradY=it["gradY"], labels=Y[r0:r0 + n])[0]
            loss_ref.backward()
            opt.zero_grad(set_to_none=True)
            losses, _ = net.forward_batch_nll(b, ds.pack(X, b), b.unpack(ds.pack(Y, b)))
            losses.sum().backward()
            assert O.rel_err(losses.sum().item(), loss_ref.item()) < 1e-5
            for (name, p_), q_ in zip(net.named_parameters(), ref.parameters()):
                assert O.rel_err(p_.grad.cpu().numpy(), q_.grad.cpu().numpy()) < 1e-4, (steps, name)
            opt.step()
            steps += 1
    assert steps == 6


# ---- GPU: no host synchronisation, one launch --------------------------------------------------------------------------
@gpu
def test_batch_and_pack_do_not_synchronise(cuda):
    items = _net_meshes(64, lap=True)
    for it in items:
        dn.ops.prepare_laplacian(it["L"])                     # memoised: b.lap below only gathers
    ds = dn.MeshDataset(items)
    X, Y = _features(ds)
    ids = [4, 0, 2, 2]
    ds.pack(Y, ds.batch(ids)).sum().item()                    # warm the caching allocators
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        l0 = _launches()
        b = ds.batch(ids)
        l1 = _launches()
        x = ds.pack(X, b)
        lab = ds.pack(Y, b)
        l2 = _launches()
        b.lap
        l3 = _launches()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert (l1 - l0, l2 - l1, l3 - l2) == (1, 2, 1)
    assert x.shape == (b.V, 16) and lab.shape == (b.V,) and lab.dtype == torch.int64
    for k, i in enumerate(ids):
        r0, n, s0 = b.row_begin[k], b.n_rows[k], ds.row_begin[i]
        assert torch.equal(x[r0:r0 + n], X[s0:s0 + n]) and torch.equal(lab[r0:r0 + n], Y[s0:s0 + n])
    pad = torch.ones(b.V, dtype=torch.bool, device="cuda")
    for k in range(len(ids)):
        pad[b.row_begin[k]:b.row_begin[k] + b.n_rows[k]] = False
    assert bool((x[pad] == 0).all()) and bool((lab[pad] == 0).all())
    # the call returns while earlier work is still running on the stream
    torch.cuda.synchronize()
    torch.cuda._sleep(50_000_000)                              # tens of milliseconds at H100 clocks
    ev = torch.cuda.Event()
    ev.record()
    b2 = ds.batch(ids)
    assert not ev.query(), "ds.batch waited for the device"
    torch.cuda.synchronize()
    assert torch.equal(b2.mass, b.mass) and torch.equal(b2.gops.csr[2], b.gops.csr[2])


@gpu
def test_refusals_before_any_launch(cuda):
    items = _net_meshes(64)
    ds = dn.MeshDataset(items)
    X, _ = _features(ds)
    b = ds.batch([0, 1])
    other = dn.MeshDataset(items[:2]).batch([0, 1])
    torch.cuda.synchronize()
    l0 = _launches()
    with pytest.raises(ValueError, match="at least one"):
        ds.batch([])
    with pytest.raises(IndexError, match="outside"):
        ds.batch([0, len(items)])
    with pytest.raises(IndexError, match="outside"):
        ds.batch([-1])
    with pytest.raises(ValueError, match="host"):
        ds.batch(torch.tensor([0, 1], device="cuda"))
    with pytest.raises(TypeError):
        ds.batch(torch.tensor([0.0, 1.0]))
    with pytest.raises(RuntimeError, match="unsupported"):
        ds.batch([0] * 1025)
    with pytest.raises(ValueError, match="dataset layout"):
        ds.pack(X[:-1], b)
    with pytest.raises(ValueError, match="dataset layout"):
        ds.pack(X.double(), b)
    with pytest.raises(ValueError, match="requires grad"):
        ds.pack(X.clone().requires_grad_(True), b)
    with pytest.raises(ValueError, match="not drawn from this dataset"):
        ds.pack(X, other)
    assert _launches() == l0
    assert ds.batch(torch.tensor([1, 0])).n_rows == [items[1]["mass"].shape[0], items[0]["mass"].shape[0]]


@gpu
def test_malformed_items_are_refused_before_any_copy_or_launch(cuda):
    """Every per-mesh array must have its mesh's row count (the dataset places a mesh's rows by its mass alone): an
    evecs with other rows than the mass, a 2-D mass, evals of another shape and gradient operators of another size are
    refused by MeshBatch and MeshDataset alike, before anything is copied or launched."""
    items = _net_meshes(64)
    bad = []
    it = dict(items[2]); it["evecs"] = it["evecs"][:-1]
    bad.append((it, "evecs of shape"))
    it = dict(items[4]); it["evecs"] = torch.cat([it["evecs"], it["evecs"][:3]])
    bad.append((it, "evecs of shape"))
    it = dict(items[1]); it["mass"] = it["mass"][:, None]
    bad.append((it, "mass must be 1-D"))
    it = dict(items[3]); it["evals"] = it["evals"][None]
    bad.append((it, "eigenpairs"))
    it = dict(items[0]); it["gradX"], it["gradY"] = items[1]["gradX"], items[1]["gradY"]
    bad.append((it, "gradient operators of shape"))
    it = dict(items[0]); it["gradX"] = dn.ops.prepare_operators(items[1]["gradX"], items[1]["gradY"])
    bad.append((it, "gradient operators of shape"))
    torch.cuda.synchronize()
    l0 = _launches()
    for it, msg in bad:
        for make in (dn.MeshBatch, dn.MeshDataset):
            with pytest.raises(ValueError, match=msg):
                make(items[:-1] + [it])
    assert _launches() == l0


@gpu
def test_pack_of_zero_columns_and_laplacian_kept_once(cuda):
    """ds.pack of a (V_total, 0) tensor gives the (V, 0) result without a launch; a MeshBatch(items) that built its
    Laplacian no longer holds the dataset-layout copy it was gathered from (a ds.batch keeps the shared dataset's)."""
    items = _net_meshes(64, lap=True)
    ds = dn.MeshDataset(items)
    b = ds.batch([2, 0])
    torch.cuda.synchronize()
    l0 = _launches()
    out = ds.pack(torch.zeros(ds.V, 0, device="cuda"), b)
    assert out.shape == (b.V, 0) and _launches() == l0
    mb = dn.MeshBatch(items)
    assert mb._source is not None
    lap = mb.lap
    assert mb._source is None and mb.lap is lap and lap.nnz > 0
    assert b.lap is not None and b._source is ds._lap
