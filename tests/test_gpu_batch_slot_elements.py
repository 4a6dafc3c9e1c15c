"""BatchSlot element layouts: a slot drawn from a dataset whose items carry faces and edges holds them in a
fixed-capacity element layout (every mesh's elements on 128-element tiles), planned by the same device planner and
gathered by the same dn_batch_gather launch, so a 'faces' / 'edges' segmentation net trains on shuffled batches in one
CUDA graph.

The gold is the host restatement of the element plan, ds.batch(ids)'s elements and ops.element_csr of them, and the
eager ds.batch(ids) training step with per-mesh label lists."""
import copy
import json
import os
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
KINDS = (("faces", B.R_FACES, B.R_FACES_CSR, 3), ("edges", B.R_EDGES, B.R_EDGES_CSR, 2))
BOTH = ("faces", "edges")


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def test_slot_element_capacity():
    """The n largest element counts, each padded to a tile; at least one tile."""
    assert B.slot_element_capacity([2, 254, 256, 258, 6000], 1) == 6016
    assert B.slot_element_capacity([2, 254, 256, 258, 6000], 2) == 6016 + 384
    assert B.slot_element_capacity([2, 254, 256, 258, 6000], 3) == 6016 + 384 + 256
    assert B.slot_element_capacity([0, 0], 2) == 128


# ---- GPU helpers --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    dn._lib.load()
    yield torch.device("cuda")
    dn.set_engine("tc3x")


def _launches():
    return dn._lib.load().dn_kernel_launch_count()


# torus grids (and one open patch) of the row counts the layout must handle: 1 and 127 rows (degenerate tori), exact
# tiles (128, 256), one row past a tile (129), a large mesh (3000)
GRIDS = [("torus", 1, 1), ("torus", 1, 127), ("torus", 8, 16), ("torus", 3, 43), ("torus", 16, 16),
         ("torus", 50, 60), ("patch", 6, 7), ("torus", 5, 8)]


def _elements(kind, n, m):
    f = (dn.synthetic.torus_mesh if kind == "torus" else dn.synthetic.patch_mesh)(n, m)[1]
    e = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).sort(dim=1).values.unique(dim=0)
    return f, e


def _items(K=16, seed=0, grids=GRIDS):
    """Meshes with random gradient CSRs and eigenpairs, and the faces and edges of their grids."""
    rs = np.random.RandomState(seed)
    items = []
    for kind, n, m in grids:
        V = n * m
        deg = np.minimum(rs.randint(0, 6, V), V)
        rowptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int32)
        cols = np.concatenate([np.sort(rs.choice(V, d, replace=False)) for d in deg] + [np.zeros(0)]).astype(np.int32)
        vals = (rs.randn(len(cols), 2) * 0.3).astype(np.float32)
        t = lambda a: torch.from_numpy(a).cuda()
        g = dn.ops.GradOperators.from_csr(V, t(rowptr), t(cols), t(vals))
        f, e = _elements(kind, n, m)
        items.append(dict(mass=t(rs.rand(V).astype(np.float32) + 0.5), evals=t(rs.rand(K).astype(np.float32)),
                          evecs=t((rs.randn(V, K) * 0.3).astype(np.float32)), gradX=g, faces=f.cuda(), edges=e.cuda()))
    return items


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int32 if t.dtype == torch.float32 else t.dtype)


def _eq(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _host_element_plan(ids, counts, k, cap):
    """The element plan restated on the host: begins, counts, tile_seg, and the corner and CSR ranges per mesh."""
    c = np.asarray(counts, np.int64)[ids]
    pe = (c + 127) // 128 * 128
    begin = np.concatenate([[0], np.cumsum(pe)])
    csr0 = np.concatenate([[0], np.cumsum(c * k)])
    src = B._starts(counts)[ids]
    tile_seg = np.asarray(dn.ops.Segments.tile_table(begin[:-1], c, cap), np.int32)
    rng = np.stack([src, begin[:-1], c, pe], 1)
    csr = np.stack([src * k, csr0[:-1], c * k, c * k], 1)
    return begin, c, tile_seg, rng, csr, int(csr0[-1])


def _check_element_plan(slot, ds, ids):
    nb = len(ids)
    tab = slot._table.cpu().numpy()
    assert tab.shape == (2 * nb, B.N_SLOT_RANGES, 4)
    t = B.batch_tables(ids, ds.n_rows, ds._grad_nnz, sm_count=ds._sm)
    assert np.array_equal(tab[:nb, :B.R_FACES], t["table"][:, :B.R_FACES])       # rows, meshes, pointers, entries
    row_begin = t["row_begin"]
    assert np.array_equal(tab[:nb, B.R_CORNER_OFF], np.stack([0 * row_begin[:-1], row_begin[:-1], 0 * row_begin[:-1],
                                                               0 * row_begin[:-1]], 1))
    assert not tab[nb:, B.R_CORNER_OFF].any()                  # tail corners: offset 0, padded with row 0
    for name, rng, csr_rng, k in KINDS:
        cap = slot.element_capacity[name]
        begin, c, tile_seg, r, csr, n_corners = _host_element_plan(ids, ds._elems[name][1], k, cap)
        seg = slot.element_segments[name]
        assert np.array_equal(slot._elem_begin[name].cpu().numpy(), begin)
        assert np.array_equal(seg.rows.cpu().numpy(), c) and np.array_equal(seg.begin.cpu().numpy(), begin[:-1])
        st = seg.tile_seg.cpu().numpy()
        assert np.array_equal(st[:len(tile_seg)], tile_seg) and (st[len(tile_seg):] == -1).all()
        assert np.array_equal(tab[:nb, rng], r) and np.array_equal(tab[:nb, csr_rng], csr)
        tail = tab[nb:, rng]
        assert (tail[:, 0] == 0).all() and (tail[:, 2] == 0).all() and tail[0, 1] == begin[-1]
        assert tail[:, 3].sum() == cap - begin[-1] and (tail[:, 3] <= slot._elem_tail[name]).all()
        assert (tab[nb:, csr_rng] == np.array([0, n_corners, 0, 0])).all()
    assert slot.status.cpu().tolist() == [0, 0, 0]


def _check_element_layout(slot, ds, ids):
    """Elements bitwise ds.batch(ids)'s at the aligned offsets, padding corners the mesh's first row (row 0 past the
    batch), and the gathered CSR ops.element_csr of the batch's elements with elements renumbered to the slot."""
    b = ds.batch(ids)
    for name, _, _, k in KINDS:
        els, ref = getattr(slot, name), getattr(b, name)
        begin = slot._elem_begin[name].cpu().tolist()
        counts = b.elem_counts(name)
        to_slot = torch.cat([torch.arange(c) + begin[m] for m, c in enumerate(counts)]).cuda()
        assert _eq(els[to_slot], ref)
        pad = torch.ones(els.shape[0], dtype=torch.bool, device="cuda")
        pad[to_slot] = False
        row_of = torch.zeros(els.shape[0], dtype=torch.int64, device="cuda")
        for m in range(len(ids)):
            row_of[begin[m]:begin[m + 1]] = b.row_begin[m]
        assert (els[pad] == row_of[pad][:, None]).all()
        rowptr, ent = slot.element_csr(name)
        r_rowptr, r_ent = dn.ops.element_csr(ref, b.V)
        nnz = int(r_rowptr[-1])
        assert _eq(rowptr[:b.V + 1], r_rowptr) and (rowptr[b.V:] == nnz).all()
        assert _eq(ent[:nnz], to_slot[r_ent.long()].int())
    return b


# ---- GPU: the plan and the layout ----------------------------------------------------------------------------------------
@gpu
def test_element_plan_matches_host_restatement(cuda):
    """Many random id lists (B = 1 .. 12, repeats): the element ranges, segments and tile_seg equal the host
    restatement, the row ranges batch_tables'.  A slot made without elements= (over a dataset whose items carry them,
    or one whose items do not) holds none and keeps batch_tables' six ranges and the nine gather parts, bitwise."""
    ds = dn.MeshDataset(_items())
    rs = np.random.RandomState(0)
    for nb in (1, 2, 3, 5, 8, 12):
        slot = ds.slot(nb, max_rows=nb * 3072, max_entries=nb * 6 * 3000, elements=BOTH, max_elements=nb * 9216)
        for _ in range(8):
            ids = rs.randint(0, len(GRIDS), nb).tolist()
            slot.fill(torch.tensor(ids, device="cuda"))
            _check_element_plan(slot, ds, ids)
    plain = dn.MeshDataset([{k: v for k, v in it.items() if k not in BOTH} for it in _items()])
    for d in (plain, ds):
        slot = d.slot(3)
        assert slot.faces is None and slot.edges is None and slot._table.shape == (6, B.N_RANGES, 4)
        assert len(slot._parts) == 9 and slot._sizes.shape == (len(GRIDS), 4) and not slot.element_capacity
        for ids in ([5, 0, 2], [3, 3, 1]):
            slot.fill(ids)
            t = B.batch_tables(ids, d.n_rows, d._grad_nnz, sm_count=d._sm)
            assert np.array_equal(slot._table[:3].cpu().numpy(), t["table"])


@gpu
def test_element_layout_and_csr_bitwise_and_no_stale_entries(cuda):
    """After every fill, faces / edges are ds.batch(ids)'s at the slot's offsets and the gathered CSR is element_csr's;
    a small batch after a large one leaves no stale element or CSR entry reachable."""
    ds = dn.MeshDataset(_items(seed=1))
    slot = ds.slot(4, max_rows=4 * 3072, max_entries=4 * 6 * 3000, elements=BOTH,   # room for repeats
                   max_elements=4 * 9216)
    for ids in ([5, 4, 3, 2], [0, 1, 0, 1], [5, 5, 7, 6], [2, 2, 2, 2], [7, 0, 3, 1]):
        slot.fill(ids if ids[0] != 5 else torch.tensor(ids, device="cuda"))
        _check_element_layout(slot, ds, ids)
    F = torch.randn(ds._elems["faces"][0].shape[0], 3, device="cuda")
    YE = torch.randint(0, 8, (ds._elems["edges"][0].shape[0],), device="cuda")
    ids = [3, 6, 1, 5]
    b = ds.batch(ids)
    slot.fill(ids)
    for name, T in (("faces", F), ("edges", YE)):
        out = slot.pack_elements(T, name)
        assert out is slot.pack_elements(T, name)
        begin = slot._elem_begin[name].cpu().tolist()
        starts = B._starts(ds._elems[name][1])
        for m, i in enumerate(ids):
            c = ds._elems[name][1][i]
            assert _eq(out[begin[m]:begin[m] + c], T[starts[i]:starts[i] + c])
            assert not out[begin[m] + c:begin[m + 1]].any()
        assert not out[begin[-1]:].any()
    assert b.V <= slot.V


# ---- GPU: training -------------------------------------------------------------------------------------------------------
def _net(outputs_at="faces", seed=0):
    torch.manual_seed(seed)
    net = dn.DiffusionNet(C_in=16, C_out=8, C_width=64, N_block=2, dropout=False, outputs_at=outputs_at).cuda().train()
    with torch.no_grad():
        for n_, p_ in net.named_parameters():
            if n_.endswith("diffusion_time"):
                p_.uniform_(1e-3, 0.3)
    return net


def _step(net, batch, x, lab):
    net.zero_grad(set_to_none=True)
    x = x.clone().requires_grad_(True)
    losses, pred = net.forward_batch_nll(batch, x, lab)
    losses.sum().backward()
    return losses.detach(), pred, {k: p.grad.clone() for k, p in net.named_parameters()}, x.grad


def _labels(ds, seed):
    g = torch.Generator().manual_seed(seed)
    return {name: torch.randint(0, 8, (ds._elems[name][0].shape[0],), generator=g).cuda() for name, *_ in KINDS}


def _per_mesh(ds, Y, name, ids):
    s = B._starts(ds._elems[name][1])
    return [Y[s[i]:s[i] + ds._elems[name][1][i]] for i in ids]


@gpu
@pytest.mark.parametrize("engine", ["simt", "tc3x", "tc1x", "bf16"])
def test_element_training_against_ds_batch(cuda, engine):
    """forward_batch_nll of a 'faces' and an 'edges' net on a slot with labels in its element layout against the same
    step on ds.batch(ids) with per-mesh label lists: per-mesh losses within the vertex-layout route's 1e-6, predictions
    on real elements bitwise, parameter gradients within 1e-4 (the weight reductions run over the slot's capacity),
    input gradients on real rows within 1e-5.  Garbage in the padding rows, padding labels and padding corners (any
    row of the slot) changes no loss or gradient bit.  The simt engine refuses both routes alike."""
    dn.set_engine(engine)
    try:
        ds = dn.MeshDataset(_items(seed=2))
        X = torch.randn(ds.V, 16, generator=torch.Generator().manual_seed(3)).cuda()
        Y = _labels(ds, 4)
        slot = ds.slot(3, elements=BOTH)
        if engine == "simt":
            slot.fill([5, 0, 2])
            b = ds.batch([5, 0, 2])
            with pytest.raises(RuntimeError, match="unsupported"):
                _step(_net(), slot, slot.pack(X), slot.pack_elements(Y["faces"], "faces"))
            with pytest.raises(RuntimeError, match="unsupported"):
                _step(_net(), b, ds.pack(X, b), _per_mesh(ds, Y["faces"], "faces", [5, 0, 2]))
            return
        worst = {}
        for ids in ([5, 0, 2], [3, 3, 1], [1, 4, 6], [7, 2, 5]):
            slot.fill(torch.tensor(ids, device="cuda"))
            b = ds.batch(ids)
            real = torch.zeros(slot.V, dtype=torch.bool, device="cuda")
            for r0, n in zip(b.row_begin, b.n_rows):
                real[r0:r0 + n] = True
            for name, *_ in KINDS:
                lab = slot.pack_elements(Y[name], name)
                a = _step(_net(name), slot, slot.pack(X), lab)
                r = _step(_net(name), b, ds.pack(X, b), _per_mesh(ds, Y[name], name, ids))
                begin = slot._elem_begin[name].cpu().tolist()
                to_slot = torch.cat([torch.arange(c) + begin[m] for m, c in enumerate(b.elem_counts(name))]).cuda()
                assert a[0].shape == (3,) and a[1].shape == (slot.element_capacity[name],)
                w = {"loss": O.rel_err(a[0].cpu().numpy(), r[0].cpu().numpy())}
                assert w["loss"] < 1e-6, (name, a[0], r[0])
                assert _eq(a[1][to_slot], torch.cat(r[1]))
                w["param_grad"] = max(O.rel_err(a[2][k].cpu().numpy(), r[2][k].cpu().numpy()) for k in a[2])
                assert w["param_grad"] < 1e-4, (name, w)
                w["x_grad"] = O.rel_err(a[3][:b.V][real[:b.V]].cpu().numpy(), r[3][real[:b.V]].cpu().numpy())
                assert w["x_grad"] < 1e-5, (name, w)
                assert not a[3][~real].any()
                for key, v in w.items():
                    worst[key] = max(worst.get(key, 0.0), v)
                # garbage in every padding: rows of x, labels, corners
                x = slot.pack(X).clone()
                lab = lab.clone()
                els = getattr(slot, name)
                pad_el = torch.ones(els.shape[0], dtype=torch.bool, device="cuda")
                pad_el[to_slot] = False
                n_pad = int(pad_el.sum())
                with torch.no_grad():
                    x[~real] = torch.randn(int((~real).sum()), 16, device="cuda") * 50
                    lab[pad_el] = torch.tensor([7777, -5, 3], device="cuda").repeat(n_pad // 3 + 1)[:n_pad]
                    els[pad_el] = torch.randint(0, slot.V, (n_pad, els.shape[1]), device="cuda")
                got = _step(_net(name), slot, x, lab)
                assert _eq(got[0], a[0]) and all(_eq(got[2][k], a[2][k]) for k in a[2]), name
                assert _eq(got[1][to_slot], a[1][to_slot]) and _eq(got[3][real], a[3][real])
        print(json.dumps({"engine": engine, "worst_rel_err_slot_vs_ds_batch": worst}))
    finally:
        dn.set_engine("tc3x")


# ---- GPU: graphs, no host work -------------------------------------------------------------------------------------------
@gpu
def test_graph_replay_matches_eager_slot_without_host_sync(cuda):
    """A graph-captured 'faces' step (fill and pack_elements inside) replays with new device ids bitwise what the eager
    slot step computes; a fill stays two library launches and pack_elements one, none of them synchronising."""
    dn.set_engine("tc3x")
    ds = dn.MeshDataset(_items(seed=5))
    X = torch.randn(ds.V, 16, device="cuda")
    Y = _labels(ds, 6)
    nb = 2
    slot = ds.slot(nb, elements="faces")
    ids = torch.tensor([0, 1], device="cuda")

    def step(net, ids_):
        slot.fill(ids_)
        return net.forward_batch_nll(slot, slot.pack(X), slot.pack_elements(Y["faces"], "faces"))[0].sum()

    net = _net(seed=7)
    gs = dn.graphs.GraphedTrainStep(net, step, (ids,))
    for new in ([5, 2], [3, 3], [6, 0]):
        ids.copy_(torch.tensor(new, device="cuda"))
        eager = copy.deepcopy(net)
        eager.zero_grad(set_to_none=True)
        le = step(eager, ids)
        le.backward()
        gs.zero_grads(net)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            loss = gs.replay()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert _eq(loss, le.detach()), new
        assert all(_eq(p.grad, q.grad) for p, q in zip(net.parameters(), eager.parameters())), new
    slot.check()
    counts = []
    for nb_ in (1, 4):
        s = ds.slot(nb_, elements=BOTH)
        d_ids = torch.arange(nb_, device="cuda")
        s.fill(d_ids), s.pack_elements(Y["edges"], "edges")
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            l0 = _launches()
            s.fill(d_ids)
            l1 = _launches()
            s.pack_elements(Y["edges"], "edges")
            l2 = _launches()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        counts.append((l1 - l0, l2 - l1))
        assert len(s._parts) == 15
    assert counts == [(2, 1), (2, 1)]


# ---- GPU: errors ---------------------------------------------------------------------------------------------------------
@gpu
def test_element_capacity_errors_and_mislabelled_shapes(cuda):
    """Over the element capacity: a device fill plans every mesh empty (NaN losses) and check() raises ValueError naming
    the position; a host fill raises before launching.  Mislabelled shapes keep their errors."""
    items = _items(seed=8)
    ds = dn.MeshDataset(items)
    X = torch.randn(ds.V, 16, device="cuda")
    Y = _labels(ds, 9)
    slot = ds.slot(2, elements=BOTH, max_elements={"faces": 256})   # mesh 3 (129 rows) has 258 faces: 384 padded
    assert slot.element_capacity == {"faces": 256, "edges": B.slot_element_capacity(ds._elems["edges"][1], 2)}
    slot.fill(torch.tensor([3, 0], device="cuda"))
    assert int(slot._elem_begin["faces"][-1]) == 0 and int(slot._row_begin[-1]) == 0
    losses, _ = _net().forward_batch_nll(slot, slot.pack(X), slot.pack_elements(Y["faces"], "faces"))
    assert torch.isnan(losses).all()
    with pytest.raises(ValueError, match="256 faces .*at position 0"):
        slot.check()
    slot.check()
    slot.fill(torch.tensor([0, 6], device="cuda"))
    _check_element_layout(slot, ds, [0, 6])
    faces_only = dn.MeshDataset([{k: v for k, v in it.items() if k != "edges"} for it in items[:3]])
    s = faces_only.slot(1, elements="faces")
    torch.cuda.synchronize()
    l0 = _launches()
    with pytest.raises(ValueError, match="capacity"):
        slot.fill([0, 3])
    net = _net()
    x = torch.zeros(slot.V, 16, device="cuda")
    E = slot.element_capacity["faces"]
    assert slot.V != E
    with pytest.raises(NotImplementedError, match="per vertex"):
        net.forward_batch_nll(slot, x, torch.zeros(slot.V, dtype=torch.int64, device="cuda"))
    with pytest.raises(NotImplementedError, match="per vertex"):
        net.forward_batch_nll(slot, x, torch.zeros(E, 2, dtype=torch.int64, device="cuda"))
    with pytest.raises(ValueError, match="int64 tensor of shape"):
        net.forward_batch_nll(slot, x, torch.zeros(E, device="cuda"))
    with pytest.raises(ValueError, match="dataset layout"):
        slot.pack_elements(Y["faces"][:-1], "faces")
    with pytest.raises(ValueError, match="holds no 'vertices'"):
        slot.pack_elements(Y["faces"], "vertices")
    with pytest.raises(NotImplementedError, match="no host copy"):
        slot.elem_counts("faces")
    with pytest.raises(NotImplementedError, match="forward_batch"):
        net.forward_batch(slot, x)
    assert s.edges is None and s._table.shape[1] == B.N_SLOT_RANGES
    with pytest.raises(NotImplementedError, match="per vertex"):
        _net("edges").forward_batch_nll(s, torch.zeros(s.V, 16, device="cuda"),
                                        torch.zeros(s.element_capacity["faces"], dtype=torch.int64, device="cuda"))
    assert _launches() == l0
    bad = [dict(it) for it in items[:2]]
    bad[1]["faces"] = bad[1]["faces"].clone()
    bad[1]["faces"][4, 1] = bad[1]["mass"].shape[0]
    with pytest.raises(ValueError, match="face 4 of mesh 1 has a corner outside"):
        dn.MeshDataset(bad).slot(1, elements="faces")
    dn.MeshDataset(bad).slot(1)                                # a slot without elements never reads them
    with pytest.raises(ValueError, match="carry no 'edges'"):
        faces_only.slot(1, elements=BOTH)
    with pytest.raises(ValueError, match="each once"):
        ds.slot(1, elements=("faces", "faces"))
    with pytest.raises(ValueError, match="pass elements="):
        ds.slot(1, max_elements=256)
    with pytest.raises(ValueError, match="does not hold"):
        ds.slot(1, elements="faces", max_elements={"edges": 256})


@gpu
def test_pair_slot_over_a_face_carrying_dataset(cuda):
    """A PairDataset over meshes that carry faces of unequal counts, drawn with a repeated shape: the pair slot holds
    no elements (it never asks for them), fills clean and computes bitwise what it computes when the items carry no
    faces, where an element layout of the distinct-mesh default would have been over capacity."""
    torch.manual_seed(0)
    m = dn.FunctionalMapCorrespondenceWithDiffusionNetFeatures(n_feat=128, input_features="xyz").cuda().eval()
    shapes = [(40, 25), (10, 10), (8, 12)]                     # 2000, 200 and 192 faces
    items = []
    for i, (a, b) in enumerate(shapes):
        mass, _, evals, evecs, gX, gY = dn.synthetic.structural_operators(a, b, 64, seed=30 + i, device="cuda")
        items.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY,
                          faces=dn.synthetic.torus_mesh(a, b)[1].cuda()))
    rs = np.random.RandomState(1)
    vts = [torch.from_numpy(rs.randint(0, it["mass"].shape[0], 60).astype(np.int64)) for it in items]
    X = torch.randn(sum(it["mass"].shape[0] for it in items), 3, generator=torch.Generator().manual_seed(2)).cuda()
    out = []
    for with_faces in (True, False):
        ds = dn.MeshDataset([it if with_faces else {k: v for k, v in it.items() if k != "faces"} for it in items])
        pds = dn.PairDataset(ds, vts, [(0, 1), (0, 2)])
        slot = pds.slot(2)
        assert slot.mesh_batch.faces is None and not slot.mesh_batch.element_capacity
        if with_faces:         # shapes 0, 0, 1, 2: 2 x 2048 + 2 x 256 padded faces, past any 4 distinct meshes'
            assert 2 * 2048 + 512 > B.slot_element_capacity(ds._elems["faces"][1], 4)
        slot.fill(torch.tensor([0, 1], device="cuda"))
        with torch.no_grad():
            C, _ = m.forward_pairs(slot, slot.pack(X))
        slot.check()
        assert torch.isfinite(C).all()
        out.append(C)
    assert _eq(out[0], out[1])
