"""BatchSlot: a fixed-capacity batch refilled on the device from any mesh ids (dn_mesh_batch_plan_device + one
dn_batch_gather), so a shuffled training step can be captured in one CUDA graph.

The gold is what the parent computes for the same ids: batch_tables (the host plan and gather table) and every array of
ds.batch(ids), bitwise, on the batch's rows; the rows past them must follow the padding conventions.  The CPU tests
check the capacity, the CTA bound the slot's fixed to_basis grid rests on (against the host planner on adversarial size
mixes), host id validation and the planner kernel's registers."""
import copy
import json
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


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def test_slot_capacity():
    """V_cap: the n largest padded row counts (at least one tile); entries: the n largest entry counts, on their own;
    the to_basis grid min(1024, sm + n)."""
    n_rows = [1, 300, 129, 128, 1000, 5]
    n_ent = [900, 10, 20, 30, 40, 800]                 # the largest entry counts belong to the smallest meshes
    assert B.slot_capacity(n_rows, n_ent, 1, 132) == (1024, 900, 133)
    assert B.slot_capacity(n_rows, n_ent, 2, 132) == (1024 + 384, 1700, 134)
    assert B.slot_capacity(n_rows, n_ent, 3, 132) == (1024 + 384 + 256, 1740, 135)
    assert B.slot_capacity([0, 0], [0, 0], 2, 132) == (128, 0, 134)
    assert B.slot_capacity([7] * 2000, [1] * 2000, 1000, 132)[2] == 1024


def _adversarial_mixes(rs):
    yield [1] * 1024                                       # every mesh one chunk
    yield [100_000] + [1] * 1023                           # one mesh wants everything
    yield [3000] * 1024                                    # the cap rule on every mesh
    yield [16 * 132] * 7 + [17] * 50                       # shares just above 1/2
    for B_ in (1, 2, 5, 33, 131, 132, 133, 700, 1024):
        for _ in range(6):
            kind = rs.randint(4)
            if kind == 0:
                n = rs.randint(1, 20_000, B_)
            elif kind == 1:
                n = np.where(rs.rand(B_) < 0.1, rs.randint(10_000, 200_000, B_), rs.randint(0, 40, B_))
            elif kind == 2:
                n = rs.randint(0, 17, B_)
            else:
                n = (rs.randint(1, 8, B_) * 16 * 132 // max(B_ // 4, 1)) + rs.randint(-1, 2, B_)
            yield [max(int(v), 0) for v in n]


@pytest.mark.parametrize("sm", [132, 114, 1])
def test_cta_bound_on_adversarial_size_mixes(sm):
    """The host planner never uses more to_basis CTAs than min(1024, sm + n_meshes): the slot's fixed grid holds any
    batch (slot_capacity's argument: each mesh gets at most chunks_b sm / total + 1)."""
    rs = np.random.RandomState(sm)
    n_mixes = 0
    for n_rows in _adversarial_mixes(rs):
        n_ctas = B.plan_rows(n_rows, sm)[4]
        assert n_ctas <= min(1024, sm + len(n_rows)), (len(n_rows), n_ctas)
        n_mixes += 1
    assert n_mixes > 50


def _host_slot(n_rows, n_ent, n_meshes):
    """A slot over a dataset that exists only as sizes: fill's host checks run before anything touches a device."""
    ds = B.MeshDataset.__new__(B.MeshDataset)
    ds.n_meshes, ds.n_rows, ds._grad_nnz = len(n_rows), list(n_rows), list(n_ent)
    slot = B.BatchSlot.__new__(B.BatchSlot)
    slot._ds, slot.n_meshes = ds, n_meshes
    slot.V, _, _ = B.slot_capacity(n_rows, n_ent, n_meshes, 132)
    slot.entry_capacity = B.slot_capacity(n_rows, n_ent, n_meshes, 132)[1]
    return slot


def test_host_id_validation():
    slot = _host_slot([100, 300, 50], [10, 5, 400], 2)
    with pytest.raises(IndexError, match="outside"):
        slot.fill([0, 3])
    with pytest.raises(IndexError, match="outside"):
        slot.fill(torch.tensor([-1, 0]))
    with pytest.raises(ValueError, match="at least one"):
        slot.fill([])
    with pytest.raises(TypeError):
        slot.fill(torch.tensor([0.0, 1.0]))
    with pytest.raises(ValueError, match="2 meshes"):
        slot.fill([0, 1, 2])
    with pytest.raises(ValueError, match="capacity"):          # rows: 300 twice pads to 768 > 384 + 128
        slot.fill([1, 1])
    with pytest.raises(ValueError, match="capacity"):          # entries: 400 twice > 400 + 10
        slot.fill([2, 2])


def test_planner_kernel_does_not_spill(tmp_path):
    if shutil.which(NVCC) is None and not os.path.exists(NVCC):
        pytest.skip("needs nvcc")
    flags = [f for f in dn._lib.NVCC_FLAGS if f != "-shared"]
    cmd = [NVCC] + flags + ["-Xptxas", "-v", "-c", os.path.join(dn._lib._CSRC, "dn_batch_plan.cu"), "-o",
                            str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    out = r.stdout + r.stderr
    lines = [l for l in out.splitlines() if "spill stores" in l]
    assert len(lines) == 1
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", lines[0])
    assert m and m.groups() == ("0", "0", "0"), lines[0]
    regs = int(re.search(r"Used (\d+) registers", out).group(1))
    assert regs <= 64                                          # 1024 threads per CTA


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


def _csr_items(sizes, K, seed=0):
    """Items with random gradient CSRs (prepared operators built from host arrays, quick for a thousand meshes)."""
    rs = np.random.RandomState(seed)
    items = []
    for V in sizes:
        deg = np.minimum(rs.randint(0, 6, V), V)
        rowptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int32)
        cols = np.concatenate([np.sort(rs.choice(V, d, replace=False)) for d in deg] + [np.zeros(0)]).astype(np.int32)
        vals = rs.randn(len(cols), 2).astype(np.float32)
        t = lambda a: torch.from_numpy(a).cuda()
        g = dn.ops.GradOperators.from_csr(V, t(rowptr), t(cols), t(vals))
        items.append(dict(mass=t(rs.rand(V).astype(np.float32) + 0.5), evals=t(rs.rand(K).astype(np.float32)),
                          evecs=t(rs.randn(V, K).astype(np.float32)), gradX=g))
        if K == 0:
            items[-1]["L"] = torch.eye(V).to_sparse().cuda()
    return items


def _plan_of(slot):
    return dict(row_begin=slot._row_begin, tile_mesh=slot._tile_mesh, tb_rows=slot._tb_rows,
                cta_begin=slot._cta_begin, seg_begin=slot.segments.begin, seg_rows=slot.segments.rows,
                tile_seg=slot.segments.tile_seg, table=slot._table)


def _check_plan(slot, ds, ids):
    """The device plan of a filled slot against batch_tables: bitwise on the batch, padding conventions past it."""
    t = B.batch_tables(ids, ds.n_rows, ds._grad_nnz, sm_count=ds._sm)
    p = {k: v.cpu().numpy() for k, v in _plan_of(slot).items()}
    V, nb, n_ctas, tiles = t["V"], len(ids), t["n_ctas"], t["V"] // 128
    assert np.array_equal(p["row_begin"], t["row_begin"])
    assert np.array_equal(p["cta_begin"], t["cta_begin"])
    assert np.array_equal(p["tb_rows"][:2 * n_ctas], t["tb_rows"])
    assert (p["tb_rows"][2 * n_ctas:] == V).all()               # surplus CTAs: empty, outside every mesh's range
    assert np.array_equal(p["tile_mesh"][:tiles], t["tile_mesh"][:tiles])
    assert (p["tile_mesh"][tiles:] == nb - 1).all()
    assert np.array_equal(p["seg_begin"], t["seg_begin"]) and np.array_equal(p["seg_rows"], t["seg_rows"])
    assert np.array_equal(p["tile_seg"][:tiles], t["tile_seg"]) and (p["tile_seg"][tiles:] == -1).all()
    assert np.array_equal(p["table"][:nb], t["table"])
    tail = p["table"][nb:]                                      # the tail pieces cover [V, V_cap) as padding
    assert (tail[:, B.R_ROWS, 2] == 0).all() and tail[:, B.R_ROWS, 3].sum() == slot.V - V
    assert tail[0, B.R_ROWS, 1] == V and (tail[:, B.R_ENT, 1] == t["nnz"]).all()
    assert (tail[:, B.R_ROWS, 3] <= slot._tail).all()
    assert slot.status.cpu().tolist() == [0, 0, 0]
    return t


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int32 if t.dtype == torch.float32 else t.dtype)


def _eq(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


SIZES = [1, 15, 16, 127, 128, 129, 300, 3000, 700, 40, 200, 128]


# ---- GPU: the plan and the layout ----------------------------------------------------------------------------------------
@gpu
def test_device_plan_matches_the_host_plan(cuda):
    """Many random id lists (B = 1 .. 12, repeats within capacity, meshes under 16 rows and of exactly 128): the
    device plan, segments and gather table are bitwise batch_tables'."""
    items = _csr_items(SIZES, 8)
    ds = dn.MeshDataset(items)
    rs = np.random.RandomState(0)
    for nb in (1, 2, 5, 12):
        slot = ds.slot(nb, max_rows=nb * 3072, max_entries=nb * 6 * 3000)   # room for any repeats
        for _ in range(12):
            ids = rs.randint(0, len(SIZES), nb).tolist()
            slot.fill(torch.tensor(ids, device="cuda"))
            _check_plan(slot, ds, ids)
    slot = ds.slot(3)
    for ids in ([7, 8, 6], [0, 1, 2], [4, 11, 3]):
        slot.fill(ids)                                         # host ids
        _check_plan(slot, ds, ids)


@gpu
def test_device_plan_at_1024_meshes(cuda):
    """A 1024-mesh dataset at B = 1024 and B = 1000: the running-count rule of the host planner fires and the
    device planner follows it bitwise."""
    rs = np.random.RandomState(1)
    sizes = rs.randint(1, 400, 1024).tolist()
    sizes[5], sizes[900] = 2000, 3000
    ds = dn.MeshDataset(_csr_items(sizes, 4, seed=3))
    for nb in (1024, 1000):
        slot = ds.slot(nb)
        for k in range(3):
            ids = rs.permutation(1024)[:nb].tolist()
            slot.fill(torch.tensor(ids, device="cuda"))
            t = _check_plan(slot, ds, ids)
            if nb == 1024:                 # the 3000-row mesh wants two CTAs: the rule leaves every mesh one
                assert t["n_ctas"] == 1024
    _check_layout(slot, ds, ids)


def _check_layout(slot, ds, ids, X=None):
    b = ds.batch(ids)
    V, nnz = b.V, b.gops.nnz
    assert _eq(slot.mass[:V], b.mass) and _eq(slot.evecs[:V], b.evecs) and _eq(slot.evals, b.evals)
    assert (slot.mass[V:] == 0).all() and (slot.evecs[V:] == 0).all()
    for mine, theirs in ((slot.gops.csr, b.gops.csr), (slot.gops.csr_t, b.gops.csr_t)):
        assert _eq(mine[1][:V + 1], theirs[1]) and (mine[1][V:] == nnz).all()
        assert _eq(mine[2][:nnz], theirs[2][:nnz])
        assert _eq(mine[3].reshape(-1)[:2 * nnz], theirs[3].reshape(-1)[:2 * nnz])
    if X is not None:
        x = slot.pack(X)
        assert _eq(x[:V], ds.pack(X, b)) and (x[V:] == 0).all()
    return b


@gpu
def test_layout_bitwise_and_no_stale_rows(cuda):
    """Every gathered array, the transposed CSR included, is ds.batch(ids)'s on the batch's rows, and padding past
    them; a short batch after a long one leaves nothing of it behind.  The slot never calls dn_csr_transpose."""
    items = _csr_items(SIZES, 16, seed=4)
    ds = dn.MeshDataset(items)
    X = torch.randn(ds.V, 5, device="cuda")
    Y = torch.randint(0, 9, (ds.V,), device="cuda")
    slot = ds.slot(4)
    assert slot.gops._csr_t is not None
    for ids in ([7, 8, 6, 9], [0, 1, 2, 3], [7, 6, 8, 10], [0, 0, 1, 4], [11, 3, 5, 2]):
        slot.fill(ids)
        b = _check_layout(slot, ds, ids, X)
        y = slot.pack(Y)
        assert _eq(y[:b.V], ds.pack(Y, b)) and (y[b.V:] == 0).all()
    assert slot.pack(X) is slot.pack(X)


# ---- GPU: the routes -----------------------------------------------------------------------------------------------------
SHAPES = [(12, 11), (36, 50), (8, 10), (16, 8), (20, 13), (30, 30)]


def _net_items(K=64, seed=0):
    out = []
    for i, (n, m) in enumerate(SHAPES):
        mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=seed + i, device="cuda")
        out.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY))
    return out


def _net(C_out=5, outputs_at="vertices", seed=0):
    torch.manual_seed(seed)
    net = dn.DiffusionNet(C_in=16, C_out=C_out, C_width=64, N_block=2, dropout=False,
                          outputs_at=outputs_at).cuda().train()
    with torch.no_grad():
        for n_, p_ in net.named_parameters():
            if n_.endswith("diffusion_time"):
                p_.uniform_(1e-3, 0.3)
    return net


def _real_rows(b, V):
    m = torch.zeros(V, dtype=torch.bool, device="cuda")
    for r0, n in zip(b.row_begin, b.n_rows):
        m[r0:r0 + n] = True
    return m


def _step(net, batch, x, lab, route):
    net.zero_grad(set_to_none=True)
    x = x.clone().requires_grad_(True)
    if route == "global":
        losses, pred = net.forward_batch_global_nll(batch, x, lab, label_smoothing=0.1)
    else:
        losses, pred = net.forward_batch_nll(batch, x, lab)
    losses.sum().backward()
    return losses.detach(), pred, {k: p.grad.clone() for k, p in net.named_parameters()}, x.grad


@gpu
@pytest.mark.parametrize("engine", ["tc3x", "bf16"])
def test_routes_against_ds_batch(cuda, engine):
    """forward_batch_global_nll and layout-label forward_batch_nll on a slot against the same step on ds.batch(ids):
    per-mesh losses, predictions and input gradients on the batch's rows bitwise; parameter gradients within the
    shuffled run's tc3x bound (the weight reductions run over V_cap rows instead of V), worst difference recorded.
    The layout-label route on a MeshBatch agrees with its per-mesh list route."""
    dn.set_engine(engine)
    try:
        ds = dn.MeshDataset(_net_items())
        g = torch.Generator().manual_seed(0)
        X = torch.randn(ds.V, 16, generator=g).cuda()
        Y = torch.randint(0, 5, (ds.V,), generator=g).cuda()
        Yg = torch.randint(0, 4, (len(SHAPES),), generator=g).cuda()
        slot = ds.slot(3)
        worst = 0.0
        for ids in ([1, 3, 5], [0, 2, 4], [4, 4, 1]):
            slot.fill(ids)
            b = ds.batch(ids)
            real = _real_rows(b, b.V)
            for route, mk in (("global", lambda: _net(C_out=4, outputs_at="global_mean")), ("vertices", _net)):
                if route == "global":
                    a = _step(mk(), slot, slot.pack(X), slot.take(Yg), route)
                    r = _step(mk(), b, ds.pack(X, b), Yg[ids], route)
                else:
                    a = _step(mk(), slot, slot.pack(X), slot.pack(Y), route)
                    r = _step(mk(), b, ds.pack(X, b), ds.pack(Y, b), route)
                    assert _eq(a[1][:b.V][real], r[1][real])
                    lst = _step(mk(), b, ds.pack(X, b), b.unpack(ds.pack(Y, b)), route)
                    assert O.rel_err(r[0].cpu().numpy(), lst[0].cpu().numpy()) < 1e-6
                    assert all(torch.equal(u, r[1][r0:r0 + n]) for u, r0, n in zip(lst[1], b.row_begin, b.n_rows))
                    assert not r[3][~real].any()
                assert _eq(a[0], r[0]), (route, a[0], r[0])
                assert _eq(a[3][:b.V][real], r[3][real]) and not a[3][~torch.cat([real, real.new_zeros(
                    slot.V - b.V)])].any()
                for k in a[2]:
                    e = O.rel_err(a[2][k].cpu().numpy(), r[2][k].cpu().numpy())
                    worst = max(worst, e)
                    assert e < 1e-4, (route, k, e)
        print(json.dumps({"engine": engine, "param_grad_rel_err_slot_vs_ds_batch": worst}))
    finally:
        dn.set_engine("tc3x")


@gpu
def test_padding_contents_change_nothing(cuda):
    """Finite garbage in the padding rows of the static feature and label buffers changes no loss or gradient."""
    ds = dn.MeshDataset(_net_items())
    g = torch.Generator().manual_seed(1)
    X = torch.randn(ds.V, 16, generator=g).cuda()
    Y = torch.randint(0, 5, (ds.V,), generator=g).cuda()
    slot = ds.slot(2)
    ids = [4, 1]
    slot.fill(ids)
    pad = ~_real_rows(ds.batch(ids), slot.V)
    x, y = slot.pack(X), slot.pack(Y)
    ref = _step(_net(), slot, x, y, "vertices")
    with torch.no_grad():
        x[pad] = torch.randn(int(pad.sum()), 16, device="cuda") * 50
        y[pad] = torch.tensor([7777, -5, 3], device="cuda").repeat(int(pad.sum()) // 3 + 1)[:int(pad.sum())]
    got = _step(_net(), slot, x, y, "vertices")
    assert _eq(got[0], ref[0]) and all(_eq(got[2][k], ref[2][k]) for k in ref[2])
    assert _eq(got[3][~pad], ref[3][~pad])
    refg = _step(_net(C_out=4, outputs_at="global_mean"), slot, slot.pack(X), slot.take(Y[:len(SHAPES)] % 4), "global")
    x = slot.pack(X)
    with torch.no_grad():
        x[pad] = 1e3
    gotg = _step(_net(C_out=4, outputs_at="global_mean"), slot, x, slot.take(Y[:len(SHAPES)] % 4), "global")
    assert _eq(gotg[0], refg[0]) and all(_eq(gotg[2][k], refg[2][k]) for k in refg[2])


# ---- GPU: graphs, no host work -------------------------------------------------------------------------------------------
@gpu
def test_graph_replay_and_shuffled_sgd(cuda):
    """A graph-captured slot step (fill inside) replays bitwise what the eager slot step computes, reproducibly; two
    epochs of graph-replayed SGD over randperm chunks follow the eager ds.batch loop within the tc3x bound."""
    dn.set_engine("tc3x")
    ds = dn.MeshDataset(_net_items(seed=7))
    g = torch.Generator().manual_seed(2)
    X = torch.randn(ds.V, 16, generator=g).cuda()
    Yg = torch.randint(0, 4, (len(SHAPES),), generator=g).cuda()
    nb = 2
    slot = ds.slot(nb)
    ids = torch.zeros(nb, dtype=torch.int64, device="cuda")

    def step(net, ids):
        slot.fill(ids)
        return net.forward_batch_global_nll(slot, slot.pack(X), slot.take(Yg), label_smoothing=0.2)[0].sum()

    net = _net(C_out=4, outputs_at="global_mean", seed=3)
    ref = copy.deepcopy(net)
    gs = dn.graphs.GraphedTrainStep(net, step, (ids,))
    # replay against the eager slot step, twice
    ids.copy_(torch.tensor([3, 0], device="cuda"))
    eager = copy.deepcopy(net)
    eager.zero_grad(set_to_none=True)
    le = step(eager, ids)
    le.backward()
    outs = []
    for _ in range(2):
        gs.zero_grads(net)
        loss = gs.replay().clone()
        outs.append((loss, [p.grad.clone() for p in net.parameters()]))
    for loss, grads in outs:
        assert _eq(loss, le.detach())
        assert all(_eq(u, p.grad) for u, p in zip(grads, eager.parameters()))
    # two epochs against the eager ds.batch loop
    opt = torch.optim.SGD(net.parameters(), lr=1e-2)
    opt_ref = torch.optim.SGD(ref.parameters(), lr=1e-2)
    gen = torch.Generator(device="cuda").manual_seed(4)
    steps = 0
    for epoch in range(2):
        for chunk in torch.randperm(len(SHAPES), device="cuda", generator=gen).split(nb):
            ids.copy_(chunk)
            gs.zero_grads(net)
            loss = gs.replay()
            b = ds.batch(chunk.tolist())
            opt_ref.zero_grad(set_to_none=True)
            lr_ = ref.forward_batch_global_nll(b, ds.pack(X, b), Yg[chunk], label_smoothing=0.2)[0].sum()
            lr_.backward()
            assert O.rel_err(loss.item(), lr_.item()) < 1e-5
            for (name, p_), q_ in zip(net.named_parameters(), ref.parameters()):
                assert O.rel_err(p_.grad.cpu().numpy(), q_.grad.cpu().numpy()) < 1e-4, (steps, name)
            opt.step()
            opt_ref.step()
            steps += 1
    assert steps == 6
    slot.check()


@gpu
def test_fill_pack_take_and_replay_do_not_synchronise(cuda):
    ds = dn.MeshDataset(_net_items())
    X = torch.randn(ds.V, 16, device="cuda")
    Yg = torch.randint(0, 4, (len(SHAPES),), device="cuda")
    counts = []
    for nb in (1, 4):
        slot = ds.slot(nb)
        ids = torch.arange(nb, device="cuda")
        slot.fill(ids), slot.pack(X), slot.take(Yg)            # warm the allocators
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            l0 = _launches()
            slot.fill(ids)
            l1 = _launches()
            slot.pack(X)
            l2 = _launches()
            slot.take(Yg)
            l3 = _launches()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        counts.append((l1 - l0, l2 - l1, l3 - l2))
    assert counts == [(2, 1, 0), (2, 1, 0)]
    net = _net(C_out=4, outputs_at="global_mean")
    slot = ds.slot(2)
    ids = torch.tensor([1, 2], device="cuda")

    def step(net_, ids_):
        slot.fill(ids_)
        return net_.forward_batch_global_nll(slot, slot.pack(X), slot.take(Yg))[0].sum()
    gs = dn.graphs.GraphedTrainStep(net, step, (ids,))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ids.fill_(3)
        gs.zero_grads(net)
        gs.replay()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


# ---- GPU: invalid fills and refusals -------------------------------------------------------------------------------------
def _snapshot(slot):
    """Every array a step reads: the CSR entries up to the batch's count (entries past it are never read)."""
    nnz = int(slot.gops.csr[1][-1])
    csrs = [c for csr in (slot.gops.csr, slot.gops.csr_t) for c in (csr[1], csr[2][:nnz], csr[3].reshape(-1)[:2 * nnz])]
    return [t.clone() for t in [slot.mass, slot.evecs, slot.evals, slot.status] + csrs + list(_plan_of(slot).values())]


@gpu
def test_invalid_device_fills(cuda):
    """An out-of-range device id and an over-capacity repeat batch set the sticky status, read nothing through the
    ids, plan every mesh empty (every loss NaN); check() names the position and clears; the next valid fill is bitwise
    a fresh slot's."""
    ds = dn.MeshDataset(_net_items())
    X = torch.randn(ds.V, 16, device="cuda")
    Yg = torch.randint(0, 4, (len(SHAPES),), device="cuda")
    Y = torch.randint(0, 5, (ds.V,), device="cuda")
    slot = ds.slot(3)
    slot.check()                                               # nothing to report
    big = int(np.argmax(ds.n_rows))
    for bad, err, msg in (([0, 2, 99], IndexError, "id 99 at position 2"), ([1, -3, 0], IndexError, "position 1"),
                          ([big, big, big], ValueError, "capacity .* at position 1")):
        slot.fill(torch.tensor(bad, device="cuda"))
        assert int(slot._row_begin[-1]) == 0 and not slot.mass.any() and not slot.evals.any()
        slot.fill(torch.tensor([0, 1, 2], device="cuda"))      # sticky: the first invalid fill is kept
        slot.fill(torch.tensor(bad, device="cuda"))
        losses, _ = _net(C_out=4, outputs_at="global_mean").forward_batch_global_nll(slot, slot.pack(X), slot.take(Yg))
        assert torch.isnan(losses).all()
        losses, _ = _net().forward_batch_nll(slot, slot.pack(X), slot.pack(Y))
        assert torch.isnan(losses).all()
        with pytest.raises(err, match=msg):
            slot.check()
        slot.check()                                           # cleared
        slot.fill(torch.tensor([4, 2, 0], device="cuda"))
        fresh = ds.slot(3).fill(torch.tensor([4, 2, 0], device="cuda"))
        assert all(_eq(u, v) for u, v in zip(_snapshot(slot), _snapshot(fresh)))
        assert _eq(slot.pack(X), fresh.pack(X)) and _eq(slot.take(Yg), fresh.take(Yg))
        slot.check()


@gpu
def test_refusals_before_any_launch(cuda):
    items = _net_items()
    ds = dn.MeshDataset(items)
    implicit_only = dn.MeshDataset(_csr_items([30, 40], 0))
    slot = ds.slot(2)
    X = torch.randn(ds.V, 16, device="cuda")
    Y = torch.randint(0, 5, (ds.V,), device="cuda")
    torch.cuda.synchronize()
    l0 = _launches()
    with pytest.raises(ValueError, match="at least one"):
        ds.slot(0)
    with pytest.raises(RuntimeError, match="unsupported"):
        ds.slot(1025)
    with pytest.raises(ValueError, match="no eigenpairs"):
        implicit_only.slot(1)
    with pytest.raises(RuntimeError, match="unsupported"):
        ds.slot(2, max_rows=2 ** 31)
    with pytest.raises(ValueError, match="more than int32"):
        ds.slot(2, max_entries=2 ** 31)
    with pytest.raises(IndexError, match="outside"):
        slot.fill([0, len(items)])
    with pytest.raises(ValueError, match="2 meshes"):
        slot.fill([0])
    big = int(np.argmax(ds.n_rows))
    with pytest.raises(ValueError, match="capacity"):
        slot.fill([big, big])
    with pytest.raises(ValueError, match="int64 tensor of shape"):
        slot.fill(torch.tensor([0, 1], device="cuda", dtype=torch.int32))
    with pytest.raises(ValueError, match="int64 tensor of shape"):
        slot.fill(torch.tensor([0, 1, 2], device="cuda"))
    with pytest.raises(ValueError, match="dataset layout"):
        slot.pack(X[:-1])
    with pytest.raises(ValueError, match="requires grad"):
        slot.pack(X.clone().requires_grad_(True))
    with pytest.raises(NotImplementedError):
        slot.pack([X[:10]])
    with pytest.raises(ValueError, match="one per dataset mesh"):
        slot.take(Y)
    for what in ("n_rows", "row_begin"):
        with pytest.raises(NotImplementedError, match="no host copy"):
            getattr(slot, what)
    with pytest.raises(NotImplementedError, match="no host copy"):
        slot.unpack(X)
    with pytest.raises(NotImplementedError, match="no host copy"):
        slot.elem_counts("faces")
    x = torch.zeros(slot.V, 16, device="cuda")
    with pytest.raises(NotImplementedError, match="forward_batch"):
        _net().forward_batch(slot, x)
    with pytest.raises(NotImplementedError, match="batch layout"):
        _net().forward_batch_nll(slot, x, [Y[:10], Y[:20]])
    with pytest.raises(NotImplementedError, match="per vertex"):
        _net(outputs_at="faces").forward_batch_nll(slot, x, torch.zeros(slot.V, dtype=torch.int64, device="cuda"))
    with pytest.raises(ValueError, match="int64 tensor of shape"):
        _net().forward_batch_nll(slot, x, torch.zeros(slot.V - 1, dtype=torch.int64, device="cuda"))
    torch.manual_seed(0)
    implicit = dn.DiffusionNet(C_in=16, C_out=4, C_width=32, N_block=1, dropout=False, outputs_at="global_mean",
                               diffusion_method="implicit_dense").cuda()
    with pytest.raises(NotImplementedError, match="spectral nets only"):
        implicit.forward_batch_global_nll(slot, x, torch.zeros(2, dtype=torch.int64, device="cuda"))
    assert _launches() == l0
