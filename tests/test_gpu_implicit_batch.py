"""Implicit heat diffusion over mesh batches (dn_implicit_diffusion_fwd_batched / _bwd_batched behind
ops.BatchedImplicitDiffusionFn and DiffusionNet.forward_batch*) against a dense fp64 solve per mesh, and the batch
routes of implicit nets against the per-mesh loop.

The gold solves (M_b + t_c L_b) y = M_b x per mesh and channel with numpy, from the fp32-rounded L and mass the GPU
sees (as tests/test_gpu_implicit.py does), and the adjoint for grad_x = M w and grad_time[c] = -sum_b w.(L_b y).  Bounds
are test_gpu_implicit.py's: 1e-5 for outputs, 1e-4 for parameter gradients, as max-abs error over max-abs gold.  Each
gold check has a negative control (one mesh's t perturbed, or one L row dropped) that must fail the same bound.  The
spill check runs on the CPU; everything else needs an H100."""
import ctypes as ct
import os
import re
import shutil
import subprocess
import sys
import warnings

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "oracle"))
from ref_import import _cotan_laplacian, _vertex_areas  # noqa: E402

import diffusion_net_b200 as dn  # noqa: E402

gpu = pytest.mark.gpu
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.mark.skipif(shutil.which(NVCC) is None and not os.path.exists(NVCC), reason="nvcc not found")
def test_batched_implicit_kernels_do_not_spill(tmp_path):
    flags = [f for f in dn._lib.NVCC_FLAGS if f != "-shared"]
    cmd = [NVCC] + flags + ["-Xptxas", "-v", "-c", os.path.join(dn._lib._CSRC, "dn_implicit_batch.cu"), "-o",
                            str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [l for l in (r.stdout + r.stderr).splitlines() if "spill stores" in l]
    assert len(lines) == 8                      # one per column-count instantiation
    for l in lines:
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", l)
        assert m and m.group(1) == "0" and m.group(2) == "0", l


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    dn._lib.load()
    return torch.device("cuda")


def _np(t):
    return t.detach().cpu().numpy().astype(np.float64)


def _err(mine, gold):
    mine, gold = np.asarray(mine, dtype=np.float64), np.asarray(gold, dtype=np.float64)
    return np.abs(mine - gold).max() / max(np.abs(gold).max(), 1e-30)


def _close(mine, gold, tol=1e-5):
    err = _err(mine, gold)
    assert err <= tol, err
    return err


# ---------------------------------------------------------------------------------------------------------------
# meshes, batches and the dense fp64 gold
# ---------------------------------------------------------------------------------------------------------------
def _mesh(kind, a, b, seed):
    if kind == "tri":                                   # one triangle: fewer rows than a warp's share of a chunk
        return torch.tensor([[0., 0., 0.], [1., 0., 0.], [0.2, 0.9, 0.1]]), torch.tensor([[0, 1, 2]])
    return (dn.synthetic.torus_mesh if kind == "torus" else dn.synthetic.patch_mesh)(a, b, seed=seed)


def _operators(verts, faces):
    """L (fp32-rounded, scipy fp64) and mass (fp32-rounded, fp64), normalised to unit max radius."""
    v = verts.numpy().astype(np.float64)
    v = v - v.mean(0)
    v /= np.linalg.norm(v, axis=1).max()
    f = faces.numpy()
    L = sp.csr_matrix(_cotan_laplacian(v, f, denom_eps=1e-10)).astype(np.float32).astype(np.float64)
    m = _vertex_areas(v, f)
    m = (m + 1e-8 * m.mean()).astype(np.float32).astype(np.float64)
    return L, m


def _sparse(M, device):
    c = M.tocoo()
    idx = torch.from_numpy(np.stack((c.row, c.col)).astype(np.int64))
    return torch.sparse_coo_tensor(idx, torch.from_numpy(c.data.astype(np.float32)), M.shape).coalesce().to(device)


def _meshes(spec, seed=0):
    """spec: list of (kind, a, b) -> list of (L, m)."""
    return [_operators(*_mesh(k, a, b, seed + i)) for i, (k, a, b) in enumerate(spec)]


def _batch(meshes, device):
    """A solve-only MeshBatch (no eigenpairs; the gradient operators are identities, unused by the solve)."""
    items = []
    for L, m in meshes:
        eye = _sparse(sp.identity(L.shape[0], format="csr"), device)
        items.append(dict(mass=torch.from_numpy(m.astype(np.float32)).to(device), L=_sparse(L, device), gradX=eye,
                          gradY=eye))
    return dn.batch.MeshBatch(items)


def _gold(meshes, xs, t, gs=None):
    """Per mesh: y (V_b, C), and with gs the adjoint grad_x and the mesh's grad_time contribution (C,)."""
    tc = np.maximum(t.astype(np.float64), 1e-8)
    out = []
    for (L, m), x, g in zip(meshes, xs, gs if gs is not None else [None] * len(xs)):
        Ld, M = L.toarray(), np.diag(m)
        y = np.empty(x.shape)
        gx = np.empty(x.shape)
        gt = np.empty(x.shape[1])
        for c in range(x.shape[1]):
            A = M + tc[c] * Ld
            y[:, c] = np.linalg.solve(A, m * x[:, c])
            if g is not None:
                w = np.linalg.solve(A.T, g[:, c])
                gx[:, c] = m * w
                gt[c] = -w @ (Ld @ y[:, c])
        out.append((y, gx, gt))
    return out


def _times(C, seed=0):
    """Diffusion times from 1e-8 to 1 (iteration counts differ by far more than 10x), one negative (clamped)."""
    t = np.logspace(-8, 0, C).astype(np.float32)
    np.random.RandomState(seed).shuffle(t)
    t[C // 2] = -0.25
    return t


def _inputs(meshes, C, seed):
    rs = np.random.RandomState(seed)
    xs = [rs.randn(L.shape[0], C).astype(np.float32) for L, _ in meshes]
    gs = [rs.randn(L.shape[0], C).astype(np.float32) for L, _ in meshes]
    return xs, gs


def _padding(batch):
    rows = np.ones(batch.V, dtype=bool)
    for r0, n in zip(batch.row_begin, batch.n_rows):
        rows[r0:r0 + n] = False
    return rows


def _solve(batch, xs, t, gs, device, grad_time0=None):
    """Forward and backward through ops.BatchedImplicitDiffusionFn: (y, grad_x, grad_time, time after, status fwd)."""
    time = torch.nn.Parameter(torch.from_numpy(t.copy()).to(device))
    if grad_time0 is not None:
        time.grad = torch.from_numpy(grad_time0.copy()).to(device)
    x = batch.pack([torch.from_numpy(v).to(device) for v in xs]).requires_grad_(True)
    y = dn.ops.BatchedImplicitDiffusionFn.apply(x, time, batch)
    st = dn.ops.implicit_last_status.clone()
    y.backward(batch.pack([torch.from_numpy(v).to(device) for v in gs]))
    return y.detach(), x.grad, time.grad, time.detach(), st


RAGGED = {
    "b1_c8": ([("torus", 12, 17)], 8),
    "b3_c40": ([("torus", 10, 13), ("tri", 0, 0), ("patch", 7, 9)], 40),
    "b3_c128": ([("patch", 9, 11), ("torus", 8, 15), ("tri", 0, 0)], 128),
    "b3_c256": ([("torus", 9, 10), ("tri", 0, 0), ("patch", 5, 6)], 256),
    "b32_c64": ([("torus", 10 + i % 7, 12 + (3 * i) % 11) if i % 4 else ("patch", 4 + i % 5, 5 + i % 3)
                 for i in range(31)] + [("tri", 0, 0)], 64),
    "b2_c16_large": ([("torus", 50, 60), ("tri", 0, 0)], 16),   # 94 chunks: one pair's sums span many chunks
    "b200_c8": ([("patch", 2 + i % 9, 3 + (5 * i) % 7) for i in range(199)] + [("tri", 0, 0)], 8),
}


@gpu
@pytest.mark.parametrize("case", sorted(RAGGED))
def test_ragged_batches_against_dense_gold(cuda, case):
    spec, C = RAGGED[case]
    meshes = _meshes(spec, seed=len(spec))
    assert any(L.shape[0] % 128 for L, _ in meshes)
    batch = _batch(meshes, cuda)
    t = _times(C)
    xs, gs = _inputs(meshes, C, seed=C)
    gt0 = np.linspace(-1, 1, C).astype(np.float32)         # grad_time accumulates into what is there
    y, gx, gtime, tafter, st = _solve(batch, xs, t, gs, cuda, grad_time0=gt0)
    gold = _gold(meshes, xs, t, gs)
    gy = np.concatenate([g[0] for g in gold])
    ggx = np.concatenate([g[1] for g in gold])
    ggt = sum(g[2] for g in gold)
    my_y = np.concatenate([_np(v) for v in batch.unpack(y)])
    my_gx = np.concatenate([_np(v) for v in batch.unpack(gx)])
    e = (_close(my_y, gy), _close(my_gx, ggx), _close(_np(gtime) - gt0, ggt, tol=1e-4))
    print("{}: errors y {:.2e} grad_x {:.2e} grad_time {:.2e}; iterations {}..{}".format(
        case, *e, int(st[2:2 + len(meshes) * C].min()), int(st[1])))
    # negative control: the gold with one mesh's t perturbed by 1 % fails the bound
    tb = t.copy()
    tb[np.argmax(t)] *= 1.01
    bad = _gold(meshes[-2:-1] if len(meshes) > 1 else meshes, xs[-2:-1] if len(meshes) > 1 else xs, tb)
    sl = batch.unpack(y)[-2 if len(meshes) > 1 else 0]
    assert _err(_np(sl), bad[0][0]) > 1e-5
    # padding rows are exact zeros; the clamp is written back once (a negative t ends at 1e-8)
    pad = _padding(batch)
    if pad.any():
        assert (y.cpu().numpy()[pad] == 0).all() and (gx.cpu().numpy()[pad] == 0).all()
    want_t = np.maximum(t, np.float32(1e-8))
    assert np.array_equal(tafter.cpu().numpy(), want_t)
    # per-pair iteration counts differ by more than 10x within the batch
    its = st[2:2 + len(meshes) * C].numpy()
    assert its.max() > 10 * max(its[its > 0].min(), 1)


def _dropped_row(L, r):
    Lc = L.tolil()
    Lc[r, :] = 0
    return Lc.tocsr()


@gpu
def test_negative_control_dropped_row(cuda):
    meshes = _meshes([("torus", 10, 13), ("patch", 7, 9)])
    C = 16
    batch = _batch(meshes, cuda)
    t = _times(C)
    xs, gs = _inputs(meshes, C, seed=1)
    y = _solve(batch, xs, t, gs, cuda)[0]
    _close(_np(batch.unpack(y)[1]), _gold(meshes[1:], xs[1:], t)[0][0])
    bad = _gold([(_dropped_row(meshes[1][0], 5), meshes[1][1])], xs[1:], t)[0][0]
    assert _err(_np(batch.unpack(y)[1]), bad) > 1e-5


@gpu
def test_independence_of_a_slow_mesh(cuda):
    C = 32
    base = [("torus", 10, 13), ("patch", 6, 7), ("tri", 0, 0)]
    meshes = _meshes(base)
    slow = _meshes([("torus", 50, 70)], seed=9)           # 3500 rows: many more iterations at t ~ 1
    t = _times(C)
    xs, gs = _inputs(meshes + slow, C, seed=2)
    a = _solve(_batch(meshes, cuda), xs[:3], t, gs[:3], cuda)
    bb = _batch(meshes + slow, cuda)
    b = _solve(bb, xs, t, gs, cuda)
    P = 3 * C
    its_a, its_b = a[4][2:2 + P].numpy(), b[4][2:2 + P].numpy()
    assert np.array_equal(its_a, its_b)
    assert b[4][1] > 2 * a[4][1]                          # the slow mesh did need more iterations
    ba = _batch(meshes, cuda)
    for k in range(3):
        _close(_np(bb.unpack(b[0])[k]), _np(ba.unpack(a[0])[k]))
        _close(_np(bb.unpack(b[1])[k]), _np(ba.unpack(a[1])[k]))


@gpu
def test_nan_in_one_pair(cuda):
    meshes = _meshes([("torus", 10, 13), ("patch", 7, 9), ("torus", 8, 9)])
    C = 40
    batch = _batch(meshes, cuda)
    t = _times(C)
    xs, gs = _inputs(meshes, C, seed=3)
    xs[1][4, 33] = np.nan
    y = _solve(batch, xs, t, gs, cuda)[0]
    gold = _gold(meshes, xs, t)
    for b, (yb, g) in enumerate(zip(batch.unpack(y), gold)):
        yb = _np(yb)
        if b == 1:
            assert np.isnan(yb[:, 33]).all()
            yb, gy = np.delete(yb, 33, 1), np.delete(g[0], 33, 1)
        else:
            gy = g[0]
        assert np.isfinite(yb).all()
        _close(yb, gy)


@gpu
def test_non_convergence_raises_and_writes_nothing(cuda, monkeypatch):
    # only mesh 1 can be stuck: CG on a 3-vertex mesh ends within a few iterations, the 1200-vertex torus at t = 0.5
    # needs far more than 12
    meshes = _meshes([("tri", 0, 0), ("torus", 30, 40), ("tri", 0, 0)])
    Cc = 8
    batch = _batch(meshes, cuda)
    t = np.full(Cc, 0.5, dtype=np.float32)
    t[0] = 1e-8                                            # converges at once everywhere
    xs, _ = _inputs(meshes, Cc, seed=4)
    x = batch.pack([torch.from_numpy(v).to(cuda) for v in xs])
    time = torch.from_numpy(t).to(cuda)
    y = torch.full_like(x, 7.0)
    lib = dn._lib.load()
    monkeypatch.setattr(dn.ops, "IMPLICIT_MAX_ITER", 12)
    with pytest.raises(RuntimeError, match=r"did not converge in 12 iterations, in meshes \[1\] "):
        dn.ops._implicit_call("dn_implicit_diffusion_fwd_batched", lib.dn_implicit_diffusion_fwd_batched, batch.V, Cc,
                              cuda, (ct.byref(batch.lap.csr[0]), x.data_ptr(), batch.mass.data_ptr(), time.data_ptr(),
                                     ct.byref(batch.desc), batch._mesh_rows.data_ptr(), batch.V, Cc), (y.data_ptr(),),
                              n_meshes=batch.n_meshes)
    torch.cuda.synchronize()
    assert (y == 7.0).all()
    st = dn.ops.implicit_last_status
    its, res = st[2:2 + 3 * Cc].view(3, Cc), st[2 + 3 * Cc:].view(3, Cc)
    stuck = (its >= 12) & (res > dn.ops.IMPLICIT_RTOL)
    assert int(st[0]) == int(stuck.sum()) == 7              # every channel of mesh 1 but the t = 1e-8 one
    assert stuck[1, 1:].all() and not stuck[0].any() and not stuck[2].any()
    with pytest.raises(RuntimeError, match="did not converge"):
        dn.ops.BatchedImplicitDiffusionFn.apply(x, time, batch)


@gpu
def test_1024_meshes(cuda):
    spec = [("tri", 0, 0) if i % 97 == 0 else ("patch", 2 + i % 5, 2 + (7 * i) % 5) for i in range(1024)]
    meshes = _meshes(spec)
    C = 8
    batch = _batch(meshes, cuda)
    assert batch.n_meshes == 1024
    t = _times(C)
    xs, gs = _inputs(meshes, C, seed=5)
    y, gx, gtime, _, _ = _solve(batch, xs, t, gs, cuda)
    gold = _gold(meshes, xs, t, gs)
    _close(np.concatenate([_np(v) for v in batch.unpack(y)]), np.concatenate([g[0] for g in gold]))
    _close(np.concatenate([_np(v) for v in batch.unpack(gx)]), np.concatenate([g[1] for g in gold]))
    _close(_np(gtime), sum(g[2] for g in gold), tol=1e-4)


@gpu
def test_two_calls_are_bitwise_equal(cuda):
    meshes = _meshes([("torus", 10, 13), ("patch", 7, 9), ("tri", 0, 0), ("torus", 12, 15)])
    C = 64
    batch = _batch(meshes, cuda)
    t = _times(C)
    xs, gs = _inputs(meshes, C, seed=6)
    a, b = _solve(batch, xs, t, gs, cuda), _solve(batch, xs, t, gs, cuda)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


@gpu
def test_one_launch_and_one_status_read_per_solve(cuda):
    lib = dn._lib.load()
    C = 16
    t = _times(C)
    counts = {}
    for nb in (3, 200):
        meshes = _meshes([("patch", 3 + i % 6, 4 + i % 5) for i in range(nb)])
        batch = _batch(meshes, cuda)
        xs, gs = _inputs(meshes, C, seed=7)
        x = batch.pack([torch.from_numpy(v).to(cuda) for v in xs])
        time = torch.from_numpy(t).to(cuda)
        assert batch.lap is not None                        # the batch Laplacian is built once, before counting
        torch.cuda.synchronize()
        n0 = lib.dn_kernel_launch_count()
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                dn.ops.BatchedImplicitDiffusionFn.apply(x, time, batch)
            finally:
                torch.cuda.set_sync_debug_mode("default")
        counts[nb] = (lib.dn_kernel_launch_count() - n0, sum("called a synchronizing" in str(x.message) for x in w))
    assert counts[3] == counts[200] == (1, 1), counts


# ---------------------------------------------------------------------------------------------------------------
# whole nets: the batch routes against the per-mesh loop
# ---------------------------------------------------------------------------------------------------------------
def _net_meshes(cuda):
    out = []
    for i, (kind, a, b) in enumerate([("torus", 10, 14), ("patch", 9, 12), ("torus", 13, 17), ("patch", 6, 8),
                                      ("torus", 9, 11)]):
        v, f = _mesh(kind, a, b, 20 + i)
        v = v - v.mean(0)
        v = v / v.norm(dim=1).max()
        frames, mass, L, evals, evecs, gX, gY = dn.geometry.compute_operators(v.to(cuda), f.to(cuda), k_eig=4)
        out.append(dict(verts=v.to(cuda), faces=f.to(cuda), mass=mass, L=L, gradX=gX, gradY=gY))
    return out


def _implicit_net(C, rot, outputs_at="vertices", C_out=5):
    torch.manual_seed(C + rot)
    net = dn.DiffusionNet(C_in=3, C_out=C_out, C_width=C, N_block=2, dropout=False, outputs_at=outputs_at,
                          with_gradient_rotations=rot, diffusion_method="implicit_dense")
    with torch.no_grad():
        for blk in net.blocks:
            blk.diffusion.diffusion_time.copy_(torch.logspace(-4, -0.5, C)[torch.randperm(C)])
    return net


def _implicit_batch(ms):
    return dn.batch.MeshBatch([dict(mass=m["mass"], L=m["L"], gradX=m["gradX"], gradY=m["gradY"], faces=m["faces"])
                               for m in ms])


def _grads(net):
    return {k: p.grad.detach().clone() for k, p in net.named_parameters()}


def _compare_grads(ga, gb):
    for k in ga:
        _close(_np(ga[k]), _np(gb[k]), tol=1e-4)


@gpu
@pytest.mark.parametrize("C,rot", [(32, True), (64, False), (64, True)])
def test_forward_batch_matches_loop(cuda, C, rot):
    ms = _net_meshes(cuda)
    batch = _implicit_batch(ms)
    net = _implicit_net(C, rot).to(cuda)
    xs = [m["verts"].clone().requires_grad_(True) for m in ms]
    kw = lambda m: dict(L=m["L"], gradX=m["gradX"], gradY=m["gradY"])
    net.eval()
    with torch.no_grad():
        loop = [net(x, m["mass"], **kw(m)) for x, m in zip(xs, ms)]
        outs = net.forward_batch(batch, [x.detach() for x in xs])
    for a, b in zip(outs, loop):
        _close(_np(a), _np(b))
    net.train()
    gouts = [torch.randn_like(o) for o in loop]
    net.zero_grad()
    sum((net(x, m["mass"], **kw(m)) * g).sum() for x, m, g in zip(xs, ms, gouts)).backward()
    g_loop, x_loop = _grads(net), [x.grad.clone() for x in xs]
    net.zero_grad()
    for x in xs:
        x.grad = None
    outs = net.forward_batch(batch, xs)
    sum((o * g).sum() for o, g in zip(outs, gouts)).backward()
    _compare_grads(_grads(net), g_loop)
    for x, gl in zip(xs, x_loop):
        _close(_np(x.grad), _np(gl), tol=1e-4)


@gpu
@pytest.mark.parametrize("outputs_at", ["vertices", "faces"])
def test_forward_batch_nll_matches_loop(cuda, outputs_at):
    ms = _net_meshes(cuda)
    batch = _implicit_batch(ms)
    net = _implicit_net(32, True, outputs_at=outputs_at).to(cuda)
    rs = np.random.RandomState(8)
    n_el = lambda m: m["faces"].shape[0] if outputs_at == "faces" else m["mass"].shape[0]
    labels = [torch.from_numpy(rs.randint(0, 5, n_el(m))).to(cuda) for m in ms]
    xs = [m["verts"].clone().requires_grad_(True) for m in ms]
    net.zero_grad()
    loop = [net.forward_nll(x, m["mass"], L=m["L"], gradX=m["gradX"], gradY=m["gradY"], labels=l, faces=m["faces"])[0]
            for x, m, l in zip(xs, ms, labels)]
    sum(loop).backward()
    g_loop, x_loop = _grads(net), [x.grad.clone() for x in xs]
    net.zero_grad()
    for x in xs:
        x.grad = None
    losses, _ = net.forward_batch_nll(batch, xs, labels)
    losses.sum().backward()
    _close(_np(losses), np.array([float(v) for v in loop]))
    _compare_grads(_grads(net), g_loop)
    for x, gl in zip(xs, x_loop):
        _close(_np(x.grad), _np(gl), tol=1e-4)


@gpu
def test_forward_batch_global_nll_matches_loop(cuda):
    ms = _net_meshes(cuda)
    batch = _implicit_batch(ms)
    net = _implicit_net(64, True, outputs_at="global_mean", C_out=30).to(cuda)
    labels = torch.tensor([3, 17, 0, 29, 8], device=cuda)
    xs = [m["verts"].clone().requires_grad_(True) for m in ms]
    net.zero_grad()
    loop = [net.forward_global_nll(x, m["mass"], L=m["L"], gradX=m["gradX"], gradY=m["gradY"], labels=labels[b:b + 1],
                                   label_smoothing=0.2)[0] for b, (x, m) in enumerate(zip(xs, ms))]
    sum(loop).backward()
    g_loop, x_loop = _grads(net), [x.grad.clone() for x in xs]
    net.zero_grad()
    for x in xs:
        x.grad = None
    losses, _ = net.forward_batch_global_nll(batch, xs, labels, label_smoothing=0.2)
    losses.sum().backward()
    _close(_np(losses), np.array([float(v) for v in loop]))
    _compare_grads(_grads(net), g_loop)
    for x, gl in zip(xs, x_loop):
        _close(_np(x.grad), _np(gl), tol=1e-4)


@gpu
def test_refusals(cuda):
    ms = _net_meshes(cuda)[:2]
    implicit = _implicit_net(32, True).to(cuda)
    spectral = dn.DiffusionNet(C_in=3, C_out=5, C_width=32, N_block=2, dropout=False).to(cuda)
    l_only = _implicit_batch(ms)
    assert l_only.K == 0
    xs = [m["verts"] for m in ms]
    labels = [torch.zeros(m["mass"].shape[0], dtype=torch.int64, device=cuda) for m in ms]
    with pytest.raises(ValueError, match="eigenpairs"):
        spectral.forward_batch(l_only, xs)
    with pytest.raises(ValueError, match="eigenpairs"):
        spectral.forward_batch_nll(l_only, xs, labels)
    no_l = dn.batch.MeshBatch([dict(mass=m["mass"], evals=torch.zeros(4, device=cuda),
                                    evecs=torch.zeros(m["mass"].shape[0], 4, device=cuda), gradX=m["gradX"],
                                    gradY=m["gradY"]) for m in ms])
    assert no_l.lap is None
    for batch in (no_l, None):
        with pytest.raises(NotImplementedError, match="Laplacian"):
            implicit.forward_batch(batch, xs)
        with pytest.raises(NotImplementedError, match="Laplacian"):
            implicit.forward_batch_nll(batch, xs, labels)
    glob = _implicit_net(32, True, outputs_at="global_mean").to(cuda)
    with pytest.raises(NotImplementedError, match="Laplacian"):
        glob.forward_batch_global_nll(no_l, xs, torch.zeros(2, dtype=torch.int64, device=cuda))
    with pytest.raises(NotImplementedError):
        dn.graphs.GraphedBatch(implicit, l_only)
    with pytest.raises(NotImplementedError):
        dn.graphs.GraphedTrainStep(implicit, lambda n, *a: n(*a).sum(), (xs[0], ms[0]["mass"]))
    with pytest.raises(ValueError, match="every item or for none"):
        dn.batch.MeshBatch([dict(mass=ms[0]["mass"], L=ms[0]["L"], gradX=ms[0]["gradX"], gradY=ms[0]["gradY"]),
                            dict(mass=ms[1]["mass"], evals=torch.zeros(0, device=cuda),
                                 evecs=torch.zeros(ms[1]["mass"].shape[0], 0, device=cuda), gradX=ms[1]["gradX"],
                                 gradY=ms[1]["gradY"])])
