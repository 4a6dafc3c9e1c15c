"""Training over a batch of meshes in one launch sequence: the batched spectral diffusion C-ABI calls
(dn_learned_time_diffusion_{fwd,bwd}_batched) against the per-mesh calls, and DiffusionNet.forward_batch under
autograd against the fp64 oracle accumulated over the same meshes.

Ragged batches: meshes whose V is not a multiple of 128, one with V < 128 where the eigenbasis allows it (V >= K)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle as O  # noqa: E402  (checker only)

pytestmark = pytest.mark.gpu

RAGGED = {64: [(36, 50), (12, 11), (44, 50), (8, 10)],      # 80 vertices: a mesh shorter than one 128-row tile
          128: [(36, 50), (12, 11), (44, 50), (16, 8)]}
# batched vs per-mesh, the same engine: both sides round the same operands, only the partial-sum order differs
DIFF_TOL = {"tc3x": 1e-5, "tc1x": 1e-3, "bf16": 2e-2}
SMALL = [(12, 11), (8, 10)]        # padded V = 384


@pytest.fixture(scope="module")
def dn():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import diffusion_net_b200 as d
    d._lib.load()
    yield d
    d.set_engine("tc3x")


def _meshes(dn, shapes, K, seed=0):
    out = []
    for i, (n, m) in enumerate(shapes):
        mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=seed + i, device="cuda")
        _, faces = dn.synthetic.torus_mesh(n, m, seed=seed + i)
        out.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY, faces=faces.cuda()))
    return out


def _net(dn, C, K, C_out=5, n_block=2, dropout=False, outputs_at="vertices", seed=0):
    torch.manual_seed(seed)
    net = dn.DiffusionNet(C_in=16, C_out=C_out, C_width=C, N_block=n_block, dropout=dropout,
                          outputs_at=outputs_at).cuda().train()
    with torch.no_grad():
        for n_, p_ in net.named_parameters():
            if n_.endswith("diffusion_time"):
                p_.uniform_(1e-3, 0.3)
    return net


def _inputs(meshes, C_in=16, C_out=5, seed=0):
    xs, ys = [], []
    for i, it in enumerate(meshes):
        g = torch.Generator().manual_seed(100 + seed + i)
        V = it["mass"].shape[0]
        xs.append(torch.randn(V, C_in, generator=g).cuda())
        ys.append(torch.randint(0, C_out, (V,), generator=g).cuda())
    return xs, ys


def _grads(net):
    return {n_: p_.grad.clone() for n_, p_ in net.named_parameters()}


def _zero(net):
    for p_ in net.parameters():
        p_.grad = None


# ---- 1. the C-ABI calls against the per-mesh calls -------------------------------------------------------------
def _ws(dn, V, K, C_, extra=0):
    return dn.ops.workspace(V, K, C_, torch.device("cuda", torch.cuda.current_device()), extra=extra)


@pytest.mark.parametrize("engine", ["tc3x", "tc1x", "bf16"])
@pytest.mark.parametrize("C_,K", [(64, 64), (128, 128), (256, 128)])
def test_batched_diffusion_capi_vs_per_mesh(dn, engine, C_, K):
    lib = dn._lib.load()
    eng = dn.ops._ENGINES[engine]
    st = dn.ops._stream()
    meshes = _meshes(dn, RAGGED[K], K, seed=3)
    mb = dn.MeshBatch(meshes)
    V, B = mb.V, mb.n_meshes
    g = torch.Generator().manual_seed(7)
    time0 = (torch.rand(C_, generator=g) * 0.3).cuda()
    time0[:3] = torch.tensor([-0.1, 0.0, 1e-9])                # clamped to 1e-8 in place
    # finite garbage in the padding rows: neither call may read them
    x = torch.randn(V, C_, generator=g).cuda()
    gout = torch.randn(V, C_, generator=g).cuda()
    pad = torch.ones(V, dtype=torch.bool, device="cuda")
    for b in range(B):
        pad[mb.row_begin[b]:mb.row_begin[b] + mb.n_rows[b]] = False
    assert pad.any()

    t_b = time0.clone()
    xd = torch.empty_like(x)
    xspec = torch.empty(B, K, C_, device="cuda")
    ws = _ws(dn, V, K, C_, dn.ops.batched_diffusion_workspace_extra(B, K, C_))
    l0 = lib.dn_kernel_launch_count()
    dn._lib.check(lib.dn_learned_time_diffusion_fwd_batched(
        x.data_ptr(), mb.mass.data_ptr(), mb.evals.data_ptr(), mb.evecs.data_ptr(), t_b.data_ptr(), C.byref(mb.desc),
        V, K, C_, xd.data_ptr(), xspec.data_ptr(), ws.data_ptr(), ws.numel(), eng, st), "fwd_batched")
    l1 = lib.dn_kernel_launch_count()
    gx = torch.full_like(x, float("nan"))
    gt = torch.zeros(C_, device="cuda")
    dn._lib.check(lib.dn_learned_time_diffusion_bwd_batched(
        gout.data_ptr(), mb.mass.data_ptr(), mb.evals.data_ptr(), mb.evecs.data_ptr(), t_b.data_ptr(),
        xspec.data_ptr(), C.byref(mb.desc), V, K, C_, gx.data_ptr(), gt.data_ptr(), ws.data_ptr(), ws.numel(), eng, st),
        "bwd_batched")
    l2 = lib.dn_kernel_launch_count()
    # a fixed launch sequence: to_basis (two 128-column launches at C = 256), pack, from_basis (+ time gradient)
    extra = 1 if C_ > 128 else 0
    assert (l1 - l0, l2 - l1) == (3 + extra, 4 + extra)

    t_m = time0.clone()
    gt_m = torch.zeros(C_, device="cuda")
    ref_xd, ref_xs, ref_gx = [], [], []
    for b, it in enumerate(meshes):
        r0, n = mb.row_begin[b], mb.n_rows[b]
        xb, gb = x[r0:r0 + n].contiguous(), gout[r0:r0 + n].contiguous()
        xd_b, gx_b = torch.empty_like(xb), torch.empty_like(xb)
        xs_b = torch.empty(K, C_, device="cuda")
        t_in = t_m.clone()                                   # every mesh sees the unclamped time, as in the batch
        wsb = _ws(dn, n, K, C_)
        dn._lib.check(lib.dn_learned_time_diffusion_fwd(
            xb.data_ptr(), it["mass"].data_ptr(), it["evals"].data_ptr(), it["evecs"].data_ptr(), t_in.data_ptr(), n,
            K, C_, xd_b.data_ptr(), xs_b.data_ptr(), wsb.data_ptr(), wsb.numel(), eng, st), "fwd")
        dn._lib.check(lib.dn_learned_time_diffusion_bwd(
            gb.data_ptr(), it["mass"].data_ptr(), it["evals"].data_ptr(), it["evecs"].data_ptr(), t_in.data_ptr(),
            xs_b.data_ptr(), n, K, C_, gx_b.data_ptr(), gt_m.data_ptr(), wsb.data_ptr(), wsb.numel(), eng, st), "bwd")
        ref_xd.append(xd_b); ref_xs.append(xs_b); ref_gx.append(gx_b)
    t_m = t_in
    torch.cuda.synchronize()

    tol = DIFF_TOL[engine]
    assert torch.equal(t_b, t_m) and torch.equal(t_b, time0.clamp(min=1e-8))
    for b in range(B):
        r0, n = mb.row_begin[b], mb.n_rows[b]
        assert O.rel_err(xd[r0:r0 + n].cpu().numpy(), ref_xd[b].cpu().numpy()) < tol, b
        assert O.rel_err(xspec[b].cpu().numpy(), ref_xs[b].cpu().numpy()) < tol, b
        assert O.rel_err(gx[r0:r0 + n].cpu().numpy(), ref_gx[b].cpu().numpy()) < tol, b
    assert O.rel_err(gt.cpu().numpy(), gt_m.cpu().numpy()) < tol
    assert bool((xd[pad] == 0).all()) and bool((gx[pad] == 0).all())


# ---- 2. net gradients against the fp64 oracle accumulated over the meshes -------------------------------------
def _oracle_grads(net, meshes, xs, ys, outputs_at, NB):
    import dn_oracle_torch as T
    d = torch.float64
    prm = {k: v.detach().cpu().to(d).requires_grad_(True) for k, v in net.state_dict().items()}
    xgs = [x.detach().cpu().to(d).requires_grad_(True) for x in xs]
    for it, xg, y in zip(meshes, xgs, ys):
        mass, evals, evecs = (it[k].cpu().to(d) for k in ("mass", "evals", "evecs"))
        h = torch.addmm(prm["first_lin.bias"], xg, prm["first_lin.weight"].t()).unsqueeze(0)
        for b in range(NB):
            bp = {k[len("block_%d." % b):]: v for k, v in prm.items() if k.startswith("block_%d." % b)}
            h = T.block_forward(h, mass.unsqueeze(0), evals.unsqueeze(0), evecs.unsqueeze(0),
                                [it["gradX"].cpu().to(d)], [it["gradY"].cpu().to(d)], bp)
        logits = torch.addmm(prm["last_lin.bias"], h[0], prm["last_lin.weight"].t())
        torch.nn.functional.cross_entropy(_remap(logits, it, outputs_at, mass), y.cpu()).backward()
    return {k: v.grad for k, v in prm.items()}, [x.grad for x in xgs]


def _remap(out, it, outputs_at, mass):
    if outputs_at == "faces":
        return out[it["faces"].to(out.device)].mean(dim=1)
    if outputs_at == "global_mean":
        return (out * (mass / mass.sum()).unsqueeze(-1)).sum(dim=-2, keepdim=True)
    return out


def _targets(meshes, ys, outputs_at, C_out):
    if outputs_at == "faces":
        return [torch.randint(0, C_out, (it["faces"].shape[0],), generator=torch.Generator().manual_seed(i)).cuda()
                for i, it in enumerate(meshes)]
    if outputs_at == "global_mean":
        return [y[:1] for y in ys]
    return ys


def _batched_loss(outs, ys, outputs_at):
    if outputs_at == "global_mean":
        outs = [o.unsqueeze(0) for o in outs]
    return sum(torch.nn.functional.cross_entropy(o, y) for o, y in zip(outs, ys))


@pytest.mark.parametrize("outputs_at", ["vertices", "faces", "global_mean"])
def test_forward_batch_gradients_vs_oracle_accumulation(dn, outputs_at):
    dn.set_engine("tc3x")
    C_, K, NB, C_out = 64, 64, 2, 5
    net = _net(dn, C_, K, C_out, NB, outputs_at=outputs_at)
    meshes = _meshes(dn, RAGGED[K], K)
    mb = dn.MeshBatch(meshes)
    xs, ys = _inputs(meshes, C_out=C_out)
    ys = _targets(meshes, ys, outputs_at, C_out)
    xs = [x.clone().requires_grad_(True) for x in xs]
    _zero(net)
    outs = net.forward_batch(mb, xs)
    _batched_loss(outs, ys, outputs_at).backward()
    gold, gold_x = _oracle_grads(net, meshes, xs, ys, outputs_at, NB)
    for name, p_ in net.named_parameters():
        assert p_.grad is not None, name
        assert O.rel_err(p_.grad.cpu().numpy(), gold[name].numpy()) < 5e-5, name
    for b, (x, gx) in enumerate(zip(xs, gold_x)):
        assert O.rel_err(x.grad.cpu().numpy(), gx.numpy()) < 5e-5, b


@pytest.mark.parametrize("engine,C_,tol", [("bf16", 128, 2e-2), ("tc3x", 256, 1e-4)])
def test_forward_batch_gradients_vs_per_mesh(dn, engine, C_, tol):
    """bf16: the same engine's per-mesh route (the fp64 bound of bf16 is its own test); C_width = 256 (K = 128)."""
    dn.set_engine(engine)
    K = 128
    net = _net(dn, C_, K)
    meshes = _meshes(dn, RAGGED[K], K)
    mb = dn.MeshBatch(meshes)
    xs, ys = _inputs(meshes)
    _zero(net)
    for it, x, y in zip(meshes, xs, ys):
        out = net(x, it["mass"], evals=it["evals"], evecs=it["evecs"], gradX=it["gradX"], gradY=it["gradY"])
        torch.nn.functional.cross_entropy(out, y).backward()
    ref = _grads(net)
    _zero(net)
    _batched_loss(net.forward_batch(mb, xs), ys, "vertices").backward()
    for name, p_ in net.named_parameters():
        assert O.rel_err(p_.grad.cpu().numpy(), ref[name].cpu().numpy()) < tol, name


# ---- 3. padding rows never reach a real row --------------------------------------------------------------------
def test_padding_rows_are_isolated(dn):
    dn.set_engine("tc3x")
    net = _net(dn, 64, 64)
    meshes = _meshes(dn, SMALL, 64)
    mb = dn.MeshBatch(meshes)
    assert mb.V <= 512 and mb.V > sum(mb.n_rows)
    xs, ys = _inputs(meshes)
    clean = mb.pack(xs)
    dirty = clean.clone()
    g = torch.Generator().manual_seed(9)
    for b in range(mb.n_meshes):
        end = mb.row_begin[b + 1]
        r1 = mb.row_begin[b] + mb.n_rows[b]
        dirty[r1:end] = torch.randn(end - r1, 16, generator=g).cuda() * 3.0
    runs = []
    for x in (clean, dirty):
        _zero(net)
        outs = net.forward_batch(mb, x)
        _batched_loss(outs, ys, "vertices").backward()
        runs.append(([o.detach().clone() for o in outs], _grads(net)))
    (o0, g0), (o1, g1) = runs
    assert all(torch.equal(a, b) for a, b in zip(o0, o1))
    for name in g0:
        assert torch.equal(g0[name], g1[name]), name


# ---- 4. one launch sequence whatever the mesh count ------------------------------------------------------------
def test_launch_count_independent_of_mesh_count(dn):
    dn.set_engine("tc3x")
    lib = dn._lib.load()
    net = _net(dn, 64, 64)
    meshes = _meshes(dn, [(10 + i, 9) for i in range(6)], 64)
    xs, ys = _inputs(meshes)

    def batched(n):
        mb = dn.MeshBatch(meshes[:n])
        counts = []
        for _ in range(2):                               # the first step also builds the transposed CSR
            _zero(net)
            l0 = lib.dn_kernel_launch_count()
            _batched_loss(net.forward_batch(mb, xs[:n]), ys[:n], "vertices").backward()
            counts.append(lib.dn_kernel_launch_count() - l0)
        return counts[-1]

    def per_mesh():
        counts = []
        for _ in range(2):                               # the first step also prepares the operators
            _zero(net)
            l0 = lib.dn_kernel_launch_count()
            for it, x, y in zip(meshes, xs, ys):
                out = net(x, it["mass"], evals=it["evals"], evecs=it["evecs"], gradX=it["gradX"], gradY=it["gradY"])
                torch.nn.functional.cross_entropy(out, y).backward()
            counts.append(lib.dn_kernel_launch_count() - l0)
        return counts[-1]

    n2, n6, loop6 = batched(2), batched(6), per_mesh()
    assert n2 == n6, (n2, n6)
    assert n6 < loop6, (n6, loop6)


# ---- 5. determinism and CUDA-graph capture ---------------------------------------------------------------------
def test_batched_step_determinism_and_graphed_train_step(dn):
    dn.set_engine("tc3x")
    net = _net(dn, 128, 128)
    meshes = _meshes(dn, RAGGED[128], 128)
    mb = dn.MeshBatch(meshes)
    xs, ys = _inputs(meshes)

    def loss_fn(net_, xs_, ys_):
        return _batched_loss(net_.forward_batch(mb, xs_), ys_, "vertices")

    steps = []
    for _ in range(2):
        _zero(net)
        loss_fn(net, xs, ys).backward()
        steps.append(_grads(net))
    for b in range(len(net.blocks)):
        name = "block_%d.diffusion.diffusion_time" % b
        assert torch.equal(steps[0][name], steps[1][name]), name
    ref = steps[0]
    gts = dn.graphs.GraphedTrainStep(net, loss_fn, (xs, ys))
    for _ in range(2):
        dn.graphs.GraphedTrainStep.zero_grads(net)
        loss = gts.replay()
        torch.cuda.synchronize()
        assert torch.isfinite(loss)
        for name, p_ in net.named_parameters():
            assert torch.equal(p_.grad, ref[name]), name
    gts.replay()                                          # no zeroing: the gradients accumulate
    torch.cuda.synchronize()
    for name, p_ in net.named_parameters():
        assert torch.equal(p_.grad, 2 * ref[name]), name


# ---- 6. dropout and errors -------------------------------------------------------------------------------------
def test_dropout_under_autograd_is_seeded(dn):
    dn.set_engine("tc3x")
    net = _net(dn, 64, 64, dropout=True)
    meshes = _meshes(dn, SMALL, 64)
    mb = dn.MeshBatch(meshes)
    xs, ys = _inputs(meshes)
    runs = []
    for _ in range(2):
        torch.manual_seed(77)
        _zero(net)
        outs = net.forward_batch(mb, xs)
        _batched_loss(outs, ys, "vertices").backward()
        runs.append(([o.detach().clone() for o in outs], _grads(net)))
    (o0, g0), (o1, g1) = runs
    assert all(torch.equal(a, b) for a, b in zip(o0, o1))
    for name in g0:
        assert torch.equal(g0[name], g1[name]), name
    net.eval()
    with torch.no_grad():
        oe = net.forward_batch(mb, xs)
    assert any(not torch.allclose(a, b) for a, b in zip(o0, oe))


def test_simt_engine_is_refused_before_any_launch(dn):
    lib = dn._lib.load()
    meshes = _meshes(dn, SMALL, 64)
    mb = dn.MeshBatch(meshes)
    x = torch.randn(mb.V, 64, device="cuda", requires_grad=True)
    t = torch.full((64,), 0.1, device="cuda", requires_grad=True)
    dn.set_engine("simt")
    try:
        torch.cuda.synchronize()
        l0 = lib.dn_kernel_launch_count()
        with pytest.raises(RuntimeError, match="unsupported"):
            dn.ops.BatchedDiffusionFn.apply(x, t, mb)
        assert lib.dn_kernel_launch_count() == l0
    finally:
        dn.set_engine("tc3x")
