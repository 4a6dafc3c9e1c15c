"""The fused inference forward (block_fwd_impl behind dn_block_fwd, dn_block_fwd_ex and dn_block_fwd_batched) on every
engine, at each branch of its dispatch, against ``oracle/dn_oracle_engines``: the same block in fp64 with every
tensor-core operand rounded where the kernels round it.

Metric.  The block output is x_in + MLP(...), and the skip connection dominates it (max|out| = 4.7 against
max|MLP branch| = 0.43 at V = 7000, C = 128), so errors are measured on the branch: max|(out - x_in) - (gold - x_in)|
over max|gold - x_in|.  Net outputs with a head have no skip and are measured as they are.

Bound.  FLOOR_C[engine] times the error of the same emulated computation evaluated in float32 on the CPU (the fp32
floor).  That evaluation rounds its own fp32 intermediates (S, x_diffuse, hidden activations) to TF32 / bf16 where the
GPU does, so where an fp32 intermediate lies next to a rounding boundary it flips as the GPU's may, and its error
carries a sample of those flips.  At small V the sample can be empty, so the single-pass engines' floor is at least
FLIP_FLOOR = one rounding unit of their format (2^-11 TF32, 2^-8 bf16) of max|branch|: one flipped operand moves an
output by one rounding step of the operand times one weight.  (A propagated per-element flip allowance -- one rounding
step for every operand within an fp32 margin of a boundary, pushed through |W| and the gather -- came out at 0.8 to
1.8 x max|branch| for tc1x and bf16, as loose as a componentwise bound: the gradient operators amplify it.)

FLOOR_C = 4 on every engine but tc3x.  tc3x: measured on an H100 80GB HBM3 at a 400 W power limit, the block error is
6 - 15x its fp32 floor wherever the chains and to_basis run on tensor cores, and 1.0x where every layer is on SIMT
(C = 20 / 40).  tc3x recovers fp32-grade products from hi + lo, so the excess is the wgmma fp32 accumulation, whose
rounding NVIDIA does not document; it also does not average out (a mass-weighted mean of the vertex outputs keeps it
while the CPU's fp32 noise cancels), which points to a biased (truncating) accumulation.  FLOOR_C['tc3x'] = 32 is the
measured worst (15.3x) with 2x headroom.  Mapped outputs (faces, global_mean) are held to the bound of the vertex
outputs they average.

``tests/test_oracle_engines.py`` shows on the CPU that the structural errors a kernel could make exceed these bounds."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle as O  # noqa: E402  (checker only)
import dn_oracle_engines as E  # noqa: E402  (checker only)

pytestmark = pytest.mark.gpu

ENGINES = list(E.EMU_ENGINES)
FLOOR_C = {"simt": 4.0, "tc3x": 32.0, "tc1x": 4.0, "bf16": 4.0}
FLIP_FLOOR = {"simt": 0.0, "tc3x": 0.0, "tc1x": 2.0 ** -11, "bf16": 2.0 ** -8}

# name: (n, m, K, C, block kwargs, mlp_hidden_dims, operators).  V = n * m; operators: None (torus order), "permuted"
# (a random vertex relabelling) or "long_rows" (four rows of ~300 extra entries).  The branch of block_fwd_impl /
# run_chain / to_basis_partials each reaches on the tensor-core engines is in its name.
CASES = {
    "c128_front_from_basis_p_q_fused": (20, 25, 128, 128, {}, None, False),
    "c128_front_fused_v7000": (70, 100, 128, 128, {}, None, False),
    "c128_norot_two_layer_front": (20, 25, 128, 128, {"with_gradient_rotations": False}, None, False),
    "c64_pq_one_layer_w2_split": (23, 31, 128, 64, {}, None, False),
    "c256_p_q_split_two_slice_to_basis": (30, 41, 128, 256, {}, None, False),
    "c256_norot": (30, 41, 128, 256, {"with_gradient_rotations": False}, None, False),
    "c16_narrow": (20, 25, 64, 16, {}, None, False),
    "c32_narrow": (20, 25, 64, 32, {}, None, False),
    "c48_narrow": (20, 25, 64, 48, {}, None, False),
    "c96_narrow": (20, 25, 64, 96, {}, None, False),
    "c20_dense_on_simt": (20, 25, 64, 20, {}, None, False),
    "c40_mlp_and_from_basis_on_simt": (20, 25, 64, 40, {}, None, False),
    "nograd_two_sources": (20, 25, 128, 128, {"with_gradient_features": False}, None, False),
    "k8_bf16_from_basis_tf32": (20, 25, 8, 64, {}, None, False),
    "k40_bf16_front_tf32": (20, 25, 40, 128, {}, None, False),
    "k12_from_basis_on_simt": (20, 25, 12, 48, {}, None, False),
    "k160_to_basis_on_simt": (20, 25, 160, 96, {}, None, False),
    "k256_to_basis_on_simt": (20, 25, 256, 128, {}, None, False),
    "mlp_64_32": (20, 25, 128, 128, {}, [64, 32], False),
    "mlp_hidden_256_layer_by_layer": (20, 25, 128, 128, {}, [256], False),
    "mlp_eight_layers": (20, 25, 64, 64, {}, [64] * 7, False),
    "v50_one_partial_tile": (5, 10, 40, 64, {}, None, False),
    "v128_one_full_tile": (8, 16, 64, 128, {}, None, False),
    "v129_one_row_past_a_tile": (3, 43, 64, 128, {}, None, False),
    "mlp_nine_layers_layer_by_layer": (20, 25, 64, 64, {}, [64] * 8, None),
    "mlp_twelve_layers_layer_by_layer": (20, 25, 64, 64, {}, [64] * 11, None),
    "c1_scalar_gather": (20, 25, 64, 1, {}, None, None),
    "c3_scalar_gather": (20, 25, 64, 3, {}, None, None),
    "c6_scalar_gather": (20, 25, 64, 6, {}, None, None),
    "c30_scalar_gather": (20, 25, 64, 30, {}, None, None),
    "permuted_vertex_order_patched_gather": (40, 50, 128, 128, {}, None, "permuted"),
    "long_rows_past_staged_entries": (60, 83, 128, 128, {}, None, "long_rows"),
}
# True: every dense layer and to_basis stays on tensor cores under tc3x; False: some stage leaves them (refused under
# DN_STRICT_TC=1).  test_oracle_engines.py checks that the oracle's dispatch agrees.
ROUTES = {name: not any(k in name for k in ("simt", "c20", "c40", "k12", "k160", "k256", "scalar")) for name in CASES}


@pytest.fixture(scope="module")
def dn():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import diffusion_net_b200 as d
    d._lib.load()
    yield d
    d.set_engine("tc3x")


def _csr(g, V):
    g = g.coalesce().cpu()
    return O.coo_to_csr(g.indices()[0].numpy(), g.indices()[1].numpy(), g.values().numpy().astype(np.float64), (V, V))


def case_operators(dn, n, m, K, seed, variant=None, device="cuda"):
    """(mass, evals, evecs, gradX, gradY) of a case (see CASES)."""
    mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=seed, device=device,
                                                                      permute=variant == "permuted")
    if variant == "long_rows":
        # rows 64..66 (one 64-row block of spmm_features_blk_kernel) and 3001 carry ~300 entries more each: the block
        # stages GB_NNZ = 1024 entries and reads the rest from global memory
        V = n * m
        rows, cols = (torch.from_numpy(a) for a in dn.synthetic.torus_pattern(n, m))
        g = torch.Generator().manual_seed(16 + seed)
        er = torch.tensor([64, 65, 66, 3001]).repeat_interleave(300)
        r, c = torch.cat((rows, er)), torch.cat((cols, torch.randint(0, V, (er.shape[0],), generator=g)))
        coo = lambda: torch.sparse_coo_tensor(torch.stack((r, c)), torch.randn(r.shape[0], generator=g) * 0.12 * V ** 0.5,
                                              (V, V)).coalesce().to(device)
        gX, gY = coo(), coo()
    return mass, evals, evecs, gX, gY


def _operators(dn, n, m, K, seed, variant=None):
    dev = case_operators(dn, n, m, K, seed, variant)
    mass, evals, evecs, gX, gY = dev
    V = n * m
    return dev, (mass.cpu().numpy(), evals.cpu().numpy(), evecs.cpu().numpy(), _csr(gX, V), _csr(gY, V))


def _emulate(fn, host_ops, *args, engine, **kw):
    """(fp64 gold, fp32 evaluation) of ``fn`` (dn_oracle_engines.block_forward / net_forward) on ``engine``."""
    mass, evals, evecs, gX, gY = host_ops
    gold = fn(args[0], mass, evals, evecs, gX, gY, *args[1:], engine=engine, **kw)
    f32 = fn(args[0], mass, evals, evecs, gX.astype(np.float32), gY.astype(np.float32), *args[1:], engine=engine,
             dtype=np.float32, **kw)
    return gold, f32


def forward_bound(engine, gold, f32):
    """FLOOR_C x max(fp32 floor, FLIP_FLOOR), relative to max|gold| (gold, f32: branch or head outputs)."""
    den = np.abs(gold).max()
    floor = np.abs(f32 - gold).max() / den
    return FLOOR_C[engine] * max(floor, FLIP_FLOOR[engine]), floor


def _check(label, engine, ours, gold, f32, base=None, mapped=None):
    """branch error against forward_bound.  ``mapped``: a linear map of the vertex outputs (faces, global_mean) whose
    error is held to the vertex outputs' bound."""
    ours = ours.detach().cpu().double().numpy() if torch.is_tensor(ours) else ours
    if base is not None:
        ours, gold, f32 = ours - base, gold - base, f32 - base
    bound, floor = forward_bound(engine, gold, f32)
    den = np.abs(gold).max()
    if mapped is not None:
        gold = mapped(gold)
    err = np.abs(ours - gold).max() / den
    print("[measured] {} err={:.3e} fp32-floor={:.3e} bound={:.3e} ratio={:.3f}".format(label, err, floor, bound,
                                                                                         err / bound))
    assert err <= bound, "{}: {:.3e} > {:.3e}".format(label, err, bound)
    return err, bound


def _block(dn, spec, seed=0):
    n, m, K, C, kw, hid, variant = spec
    dev_ops, host_ops = _operators(dn, n, m, K, seed, variant)
    params = dn.synthetic.block_weights(C, seed=seed, mlp_hidden_dims=hid,
                                        with_gradient_features=kw.get("with_gradient_features", True),
                                        with_gradient_rotations=kw.get("with_gradient_rotations", True))
    blk = dn.DiffusionNetBlock(C_width=C, mlp_hidden_dims=hid if hid is not None else [C, C], dropout=False, **kw)
    blk.load_state_dict(params, strict=True)
    blk = blk.cuda().eval()
    x = torch.randn(n * m, C, generator=torch.Generator().manual_seed(seed))
    mass, evals, evecs, gX, gY = dev_ops
    xc = x.cuda()

    def run():
        with torch.no_grad():
            y = blk(xc.unsqueeze(0), mass.unsqueeze(0), None, evals.unsqueeze(0), evecs.unsqueeze(0), [gX], [gY])
        torch.cuda.synchronize()
        return y[0]

    run.ops = (gX, gY)
    p_np = {k: v.numpy() for k, v in params.items()}
    return run, x.numpy(), host_ops, p_np, kw.get("with_gradient_features", True)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", list(CASES))
def test_block_forward_vs_emulated_fp64(dn, engine, name):
    dn.set_engine(engine)
    run, x, host_ops, params, wgf = _block(dn, CASES[name])
    y = run()
    if CASES[name][6] == "permuted":
        # dn_patches are built on the second use of an operator pair (ops._maybe_patch) and then run the staged gather
        y = run()
        assert dn.ops.prepare_operators(*run.ops)._patches, "the permuted mesh did not get patches"
    gold, f32 = _emulate(E.block_forward, host_ops, x, params, engine=engine, with_gradient_features=wgf)
    _check("{}/{}".format(name, engine), engine, y, gold, f32, base=x.astype(np.float64))


@pytest.mark.parametrize("engine", ["tc3x", "bf16"])
def test_block_forward_200k(dn, engine):
    """V = 200k (the benchmark's mesh size), C = K = 128: ~1560 row tiles per chain, 132 split-V to_basis partials.
    tc3x and bf16 only (the two engines the benchmark runs); tc1x shares every kernel with tc3x."""
    dn.set_engine(engine)
    run, x, host_ops, params, wgf = _block(dn, (400, 500, 128, 128, {}, None, None))
    gold, f32 = _emulate(E.block_forward, host_ops, x, params, engine=engine)
    _check("v200k/{}".format(engine), engine, run(), gold, f32, base=x.astype(np.float64))


@pytest.mark.parametrize("engine", ["tc3x", "tc1x", "bf16"])
@pytest.mark.parametrize("C", [128, 256])
def test_two_calls_bitwise_equal(dn, engine, C):
    dn.set_engine(engine)
    run, *_ = _block(dn, (30, 41, 128, C, {}, None, None), seed=3)
    assert torch.equal(run(), run())


# ---- the fused head (dn_block_fwd_ex) and the net ------------------------------------------------------------------
def _net(dn, C_out, C=128, K=128, n=20, m=25, seed=5, outputs_at="vertices"):
    dev_ops, host_ops = _operators(dn, n, m, K, seed)
    torch.manual_seed(seed)
    net = dn.DiffusionNet(C_in=16, C_out=C_out, C_width=C, N_block=2, dropout=False, outputs_at=outputs_at)
    with torch.no_grad():
        for nm, p in net.named_parameters():
            if nm.endswith("diffusion_time"):
                p.uniform_(1e-3, 0.3)
    net = net.cuda().eval()
    x = torch.randn(n * m, 16, generator=torch.Generator().manual_seed(seed))
    return net, x, dev_ops, host_ops, {k: v.detach().cpu().numpy() for k, v in net.state_dict().items()}


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("n_out", [1, 5, 8, 9])
@pytest.mark.parametrize("outputs_at", ["vertices", "faces", "global_mean"])
def test_net_head_vs_emulated_fp64(dn, engine, n_out, outputs_at):
    """n_out <= 8 rides in the last block's MiniMLP epilogue (dn_block_fwd_ex) on the tensor-core engines; n_out = 9 and
    the SIMT engine (HeadNotFused) run last_lin as its own launch.  Every ``outputs_at`` maps the same vertex output."""
    dn.set_engine(engine)
    net, x, (mass, evals, evecs, gX, gY), host_ops, params = _net(dn, n_out, outputs_at=outputs_at)
    n, m = 20, 25
    faces = dn.synthetic.torus_mesh(n, m)[1]
    with torch.no_grad():
        y = net(x.cuda(), mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY, faces=faces.cuda())
    torch.cuda.synchronize()
    gold, f32 = _emulate(E.net_forward, host_ops, x.numpy(), params, 2, engine=engine)
    m_np = host_ops[0].astype(np.float64)

    def at(v):
        if outputs_at == "faces":
            return v[faces.numpy()].mean(axis=1)
        if outputs_at == "global_mean":
            return (v * m_np[:, None]).sum(0, keepdims=True) / m_np.sum()
        return v
    _check("head{}/{}/{}".format(n_out, outputs_at, engine), engine, y.reshape(-1, n_out), gold, f32, mapped=at)


# ---- forward_batch (dn_block_fwd_batched) --------------------------------------------------------------------------
@pytest.mark.parametrize("engine", ["tc3x", "tc1x", "bf16"])
@pytest.mark.parametrize("C,K", [(64, 40), (128, 128), (256, 128)])
def test_forward_batch_ragged_vs_emulated_fp64(dn, engine, C, K):
    """A ragged batch: V = 77 (shorter than one 128-row tile; at K = 128 a mesh needs V >= K, so 143 rows there, ending in a
    15-row partial tile), 256 (an exact multiple of 128) and 1100.  Each mesh's output against the fp64 emulation of the
    net on that mesh alone."""
    dn.set_engine(engine)
    torch.manual_seed(9)
    net = dn.DiffusionNet(C_in=16, C_out=5, C_width=C, N_block=2, dropout=None)
    with torch.no_grad():
        for nm, p in net.named_parameters():
            if nm.endswith("diffusion_time"):
                p.uniform_(1e-3, 0.3)
    net = net.cuda().eval()
    params = {k: v.detach().cpu().numpy() for k, v in net.state_dict().items()}
    meshes, xs, hosts = [], [], []
    for i, (n, m) in enumerate([(7, 11) if K <= 77 else (11, 13), (16, 16), (25, 44)]):
        (mass, evals, evecs, gX, gY), host = _operators(dn, n, m, K, 40 + i)
        meshes.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY))
        xs.append(torch.randn(n * m, 16, generator=torch.Generator().manual_seed(50 + i)))
        hosts.append(host)
    with torch.no_grad():
        outs = net.forward_batch(dn.MeshBatch(meshes), [x.cuda() for x in xs])
    torch.cuda.synchronize()
    for i, (o, x, host) in enumerate(zip(outs, xs, hosts)):
        gold, f32 = _emulate(E.net_forward, host, x.numpy(), params, 2, engine=engine)
        _check("batch{}/C{}K{}/{}".format(i, C, K, engine), engine, o, gold, f32)


def test_forward_batch_simt_is_refused(dn):
    """The fused batch forward forms every mesh's spectral multiplier in the tensor-core pack launch: the exact SIMT
    engine has no batch route and refuses with a clear error (the per-mesh forward is its route)."""
    dn.set_engine("simt")
    try:
        net = dn.DiffusionNet(C_in=16, C_out=5, C_width=64, N_block=1, dropout=False).cuda().eval()
        meshes = []
        for i in range(2):
            mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(12, 14, 40, seed=i, device="cuda")
            meshes.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY))
        with torch.no_grad(), pytest.raises(RuntimeError, match="unsupported"):
            net.forward_batch(dn.MeshBatch(meshes), [torch.randn(168, 16, device="cuda") for _ in range(2)])
    finally:
        dn.set_engine("tc3x")


def test_forward_batch_k_above_128_is_refused(dn):
    """K > 128: to_basis has no batch route (its split-V kernel takes K <= 128 and mesh batches have no SIMT route), so
    the fused batch forward refuses with a clear error instead of computing something else."""
    dn.set_engine("tc3x")
    net = dn.DiffusionNet(C_in=16, C_out=5, C_width=64, N_block=1, dropout=False).cuda().eval()
    meshes = []
    for i in range(2):
        mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(12, 14, 160, seed=i, device="cuda")
        meshes.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY))
    with torch.no_grad(), pytest.raises(RuntimeError, match="unsupported"):
        net.forward_batch(dn.MeshBatch(meshes), [torch.randn(168, 16, device="cuda") for _ in range(2)])


# ---- graph replays ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("engine", ENGINES)
def test_graphed_net_replay_bitwise_equals_eager(dn, engine):
    """GraphedNet (one CUDA graph per mesh, fused head) replays give the eager forward's bits, twice."""
    dn.set_engine(engine)
    net, x, (mass, evals, evecs, gX, gY), _, _ = _net(dn, 5, C=128, K=128, n=20, m=25)
    kw = dict(x_in=x.cuda(), mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY)
    with torch.no_grad():
        eager = net(**kw).clone()
    gn = dn.graphs.GraphedNet(net)
    for _ in range(2):
        out = gn.forward_batch([kw])[0]
        torch.cuda.synchronize()
        assert torch.equal(out, eager)


@pytest.mark.parametrize("engine", ["tc3x", "tc1x", "bf16"])
def test_graphed_batch_replay_bitwise_equals_eager(dn, engine):
    """GraphedBatch (one CUDA graph over a ragged mesh batch) replays give eager forward_batch's bits, twice."""
    dn.set_engine(engine)
    torch.manual_seed(11)
    net = dn.DiffusionNet(C_in=16, C_out=5, C_width=128, N_block=2, dropout=False).cuda().eval()
    meshes, xs = [], []
    for i, (n, m) in enumerate([(11, 13), (16, 16), (25, 44)]):
        mass, evals, evecs, gX, gY = case_operators(dn, n, m, 128, 60 + i)
        meshes.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY))
        xs.append(torch.randn(n * m, 16, generator=torch.Generator().manual_seed(70 + i)).cuda())
    mb = dn.MeshBatch(meshes)
    with torch.no_grad():
        eager = [o.clone() for o in net.forward_batch(mb, xs)]
    gb = dn.graphs.GraphedBatch(net, mb)
    for _ in range(2):
        outs = gb.forward(xs)
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(outs, eager))


# ---- every case reaches the route it is named after ------------------------------------------------------------------
def _route_report():
    """Run in a DN_STRICT_TC=1 subprocess: each case's block forward under tc3x; prints one JSON line."""
    import diffusion_net_b200 as d
    d.set_engine("tc3x")
    res = {}
    for name, spec in CASES.items():
        run, *_ = _block(d, spec)
        try:
            run()
            res[name] = "ok"
        except RuntimeError as e:
            res[name] = "unsupported" if "unsupported" in str(e) else "error: " + str(e)
    print(json.dumps(res))


def test_dispatch_routes_under_strict_tc(dn):
    tests_dir = os.path.join(ROOT, "tests")
    env = dict(os.environ, DN_STRICT_TC="1")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", "import sys; sys.path[:0] = [{!r}, {!r}]; import test_gpu_forward as t; t._route_report()".format(
            tests_dir, ROOT)]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    want = {k: "ok" if v else "unsupported" for k, v in ROUTES.items()}
    assert got == want, {k: (got.get(k), want[k]) for k in want if got.get(k) != want[k]}
