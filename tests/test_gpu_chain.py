"""The fused row chain (rows_chain_kernel) where its first layer's staging decides the result: layer 0's activations
reach shared memory through 2-D TMA copies of 8-column x 128-row boxes, one tensor map per source, and the front of a
C = 128 block runs from_basis, P and Q as one chain (Q reads x_diffuse again as P's sibling).

Every chain is called directly through dn_mini_mlp_fwd / dn_from_basis (or the block) and checked against fp64 under
the suite's bounds: tc3x 1e-5, tc1x 16 u_tf32 (test_gpu_backward.py), bf16 2e-2 (test_gpu_parity.py)."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle as O  # noqa: E402  (checker only)

pytestmark = pytest.mark.gpu

TOL = {"tc3x": 1e-5, "tc1x": 16 * 2.0 ** -11, "bf16": 2e-2}
ENGINES = list(TOL)


@pytest.fixture(scope="module")
def dn():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import diffusion_net_b200 as d
    d._lib.load()
    yield d
    d.set_engine("tc3x")


def _rand(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g) * scale


def _mlp(dn, engine, src_ptrs, widths, Ws, bs, residual, V):
    """dn_mini_mlp_fwd over raw source pointers (so a test can hand it an offset pointer)."""
    lib = dn._lib.load()
    dims = [sum(widths)] + [w.shape[0] for w in Ws]
    out = torch.empty(V, dims[-1], device="cuda")
    ws = dn.ops.workspace(V, max(dims), max(dims), torch.device("cuda", torch.cuda.current_device()))
    dn._lib.check(lib.dn_mini_mlp_fwd(
        dn._lib.ptr_array(src_ptrs), dn._lib.int_array(widths), len(widths), dn._lib.ptr_array([w.data_ptr() for w in Ws]),
        dn._lib.ptr_array([b.data_ptr() for b in bs]), dn._lib.int_array(dims), len(Ws), None,
        residual.data_ptr() if residual is not None else None, V, None, out.data_ptr(), ws.data_ptr(), ws.numel(),
        dn.ops._ENGINES[engine], dn.ops._stream()), "dn_mini_mlp_fwd")
    torch.cuda.synchronize()
    return out


def _mlp_case(dn, engine, V, widths, hidden, seed=0, residual=True):
    g = torch.Generator().manual_seed(seed)
    K0 = sum(widths)
    dims = [K0] + hidden
    srcs = [_rand(g, V, w) for w in widths]
    Ws = [_rand(g, dims[i + 1], dims[i], scale=dims[i] ** -0.5) for i in range(len(hidden))]
    bs = [_rand(g, dims[i + 1], scale=0.1) for i in range(len(hidden))]
    res = _rand(g, V, dims[-1]) if residual else None
    cu = [s.cuda() for s in srcs]
    out = _mlp(dn, engine, [s.data_ptr() for s in cu], widths, [w.cuda() for w in Ws], [b.cuda() for b in bs],
               res.cuda() if res is not None else None, V)
    f = np.float64
    gold = O.mini_mlp(np.concatenate([s.numpy() for s in srcs], 1).astype(f), [w.numpy().astype(f) for w in Ws],
                      [b.numpy().astype(f) for b in bs])
    if res is not None:
        gold = gold + res.numpy().astype(f)
    return out, gold


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("V", [77, 1000])
def test_last_tile_rows_are_zero_filled(dn, engine, V):
    """V < 128 (one partial tile) and V % 128 = 104: the TMA box of the last tile reaches past row V-1 and the copy
    fills those rows with zeros (CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE); only rows < V are stored.  384 -> 128 -> 128 with
    residual is the MiniMLP shape (full-width MMAs)."""
    out, gold = _mlp_case(dn, engine, V, [128, 128, 128], [128, 128])
    assert O.rel_err(out.cpu().numpy(), gold) < TOL[engine]


@pytest.mark.parametrize("engine", ENGINES)
def test_stage_across_two_sources(dn, engine):
    """Widths 24 + 40 (8 mod 16): K stage 1 (columns 16..31) is two boxes, columns 16..23 from source 0's tensor map
    and 24..31 from source 1's -- the source lookup of the producer lane, per 8-column box."""
    out, gold = _mlp_case(dn, engine, 515, [24, 40], [48, 32], seed=1)
    assert O.rel_err(out.cpu().numpy(), gold) < TOL[engine]


@pytest.mark.parametrize("engine", ENGINES)
def test_three_sources_and_half_stage(dn, engine):
    """Three sources of widths 8, 16, 16 (K = 40): every stage straddles two sources, and the last stage is half a
    stage (one box, expect_tx of 4 KiB, second k8 slice skipped)."""
    out, gold = _mlp_case(dn, engine, 300, [8, 16, 16], [32, 16], seed=2)
    assert O.rel_err(out.cpu().numpy(), gold) < TOL[engine]


@pytest.mark.parametrize("engine", ENGINES)
def test_single_256_wide_layer(dn, engine):
    """One 128 -> 256 layer without bias (the [P|Q] shape: NMAX = 256, full-width MMAs) fed from the ring."""
    out, gold = _mlp_case(dn, engine, 700, [128], [256], seed=3, residual=False)
    assert O.rel_err(out.cpu().numpy(), gold) < TOL[engine]


@pytest.mark.parametrize("engine", ENGINES)
def test_from_basis_half_stage(dn, engine):
    """dn_from_basis with K = 56 (K % 16 = 8: the last stage is one box) and V % 128 != 0."""
    g = torch.Generator().manual_seed(4)
    V, K, C = 333, 56, 64
    basis, values = _rand(g, V, K), _rand(g, K, C, scale=0.2)
    dn.set_engine(engine)
    out = dn.ops.from_basis_raw(values.cuda(), basis.cuda())
    assert O.rel_err(out.cpu().numpy(), O.from_basis(values.double().numpy(), basis.double().numpy())) < TOL[engine]


def test_source_not_16_byte_aligned_takes_simt(dn, capfd):
    """A source 8 bytes past a 16-byte boundary cannot be a TMA tensor map: the chain refuses it and the layer runs on
    the exact fp32 SIMT kernel, which says so once on stderr (and DN_STRICT_TC=1 turns it into an error)."""
    g = torch.Generator().manual_seed(5)
    V, W = 200, 72
    buf = torch.zeros(V * W + 2, device="cuda")
    src = buf[2:].view(V, W)
    assert src.data_ptr() % 16 == 8
    src.copy_(_rand(g, V, W).cuda())
    Wt, b = _rand(g, 48, W, scale=W ** -0.5), _rand(g, 48, scale=0.1)
    strict = os.environ.get("DN_STRICT_TC", "0") not in ("", "0")
    if strict:
        with pytest.raises(RuntimeError, match="unsupported"):
            _mlp(dn, "tc3x", [src.data_ptr()], [W], [Wt.cuda()], [b.cuda()], None, V)
        return
    out = _mlp(dn, "tc3x", [src.data_ptr()], [W], [Wt.cuda()], [b.cuda()], None, V)
    gold = O.mini_mlp(src.cpu().double().numpy(), [Wt.double().numpy()], [b.double().numpy()])
    assert O.rel_err(out.cpu().numpy(), gold) < 3e-6          # the exact SIMT engine's bound
    assert "K=72, N=48 is outside the tensor-core kernels' envelope" in capfd.readouterr().err


def test_two_calls_bitwise_equal(dn):
    """The ring's slot / phase bookkeeping carries across tiles and layers: two calls give the same bits."""
    a, _ = _mlp_case(dn, "tc3x", 2000, [128, 128, 128], [128, 128], seed=6)
    b, _ = _mlp_case(dn, "tc3x", 2000, [128, 128, 128], [128, 128], seed=6)
    assert torch.equal(a, b)


def _block_case(dn, n, m, K, C, seed):
    mass, L, evals, evecs, gradX, gradY = dn.synthetic.structural_operators(n, m, K, seed=seed, device="cuda")
    params = dn.synthetic.block_weights(C, seed=seed)
    x = torch.randn(n * m, C, generator=torch.Generator().manual_seed(seed)).cuda()
    blk = dn.DiffusionNetBlock(C_width=C, mlp_hidden_dims=[C, C], dropout=False)
    blk.load_state_dict(params, strict=True)
    blk = blk.cuda().eval()

    def run():
        with torch.no_grad():
            y = blk(x.unsqueeze(0), mass.unsqueeze(0), None, evals.unsqueeze(0), evecs.unsqueeze(0), [gradX], [gradY])
        torch.cuda.synchronize()
        return y[0]

    V, f = n * m, np.float64
    gxc, gyc = gradX.coalesce().cpu(), gradY.coalesce().cpu()
    gX = O.coo_to_csr(gxc.indices()[0].numpy(), gxc.indices()[1].numpy(), gxc.values().numpy().astype(f), (V, V))
    gY = O.coo_to_csr(gyc.indices()[0].numpy(), gyc.indices()[1].numpy(), gyc.values().numpy().astype(f), (V, V))
    gold = O.diffusion_net_block(x.cpu().numpy().astype(f), mass.cpu().numpy().astype(f), evals.cpu().numpy().astype(f),
                                 evecs.cpu().numpy().astype(f), gX, gY, {k: v.numpy().astype(f) for k, v in params.items()})
    return run, gold


@pytest.mark.parametrize("engine", ENGINES)
def test_block_c128_front_chain(dn, engine):
    """C = 128 with rotations: from_basis, P and Q run as one chain (Q from the registers P read, P's epilogue keeps
    them); V = 500 ends in a partial tile.  Against the fp64 block, and two calls bitwise equal (each layer-0 ring
    slot is handed back only after its reads, behind a proxy fence)."""
    dn.set_engine(engine)
    run, gold = _block_case(dn, 20, 25, 128, 128, seed=8)
    y0 = run()
    assert O.rel_err(y0.cpu().numpy(), gold) < TOL[engine]
    assert torch.equal(run(), y0)


def test_mesh_batch_forward(dn):
    """A mesh batch: layer 0 of the front chain picks each tile's spectral multiplier (tile_group) while its
    activations come through the ring; the batched forward equals the per-mesh forward to the tc3x bound."""
    dn.set_engine("tc3x")
    K, C = 64, 64
    meshes, xs = [], []
    for i, (n, m) in enumerate([(12, 11), (9, 10), (20, 7)]):
        mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=20 + i, device="cuda")
        meshes.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY))
        xs.append(torch.randn(n * m, 16, generator=torch.Generator().manual_seed(30 + i)).cuda())
    torch.manual_seed(0)
    net = dn.DiffusionNet(C_in=16, C_out=5, C_width=C, N_block=2, dropout=False).cuda().eval()
    mb = dn.MeshBatch(meshes)
    with torch.no_grad():
        outs = net.forward_batch(mb, xs)
        for it, x, o in zip(meshes, xs, outs):
            ref = net(x, it["mass"], evals=it["evals"], evecs=it["evecs"], gradX=it["gradX"], gradY=it["gradY"])
            assert O.rel_err(o.cpu().numpy(), ref.cpu().numpy()) < 3e-5
