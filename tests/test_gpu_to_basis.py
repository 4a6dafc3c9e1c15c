"""The split-V to_basis kernel (to_basis_kernel: 16-row chunks, 128-row accumulation chains folded into fp32 sums)
against fp64.

Routes: ``dn_to_basis`` (with and without mass, C = 256 as two 128-column slices of a wider matrix), the weight
gradient of a dense layer (``atb``: mass = null, I and J <= 128) and the grouped to_basis of a mesh batch (CTA row
ranges from ``dn_mesh_batch_plan``).  Row counts sit at the edges of the pipeline: one chunk +- 1, two chunks +- 1,
partial last chunks, a split-V CTA range boundary +- 1 (ranges are multiples of 16 rows), and V = 200k.

Bound.  Componentwise: |ours - gold| <= TOL[engine] * sum_v |Phi[v][k] m[v] x[v][c]|.  tc3x recovers fp32-grade products
(hi * hi + hi * lo + lo * hi) and accumulates in fp32 over chains of at most 128 rows, then folds; 2^-13 covers a
relative error of 2^-23 per addition over a 384-term MMA chain plus the folds and the partial reduction.  tc1x (and
bf16, which runs to_basis as single-pass TF32) rounds both operands to TF32 (2^-11 each): 2^-8."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = {"tc3x": 2.0 ** -13, "tc1x": 2.0 ** -8}


@pytest.fixture(scope="module")
def dn():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import diffusion_net_b200 as d
    d._lib.load()
    yield d
    d.set_engine("tc3x")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _inputs(V, K, C_, seed, mass=True):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(V, C_, generator=g)
    phi = torch.randn(V, K, generator=g) / max(V, 1) ** 0.5
    m = (torch.rand(V, generator=g) + 0.5) / max(V, 1) if mass else None
    return x, phi, m


def _gold(x, phi, m):
    xd, pd = x.double().numpy(), phi.double().numpy()
    if m is not None:
        xd = xd * m.double().numpy()[:, None]
    return pd.T @ xd, np.abs(pd).T @ np.abs(xd)


def _check(label, engine, ours, gold, absum):
    ours = ours.detach().cpu().double().numpy()
    err = np.abs(ours - gold)
    bound = TOL[engine] * absum + 1e-30
    worst = (err / bound).max()
    print("[measured] {} max err/bound={:.3e} max err={:.3e}".format(label, worst, err.max()))
    assert worst <= 1.0, "{}: err/bound {:.3e}".format(label, worst)


def _to_basis(dn, x, phi, m):
    return dn.ops.to_basis_raw(x.cuda(), phi.cuda(), m.cuda() if m is not None else None)


def _v_edges():
    s = _sms()
    # chunk edges, then a uniform split where every CTA reduces 3 x 16 rows, +- 1
    return [1, 15, 16, 17, 31, 32, 33, 63, 65, 48 * s - 1, 48 * s, 48 * s + 1]


@pytest.mark.parametrize("engine", ["tc3x", "tc1x"])
@pytest.mark.parametrize("vi", range(12))
def test_to_basis_row_edges(dn, engine, vi):
    V = _v_edges()[vi]
    dn.set_engine(engine)
    x, phi, m = _inputs(V, 128, 128, seed=vi)
    gold, absum = _gold(x, phi, m)
    _check("V{}/{}".format(V, engine), engine, _to_basis(dn, x, phi, m), gold, absum)


@pytest.mark.parametrize("engine", ["tc3x", "tc1x"])
@pytest.mark.parametrize("K", [4, 12, 100, 128])
@pytest.mark.parametrize("C_", [16, 48, 128, 256])
@pytest.mark.parametrize("mass", [True, False])
def test_to_basis_shapes(dn, engine, K, C_, mass):
    """C % 32 == 16 and narrow C (m64n16 MMAs), K below one eigen-row block and K % 32 in {4, 12, 0}; C = 256 runs as
    two 128-column slices of the wider matrix, one bulk copy per row."""
    dn.set_engine(engine)
    V = 3 * 1000 + 17
    x, phi, m = _inputs(V, K, C_, seed=K * 1000 + C_, mass=mass)
    gold, absum = _gold(x, phi, m)
    _check("K{}C{}mass{}/{}".format(K, C_, int(mass), engine), engine, _to_basis(dn, x, phi, m), gold, absum)


@pytest.mark.parametrize("engine", ["tc3x", "tc1x"])
@pytest.mark.parametrize("C_", [128, 256])
def test_to_basis_200k(dn, engine, C_):
    dn.set_engine(engine)
    x, phi, m = _inputs(200_000, 128, C_, seed=7)
    gold, absum = _gold(x, phi, m)
    _check("V200k/C{}/{}".format(C_, engine), engine, _to_basis(dn, x, phi, m), gold, absum)


@pytest.mark.parametrize("engine", ["tc3x", "tc1x"])
@pytest.mark.parametrize("V,C_", [(33, 128), (6337, 48), (200_000, 128), (200_000, 256)])
def test_to_basis_two_calls_bitwise_equal(dn, engine, V, C_):
    dn.set_engine(engine)
    x, phi, m = _inputs(V, 128, C_, seed=11)
    a, b = _to_basis(dn, x, phi, m), _to_basis(dn, x, phi, m)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


@pytest.mark.parametrize("engine", ["tc3x", "tc1x"])
@pytest.mark.parametrize("V,I,J", [(17, 128, 128), (5000, 128, 128), (200_000, 128, 128), (4097, 48, 100)])
def test_atb_weight_gradient(dn, engine, V, I, J):
    """A dense layer's weight gradient dW = g^T x (out = x W^T + b) runs on to_basis with no mass: I = out width
    (the eigen-row side), J = in width (the channel side).  Called twice: the bits must repeat."""
    dn.set_engine(engine)
    g = torch.Generator().manual_seed(V + I + J)
    x = torch.randn(V, J, generator=g)
    gout = torch.randn(V, I, generator=g) / V ** 0.5
    w = (torch.randn(I, J, generator=g) / J ** 0.5).cuda()
    b = torch.zeros(I).cuda()
    grads = []
    for _ in range(2):
        wr = w.clone().requires_grad_(True)
        y = dn.ops.mlp_apply([x.cuda()], [wr], [b])
        y.backward(gout.cuda())
        torch.cuda.synchronize()
        grads.append(wr.grad)
    gold = gout.double().numpy().T @ x.double().numpy()
    absum = np.abs(gout.double().numpy()).T @ np.abs(x.double().numpy())
    _check("atb V{} I{} J{}/{}".format(V, I, J, engine), engine, grads[0], gold, absum)
    assert torch.equal(grads[0], grads[1])


@pytest.mark.parametrize("engine", ["tc3x", "tc1x"])
@pytest.mark.parametrize("C_", [48, 128, 256])
def test_mesh_batch_to_basis(dn, engine, C_):
    """The grouped to_basis of a mesh batch (x_spec of dn_learned_time_diffusion_fwd_batched): CTA row ranges planned
    per mesh, none crossing a mesh boundary.  Each mesh's Phi_b^T M_b x_b against fp64, and a second call's bits."""
    dn.set_engine(engine)
    K = 128
    meshes, hosts = [], []
    for i, (n, mm) in enumerate([(11, 13), (16, 16), (25, 44), (70, 100)]):
        mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, mm, K, seed=80 + i, device="cuda")
        meshes.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY))
    mb = dn.MeshBatch(meshes)
    lib = dn._lib.load()
    x = torch.randn(mb.V, C_, generator=torch.Generator().manual_seed(C_)).cuda()
    for b in range(mb.n_meshes):   # padding rows stay zero
        x[mb.row_begin[b] + mb.n_rows[b]:mb.row_begin[b + 1]] = 0
    specs = []
    for _ in range(2):
        time = torch.full((C_,), 0.05, device="cuda")
        xd = torch.empty_like(x)
        spec = torch.empty(mb.n_meshes, K, C_, device="cuda")
        ws = dn.ops.workspace(mb.V, K, C_, x.device, extra=dn.ops.batched_diffusion_workspace_extra(mb.n_meshes, K, C_))
        dn._lib.check(lib.dn_learned_time_diffusion_fwd_batched(
            x.data_ptr(), mb.mass.data_ptr(), mb.evals.data_ptr(), mb.evecs.data_ptr(), time.data_ptr(),
            C.byref(mb.desc), mb.V, K, C_, xd.data_ptr(), spec.data_ptr(), ws.data_ptr(), ws.numel(),
            dn.ops._engine, dn.ops._stream()), "dn_learned_time_diffusion_fwd_batched")
        torch.cuda.synchronize()
        specs.append(spec)
    assert torch.equal(specs[0], specs[1])
    for b in range(mb.n_meshes):
        r0, n = mb.row_begin[b], mb.n_rows[b]
        gold, absum = _gold(x[r0:r0 + n].cpu(), meshes[b]["evecs"].cpu(), meshes[b]["mass"].cpu())
        _check("batch mesh{}/C{}/{}".format(b, C_, engine), engine, specs[0][b], gold, absum)
