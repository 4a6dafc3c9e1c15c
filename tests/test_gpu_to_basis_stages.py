"""The split-V to_basis kernel at the edges of its 32-row stages (4 k8 slices per stage, TMA boxes of 8 columns x 32
rows) against fp64, with the bound of test_gpu_to_basis.py.

Row counts: one stage +- 1, two stages +- 1, a partial last stage of every length class (1, 8, 9, 24 and 31 rows past
the last full stage), and uniform CTA ranges of 16 (one half stage) and 48 rows (one and a half stages), so that a
CTA's last stage reaches into the next CTA's rows, which it must read as zeros.  The mesh batch has meshes whose
ranges end mid-stage, with padding rows filled with large values: the consumer zeroes rows past a range's end (TMA
only zero-fills past V), so none of them may reach a mesh's sum."""
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


def _stage_edges():
    s = _sms()
    # V <= 16 * sms gives one 16-row CTA range each (half a stage); 48-row ranges end mid-stage
    return [31, 32, 33, 63, 64, 65, 96 + 1, 96 + 8, 96 + 9, 96 + 24, 96 + 31,
            16 * s - 7, 48 * s - 7, 48 * s + 9, 80 * s + 24]


@pytest.mark.parametrize("engine", ["tc3x", "tc1x"])
@pytest.mark.parametrize("vi", range(15))
def test_to_basis_stage_edges(dn, engine, vi):
    V = _stage_edges()[vi]
    dn.set_engine(engine)
    x, phi, m = _inputs(V, 128, 128, seed=100 + vi)
    gold, absum = _gold(x, phi, m)
    ours = dn.ops.to_basis_raw(x.cuda(), phi.cuda(), m.cuda())
    _check("V{}/{}".format(V, engine), engine, ours, gold, absum)


@pytest.mark.parametrize("engine", ["tc3x", "tc1x"])
@pytest.mark.parametrize("K,C_", [(12, 48), (100, 16), (128, 112)])
def test_to_basis_stage_edges_narrow(dn, engine, K, C_):
    """Fewer Phi and x boxes than 16 per stage (K < 128: zero-filled columns; C < 128: m64n16 MMAs) with a partial
    last stage and mid-stage CTA ends."""
    dn.set_engine(engine)
    for V in (9, 48 * _sms() + 9):
        x, phi, m = _inputs(V, K, C_, seed=K + C_ + V)
        gold, absum = _gold(x, phi, m)
        ours = dn.ops.to_basis_raw(x.cuda(), phi.cuda(), m.cuda())
        _check("V{}K{}C{}/{}".format(V, K, C_, engine), engine, ours, gold, absum)


@pytest.mark.parametrize("engine", ["tc3x", "tc1x"])
@pytest.mark.parametrize("C_", [48, 128])
def test_mesh_batch_to_basis_mid_stage(dn, engine, C_):
    """Meshes of 133, 143, 299, 1000 and 5002 rows: CTA ranges end at mesh ends that are not stage multiples, and inside
    the larger meshes at 16-row multiples that are not 32-row multiples.  Padding rows hold 1e6: a row past a range's
    end that reached the MMAs would be far outside the bound."""
    dn.set_engine(engine)
    K = 128
    meshes = []
    for i, (n, mm) in enumerate([(7, 19), (11, 13), (13, 23), (25, 40), (41, 122)]):
        mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, mm, K, seed=90 + i, device="cuda")
        meshes.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY))
    mb = dn.MeshBatch(meshes)
    lib = dn._lib.load()
    x = torch.randn(mb.V, C_, generator=torch.Generator().manual_seed(C_ + 1)).cuda()
    for b in range(mb.n_meshes):
        x[mb.row_begin[b] + mb.n_rows[b]:mb.row_begin[b + 1]] = 1e6
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
