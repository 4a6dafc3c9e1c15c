"""Repeat calls of the fused block forward give the same bits when every CTA runs many row tiles.

At V = 200k a chain launch has ~1560 tiles over the SMs, so both rings of rows_chain_kernel (layer 0's activations and
the weight stages) wrap many times and a producer runs ahead into a CTA's next tile while its consumers are still in
the current one.  Slot hand-back races show up here as differing bits; a bf16 mesh-batch forward is the case that once
exposed one.  (tests/test_gpu_forward.py repeats a V = 1230 block, 10 tiles: fewer than the SMs.)"""
import pytest
import torch

from test_gpu_forward import _block, case_operators

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dn():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import diffusion_net_b200 as d
    d._lib.load()
    yield d
    d.set_engine("tc3x")


@pytest.mark.parametrize("engine", ["tc3x", "bf16"])
def test_two_calls_bitwise_equal_200k(dn, engine):
    dn.set_engine(engine)
    run, *_ = _block(dn, (400, 500, 128, 128, {}, None, None), seed=3)
    assert torch.equal(run(), run())


@pytest.mark.parametrize("engine", ["tc3x", "bf16"])
def test_mesh_batch_two_calls_bitwise_equal(dn, engine):
    """A batch of 12 meshes, ~105k rows in all: ~830 tiles per chain, several per CTA."""
    dn.set_engine(engine)
    torch.manual_seed(13)
    net = dn.DiffusionNet(C_in=16, C_out=5, C_width=128, N_block=2, dropout=False).cuda().eval()
    meshes, xs = [], []
    for i, (n, m) in enumerate([(11, 13), (16, 16), (25, 44), (60, 70), (70, 100), (200, 200)] * 2):
        mass, evals, evecs, gX, gY = case_operators(dn, n, m, 128, 90 + i)
        meshes.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY))
        xs.append(torch.randn(n * m, 16, generator=torch.Generator().manual_seed(100 + i)).cuda())
    mb = dn.MeshBatch(meshes)
    outs = []
    for _ in range(2):
        with torch.no_grad():
            outs.append([o.clone() for o in net.forward_batch(mb, xs)])
        torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(*outs))
