"""The fused inference block forward writes each mesh's result straight into its slice of one (B, V, n) tensor.

Against the per-mesh ``block_forward_raw`` calls (which allocate their own result), bitwise, for the block output and
for a fused linear head; the result is a fresh tensor (no storage shared with the input), and ``out=`` of the wrong
shape or dtype is refused."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dn():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import diffusion_net_b200 as d
    d._lib.load()
    yield d
    d.set_engine("tc3x")


def _setup(dn, B, C=64, K=64, n=24, m=32):
    ops_list = [dn.synthetic.structural_operators(n, m, K, seed=s, device="cuda") for s in range(B)]
    mass = torch.stack([o[0] for o in ops_list])
    evals = torch.stack([o[2] for o in ops_list])
    evecs = torch.stack([o[3] for o in ops_list])
    gX = [o[4] for o in ops_list]
    gY = [o[5] for o in ops_list]
    blk = dn.DiffusionNetBlock(C_width=C, mlp_hidden_dims=[C, C], dropout=False)
    blk.load_state_dict(dn.synthetic.block_weights(C, seed=3), strict=True)
    blk = blk.cuda().eval()
    x = torch.randn(B, n * m, C, generator=torch.Generator().manual_seed(5)).cuda()
    return blk, x, mass, evals, evecs, gX, gY


def _per_mesh(dn, blk, x, mass, evals, evecs, gX, gY, head=None):
    A_re, A_im = blk.gradient_features.weights()
    lins = blk.mlp.linears()
    outs = []
    for b in range(x.shape[0]):
        g = dn.ops.prepare_operators(gX[b], gY[b])
        outs.append(dn.ops.block_forward_raw(x[b], mass[b], evals[b], evecs[b], g, blk.diffusion.diffusion_time, A_re,
                                             A_im, [l.weight for l in lins], [l.bias for l in lins], True, head=head))
    return torch.stack(outs, 0)


@pytest.mark.parametrize("engine", ["tc3x", "tc1x", "bf16", "simt"])
@pytest.mark.parametrize("B", [1, 3])
def test_fused_block_writes_slices(dn, engine, B):
    dn.set_engine(engine)
    blk, x, mass, evals, evecs, gX, gY = _setup(dn, B)
    with torch.no_grad():
        y = blk(x, mass, None, evals, evecs, gX, gY)
        ref = _per_mesh(dn, blk, x, mass, evals, evecs, gX, gY)
    torch.cuda.synchronize()
    assert y.shape == x.shape and y.dtype == torch.float32 and y.is_contiguous()
    assert y.untyped_storage().data_ptr() != x.untyped_storage().data_ptr()
    assert torch.equal(y, ref)


@pytest.mark.parametrize("B", [1, 2])
def test_fused_head_writes_slices(dn, B):
    dn.set_engine("tc3x")
    blk, x, mass, evals, evecs, gX, gY = _setup(dn, B)
    g = torch.Generator().manual_seed(9)
    head = ((torch.randn(5, 64, generator=g) / 8).cuda(), torch.randn(5, generator=g).cuda())
    with torch.no_grad():
        y = blk(x, mass, None, evals, evecs, gX, gY, head=head)
        ref = _per_mesh(dn, blk, x, mass, evals, evecs, gX, gY, head=head)
    torch.cuda.synchronize()
    assert y.shape == (B, x.shape[1], 5)
    assert torch.equal(y, ref)


def test_out_argument_checked(dn):
    dn.set_engine("tc3x")
    blk, x, mass, evals, evecs, gX, gY = _setup(dn, 1)
    A_re, A_im = blk.gradient_features.weights()
    lins = blk.mlp.linears()
    g = dn.ops.prepare_operators(gX[0], gY[0])
    args = (x[0], mass[0], evals[0], evecs[0], g, blk.diffusion.diffusion_time, A_re, A_im,
            [l.weight for l in lins], [l.bias for l in lins], True)
    with torch.no_grad():
        out = torch.empty_like(x[0])
        assert dn.ops.block_forward_raw(*args, out=out) is out
        for bad in (torch.empty(x.shape[1], 63, device="cuda"), torch.empty_like(x[0], dtype=torch.float64),
                    torch.empty(64, x.shape[1], device="cuda").t()):
            with pytest.raises(ValueError):
                dn.ops.block_forward_raw(*args, out=bad)
