"""The row chain's output path at NMAX <= 128: each consumer warpgroup stages a layer's result in shared memory and one
lane writes it with 2-D TMA stores (rows >= V clipped by the tensor map); a layer's residual comes in through the same
buffer by TMA.  What that path can get wrong and no other test checks: writes past row V-1 of an over-allocated
buffer, a warpgroup wholly past V, reuse of the buffer across many tiles ending on a partial one, a head-only last
layer, and the alignment rule that sends other outputs to the SIMT kernel.

Results are checked against the exact fp32 SIMT engine under the suite's bounds (tc3x 1e-5, tc1x 16 u_tf32,
bf16 2e-2), and two calls must give the same bits."""
import os
import sys

import pytest
import torch

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle as O  # noqa: E402  (checker only)

pytestmark = pytest.mark.gpu

TOL = {"tc3x": 1e-5, "tc1x": 16 * 2.0 ** -11, "bf16": 2e-2}
ENGINES = list(TOL)
CANARY = -7.25e31     # what the rows past V hold before the call, and must hold after it
EXTRA = 150           # rows allocated past V: more than one 128-row tile


@pytest.fixture(scope="module")
def dn():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import diffusion_net_b200 as d
    d._lib.load()
    yield d
    d.set_engine("tc3x")


def _mlp_raw(dn, engine, srcs, Ws, bs, residual, out, hidden):
    """dn_mini_mlp_fwd over raw pointers: `out` (and each hidden output) may sit inside a larger buffer."""
    lib = dn._lib.load()
    V = srcs[0].shape[0]
    widths = [s.shape[1] for s in srcs]
    dims = [sum(widths)] + [w.shape[0] for w in Ws]
    ws = dn.ops.workspace(V, max(dims), max(dims), torch.device("cuda", torch.cuda.current_device()))
    dn._lib.check(lib.dn_mini_mlp_fwd(
        dn._lib.ptr_array([s.data_ptr() for s in srcs]), dn._lib.int_array(widths), len(srcs),
        dn._lib.ptr_array([w.data_ptr() for w in Ws]), dn._lib.ptr_array([b.data_ptr() for b in bs]),
        dn._lib.int_array(dims), len(Ws), None, residual.data_ptr() if residual is not None else None, V,
        dn._lib.ptr_array([h.data_ptr() for h in hidden]) if hidden else None, out, ws.data_ptr(), ws.numel(),
        dn.ops._ENGINES[engine], dn.ops._stream()), "dn_mini_mlp_fwd")
    torch.cuda.synchronize()


def _case(V, seed):
    g = torch.Generator().manual_seed(seed)
    srcs = [torch.randn(V, 128, generator=g).cuda() for _ in range(3)]
    Ws = [(torch.randn(128, k, generator=g) * k ** -0.5).cuda() for k in (384, 128, 128)]
    bs = [(torch.randn(128, generator=g) * 0.1).cuda() for _ in range(3)]
    res = torch.randn(V, 128, generator=g).cuda()
    return srcs, Ws, bs, res


def _run(dn, engine, V, srcs, Ws, bs, res):
    """The MiniMLP chain 384 -> 128 -> 128 -> 128 + residual with every output (hidden ones too) in a buffer of
    V + EXTRA rows filled with CANARY: returns the full buffers."""
    bufs = [torch.full((V + EXTRA, 128), CANARY, device="cuda") for _ in range(3)]
    _mlp_raw(dn, engine, srcs, Ws, bs, res, bufs[2].data_ptr(), [bufs[0], bufs[1]])
    return bufs


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("V", [37, 200_037])
def test_rows_past_v_untouched(dn, engine, V):
    """V = 37: one partial tile whose second warpgroup (rows 64..127) lies wholly past V.  V = 200k + 37: every CTA
    runs many tiles through its staging buffer and the last tile is partial.  Rows V .. V+EXTRA-1 of every output
    (the two hidden layers and the residual layer) keep their canary bits; rows < V match the SIMT engine, and two
    calls are bitwise equal."""
    srcs, Ws, bs, res = _case(V, seed=V % 1000)
    got = _run(dn, engine, V, srcs, Ws, bs, res)
    again = _run(dn, engine, V, srcs, Ws, bs, res)
    ref = _run(dn, "simt", V, srcs, Ws, bs, res)
    for a, b, r in zip(got, again, ref):
        assert torch.equal(a, b)
        assert bool((a[V:] == CANARY).all())
        assert O.rel_err(a[:V].cpu().numpy(), r[:V].cpu().numpy()) < TOL[engine]


@pytest.mark.parametrize("engine", ENGINES)
def test_head_only_last_layer(dn, engine):
    """A network's last block with its linear head fused: the MiniMLP's last layer has a residual but no `out`, so its
    staging buffer takes the residual and nothing is stored from it.  The head output matches the head applied to the
    block output of the same engine, and two calls are bitwise equal."""
    dn.set_engine(engine)
    n, m, K, C = 30, 35, 64, 128          # V = 1050: 8 full tiles and a partial one
    mass, _, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=3, device="cuda")
    blk = dn.DiffusionNetBlock(C_width=C, mlp_hidden_dims=[C, C], dropout=False)
    blk.load_state_dict(dn.synthetic.block_weights(C, seed=3), strict=True)
    blk = blk.cuda().eval()
    g = torch.Generator().manual_seed(3)
    x = torch.randn(n * m, C, generator=g).cuda()
    hw, hb = (torch.randn(5, C, generator=g) * C ** -0.5).cuda(), (torch.randn(5, generator=g) * 0.1).cuda()
    gops = dn.prepare_operators(gX, gY)
    A_re, A_im = blk.gradient_features.weights()
    lins = blk.mlp.linears()

    def fwd(head):
        with torch.no_grad():
            y = dn.ops.block_forward_raw(x, mass, evals, evecs, gops, blk.diffusion.diffusion_time, A_re, A_im,
                                         [l.weight for l in lins], [l.bias for l in lins], True, head=head)
        torch.cuda.synchronize()
        return y

    h0, h1, y = fwd((hw, hb)), fwd((hw, hb)), fwd(None)
    assert torch.equal(h0, h1)
    gold = y.double() @ hw.double().t() + hb.double()
    assert O.rel_err(h0.cpu().numpy(), gold.cpu().numpy()) < TOL[engine]


@pytest.mark.parametrize("what", ["out", "residual"])
def test_out_not_16_byte_aligned_takes_simt(dn, capfd, what):
    """An output or residual 8 bytes past a 16-byte boundary cannot be a TMA tensor map: the chain refuses it and the
    layer runs on the exact SIMT kernel (bitwise the SIMT engine's result), which says so once on stderr (DN_STRICT_TC=1
    turns it into an error)."""
    V, K = 300, 104
    N = 112 if what == "out" else 96     # shapes no other test sends to the SIMT kernel
    g = torch.Generator().manual_seed(11)
    src = torch.randn(V, K, generator=g).cuda()
    W, b = (torch.randn(N, K, generator=g) * K ** -0.5).cuda(), (torch.randn(N, generator=g) * 0.1).cuda()
    res_buf = torch.zeros(V * N + 2, device="cuda")
    res = res_buf[2:].view(V, N) if what == "residual" else res_buf[:V * N].view(V, N)
    res.copy_(torch.randn(V, N, generator=g).cuda())

    def run(engine):
        buf = torch.zeros(V * N + 2, device="cuda")
        out = buf[2:].view(V, N) if what == "out" else buf[:V * N].view(V, N)
        assert (out if what == "out" else res).data_ptr() % 16 == 8
        _mlp_raw(dn, engine, [src], [W], [b], res, out.data_ptr(), None)
        return out

    strict = os.environ.get("DN_STRICT_TC", "0") not in ("", "0")
    if strict:
        with pytest.raises(RuntimeError, match="unsupported"):
            run("tc3x")
        return
    got = run("tc3x")
    assert torch.equal(got, run("simt"))
    assert "K={}, N={} is outside the tensor-core kernels' envelope".format(K, N) in capfd.readouterr().err
