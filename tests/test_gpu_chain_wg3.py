"""The row chain on three consumer warpgroups: full-width TF32 chains of several layers at 128 without a sibling layer,
at sizes whose 128-row tiles would not fit in one wave on the SMs, run over 192-row tiles, with every later layer's
activations and the residual in the staging buffer (dn_tc.cu, `rows_chain_kernel<MODE, 128, true, 3>`).

What that path can get wrong and no other test checks: last tiles in which only consumer warpgroup 0 or 1 has rows,
or a warp only some of its rows, rows past V written, a residual loaded per warp in the columns the warp has just
read, hidden outputs stored from the same buffer the next layer reads, the fused head reading the finished rows
there, and the dispatch itself.

Results are bitwise equal to the two-warpgroup kernel's (the same chain over a slice of the rows, small enough for one
wave, takes that kernel; a row's result does not depend on the other rows), within the suite's bounds of the exact
fp32 SIMT engine (tc3x 1e-5, tc1x 16 u_tf32), and bitwise equal between two calls."""
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = {"tc3x": 1e-5, "tc1x": 16 * 2.0 ** -11}
ENGINES = list(TOL)
CANARY = -7.25e31     # what the rows past V hold before the call, and must hold after it
EXTRA = 200           # rows allocated past V: more than one 192-row tile
# rows in the last 192-row tile: 1 .. 63 (warpgroup 0 only, its last warp partly), 64, 65 (warpgroup 1 with one row),
# 127, 129 (warpgroup 2 with one row), 191, 192 (a full tile)
LAST_TILE = [1, 63, 64, 65, 127, 129, 191, 192]
CHAIN = re.compile(r"rows_chain_kernel<(\d+), (\d+), (true|false), (\d)>")


@pytest.fixture(scope="module")
def dn():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import diffusion_net_b200 as d
    d._lib.load()
    yield d
    d.set_engine("tc3x")


def _wave_rows():
    """Rows of one wave of 128-row tiles: the chain takes three warpgroups above this."""
    return 128 * torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _big(last):
    """A size past one wave of 128-row tiles whose last 192-row tile holds `last` rows."""
    return 192 * (_wave_rows() // 192 + 1) + last


def _chain_kernels(fn):
    """(mode, nmax, wide, consumer warpgroups) of every row-chain launch `fn` makes, from the profiler's kernel names."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    found = set()
    for e in prof.events():
        m = CHAIN.search(e.name)
        if m:
            found.add((int(m.group(1)), int(m.group(2)), m.group(3) == "true", int(m.group(4))))
    return found


def _mlp(dn, engine, srcs, Ws, bs, residual, out, hidden):
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


def _case(V, seed, k_in=(128, 128, 128)):
    g = torch.Generator().manual_seed(seed)
    srcs = [torch.randn(V, k, generator=g).cuda() for k in k_in]
    Ws = [(torch.randn(128, k, generator=g) * k ** -0.5).cuda() for k in (sum(k_in), 128, 128)]
    bs = [(torch.randn(128, generator=g) * 0.1).cuda() for _ in range(3)]
    res = torch.randn(V, 128, generator=g).cuda()
    return srcs, Ws, bs, res


def _rows(case, lo, hi):
    """The same chain over rows lo .. hi - 1 of the inputs."""
    srcs, Ws, bs, res = case
    return [s[lo:hi].contiguous() for s in srcs], Ws, bs, res[lo:hi].contiguous()


def _run(dn, engine, V, case, hidden):
    """The MiniMLP chain K0 -> 128 -> 128 -> 128 + residual, its output (and, with `hidden`, both hidden outputs) in
    buffers of V + EXTRA rows filled with CANARY: returns the buffers, the output last."""
    srcs, Ws, bs, res = case
    bufs = [torch.full((V + EXTRA, 128), CANARY, device="cuda") for _ in range(3 if hidden else 1)]
    _mlp(dn, engine, srcs, Ws, bs, res, bufs[-1].data_ptr(), bufs[:-1] if hidden else None)
    return bufs


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def _two_warpgroup_slices(dn, engine, V, case, hidden, got):
    """The first and the last 1000 rows, run alone (two warpgroups), equal `got`'s rows bit for bit."""
    for lo in (0, V - 1000):
        part = _run(dn, engine, 1000, _rows(case, lo, lo + 1000), hidden)
        for g, q in zip(got, part):
            assert torch.equal(g[lo:lo + 1000], q[:1000])


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("hidden", [False, True])
@pytest.mark.parametrize("last", LAST_TILE + [None])
def test_mini_mlp_tiles(dn, engine, hidden, last):
    """Every shape of the last 192-row tile past one wave, and V = 200k + 37 (many tiles per CTA through the same
    buffers).  Without hidden outputs the hidden layers leave nothing but the staging buffer; with them each is stored
    from the buffer the next layer reads.  Rows past V keep their canary bits, rows < V match the SIMT engine and,
    bitwise, the two-warpgroup kernel, and two calls are bitwise equal."""
    V = 200_037 if last is None else _big(last)
    case = _case(V, seed=V % 997)
    got = _run(dn, engine, V, case, hidden)
    again = _run(dn, engine, V, case, hidden)
    ref = _run(dn, "simt", V, case, hidden)
    for g, a, r in zip(got, again, ref):
        assert torch.equal(g, a)
        assert torch.all(g[V:] == CANARY)
        assert _rel(g[:V], r[:V]) < TOL[engine]
    _two_warpgroup_slices(dn, engine, V, case, hidden, got)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("k_in", [(128, 128, 128), (64,), (8,), (128, 120, 8)])
def test_layer0_widths(dn, engine, k_in):
    """Layer 0 as wide as the sources, narrower than its 128 outputs and with a half stage (K0 = 8, 128 + 120 + 8),
    the last tile partial."""
    V = _big(37)
    case = _case(V, seed=len(k_in) + k_in[-1], k_in=k_in)
    got = _run(dn, engine, V, case, False)
    assert torch.equal(got[0], _run(dn, engine, V, case, False)[0])
    assert torch.all(got[0][V:] == CANARY)
    assert _rel(got[0][:V], _run(dn, "simt", V, case, False)[0][:V]) < TOL[engine]
    _two_warpgroup_slices(dn, engine, V, case, False, got)


def test_dispatch(dn):
    """tc3x / tc1x full-width chains of several layers without a sibling take three consumer warpgroups past one wave
    of 128-row tiles and two within it; bf16 and single-layer chains keep two; in a block forward at C = 128 the front
    chain (from_basis, [P|Q] with Q as sibling) keeps two while the MiniMLP takes three."""
    V = _big(5)
    case = _case(V, seed=1)
    assert _chain_kernels(lambda: _run(dn, "tc3x", V, case, False)) == {(3, 128, True, 3)}
    assert _chain_kernels(lambda: _run(dn, "tc1x", V, case, False)) == {(1, 128, True, 3)}
    assert _chain_kernels(lambda: _run(dn, "bf16", V, case, False)) == {(16, 128, True, 2)}
    w = _wave_rows()
    assert _chain_kernels(lambda: _run(dn, "tc3x", w, _rows(case, 0, w), False)) == {(3, 128, True, 2)}
    assert _chain_kernels(lambda: _run(dn, "tc3x", w + 1, _rows(case, 0, w + 1), False)) == {(3, 128, True, 3)}
    srcs, Ws, bs, res = case
    one = torch.empty(V, 128, device="cuda")
    assert _chain_kernels(lambda: _mlp(dn, "tc3x", srcs, Ws[:1], bs[:1], res, one.data_ptr(), None)) == \
        {(3, 128, True, 2)}
    dn.set_engine("tc3x")
    blk, x, ops = _block(dn, 128)
    with torch.no_grad():
        kinds = _chain_kernels(lambda: blk(x, *ops))
    assert (3, 128, True, 3) in kinds and (3, 128, True, 2) in kinds, kinds


def _block(dn, C, K=64, dropout=False):
    """A C-wide block on a synthetic mesh of n x m > one wave of 128-row tiles vertices."""
    n = 150
    m = _wave_rows() // n + 3
    mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=0, device="cuda")
    blk = dn.DiffusionNetBlock(C_width=C, mlp_hidden_dims=[C, C], dropout=dropout)
    blk.load_state_dict(dn.synthetic.block_weights(C, seed=3), strict=True)
    blk = blk.cuda()
    x = torch.randn(1, n * m, C, generator=torch.Generator().manual_seed(5)).cuda()
    return blk, x, (mass.unsqueeze(0), None, evals.unsqueeze(0), evecs.unsqueeze(0), [gX], [gY])


@pytest.mark.parametrize("engine", ENGINES)
def test_fused_head(dn, engine):
    """The linear head behind the last MiniMLP layer reads the finished rows from the staging buffer: it equals the
    head applied in fp64 to the block output of the same engine, and two calls are bitwise equal."""
    dn.set_engine(engine)
    blk, x, ops = _block(dn, 128)
    blk.eval()
    g = torch.Generator().manual_seed(9)
    head = ((torch.randn(5, 128, generator=g) / 11).cuda(), torch.randn(5, generator=g).cuda())
    with torch.no_grad():
        y = blk(x, *ops)
        h = blk(x, *ops, head=head)
        h2 = blk(x, *ops, head=head)
    torch.cuda.synchronize()
    assert torch.equal(h, h2)
    ref = y.double() @ head[0].double().t() + head[1].double()
    assert _rel(h, ref) < 1e-6


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("dropout", [False, True])
def test_backward_chains(dn, engine, dropout):
    """A C = 128 block trained one step: the MiniMLP forward stores its hidden outputs from the staging buffer on three
    warpgroups (the single-layer backward chains keep two).  The block output, which that forward computes, matches the
    SIMT engine's, and the output and every gradient are bitwise equal between two steps.  (The hidden layers' weight
    and bias gradients are column sums over 19k rows behind ReLU masks and come from the backward kernels; against the
    SIMT engine they differ by up to 6e-4 in tc3x and 3e-2 in tc1x.)"""
    def step(eng):
        dn.set_engine(eng)
        torch.manual_seed(11)
        blk, x, ops = _block(dn, 128, dropout=dropout)
        blk.train()
        xg = x.clone().requires_grad_(True)
        torch.manual_seed(12)
        y = blk(xg, *ops)
        (y * torch.linspace(-1, 1, y.numel(), device="cuda").view_as(y)).sum().backward()
        torch.cuda.synchronize()
        return [y.detach(), xg.grad] + [p.grad for p in blk.parameters()]

    dn.set_engine(engine)
    kinds = _chain_kernels(lambda: step(engine))
    assert any(k[3] == 3 for k in kinds), kinds
    got, again, ref = step(engine), step(engine), step("simt")
    for g, a in zip(got, again):
        assert torch.equal(g, a)
    assert _rel(got[0], ref[0]) < TOL[engine]
