"""The mesh-batch and pair-batch routes at dataset scale against fp64: hundreds of meshes through ``forward_batch``,
``project_batched`` across its engines, widths and spectral sizes, ``pointwise_map_batch`` over several chunks and every
nearest-neighbour width NP, ``fmap_solve_batched`` at the pair cap, and ``compute_operators_batch`` on ~150 meshes.

These are the shapes a dataset of a few hundred small meshes or shape pairs sends down the batched route; the other
batch tests use a handful of meshes, so the planner branches that only run with many meshes (one CTA per mesh, the
``want = 1`` clamp of ``dn_mesh_batch_plan``, the 1024-mesh cap, pair chunking in ``dn_fmap_pointwise_map_batched``)
are exercised here, on the kernels that consume them.

Every bound is one an existing per-mesh or per-pair test already justifies, cited where it is used:
  * forward_batch output, tc3x: 1e-5 (test_gpu_operators_batch.py::test_batched_operators_drive_forward_batch);
    parameter and input gradients: 5e-5 (test_gpu_batch_train.py::test_forward_batch_gradients_vs_oracle_accumulation);
    tc1x / bf16 against the per-mesh route: DIFF_TOL of test_gpu_batch_train.py.  Gradients are compared under our
    ReLU pattern with test_gpu_backward.py's kink rule (_check_kinks): at this scale a few hidden pre-activations
    sit within rounding of zero (see test_forward_batch_many_meshes_gradients_against_fp64).
  * projection: the componentwise TOL[engine] sum_v |Phi[v][k] m[v] x[v][c]| of test_gpu_to_basis.py (2^-13 tc3x, 2^-8
    tc1x), the adjoint bounded the same way over its K terms (test_gpu_fmaps_batch.py::
    test_projection_forward_and_adjoint_against_fp64).
  * nearest neighbour / pointwise map: bitwise the per-pair ``pointwise_map``, and the certainty rule of
    test_gpu_fmaps.py::_check_nn against an fp64 brute force on the same fp32 operands.
  * batched solve: C bitwise the per-pair ``FmapSolveFn``, and against fp64 the per-row and (tol + m u) per-shape
    gradient bounds of test_gpu_fmaps_batch.py::test_solve_batched_matches_per_pair_bitwise_and_fp64.
  * operators: test_gpu_operators_batch.py::_check_against.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle as O  # noqa: E402  (checker only)
import dn_oracle_fmaps as OF  # noqa: E402
import dn_oracle_ops as OO  # noqa: E402

import diffusion_net_b200 as dn  # noqa: E402
import diffusion_net_b200.eigen  # noqa: E402,F401  (dn.eigen: not imported at package level)

from test_gpu_batch_train import DIFF_TOL, _batched_loss, _grads, _inputs, _net, _zero  # noqa: E402
from test_gpu_backward import TOL as BWD_TOL, _check_kinks, _mlp_node  # noqa: E402
from test_gpu_fmaps import U32, _check_nn  # noqa: E402
from test_gpu_fmaps_batch import LAMBDA, _kappa, _stack_inputs  # noqa: E402
from test_gpu_operators_batch import _check_against  # noqa: E402

gpu = pytest.mark.gpu
EPS64 = 2.0 ** -53
TB_TOL = {"tc3x": 2.0 ** -13, "tc1x": 2.0 ** -8}     # test_gpu_to_basis.py TOL
MAX_CTAS = 1024                                        # dn_mesh_batch_plan's to_basis CTA budget


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    dn._lib.load()
    yield torch.device("cuda")
    dn.set_engine("tc3x")


def _launches():
    return dn._lib.load().dn_kernel_launch_count()


def _np(t):
    return t.detach().cpu().numpy()


# ---- models of the host planners -----------------------------------------------------------------------------------
def _mesh_plan_model(n_rows, sm):
    """dn_mesh_batch_plan's CTAs per mesh, and which meshes took the one-CTA fallback (a proportional share below one)
    and the want = 1 clamp (a proportional share of two or more cut to one because the 1024-CTA budget is full)."""
    B = len(n_rows)
    chunks = [(v + 15) // 16 for v in n_rows]
    total = sum(chunks)
    ctas, fallback, clamped = [], [], []
    n_ctas = 0
    for b, c in enumerate(chunks):
        want = (c * sm + total // 2) // total if total > 0 else 1
        if want < 1:
            want = 1
            fallback.append(b)
        if want > c > 0:
            want = c
        if n_ctas + want + (B - 1 - b) > MAX_CTAS:
            if want > 1:
                clamped.append(b)
            want = 1
        per = -(-c // want) if c > 0 else 0
        if per > 0:
            want = -(-c // per)
        ctas.append(want)
        n_ctas += want
    return ctas, fallback, clamped


PM_CHUNK_PAIRS = 64                 # dn_fmap_batch.cu kPmChunkPairs
PM_CHUNK_FLOATS = 16 << 20          # kPmChunkFloats
NN_TILE_FLOATS, NN_THREADS, NN_TARGET_CTAS, NN_MAX_SPLIT = 8192, 128, 264, 16   # dn_fmap_common.cuh


def _np_of(n):
    p = 4
    while p < n:
        p *= 2
    return p


def _pm_plan_model(n, pairs, n_rows):
    """pm_plan of dn_fmap_batch.cu: the chunks (lists of pair indices) with their target-range splits, and the workspace
    (the largest chunk's T plus its split partials)."""
    NP = _np_of(n)
    tt = NN_TILE_FLOATS // NP
    a256 = lambda b: (b + 255) // 256 * 256
    chunks, ws, p = [], 0, 0
    while p < len(pairs):
        members, t_rows, src_rows, qblk, max_tiles = [], 0, 0, 0, 1
        while p < len(pairs) and len(members) < PM_CHUNK_PAIRS:
            x, y = pairs[p]
            vt, vs = n_rows[x], n_rows[y]
            if members and (t_rows + vt) * NP > PM_CHUNK_FLOATS:
                break
            members.append(p)
            t_rows += vt
            src_rows += vs
            qblk += -(-vs // NN_THREADS)
            max_tiles = max(max_tiles, -(-vt // tt))
            p += 1
        s = -(-NN_TARGET_CTAS // qblk) if qblk > 0 else 1
        s = min(max(s, 1), NN_MAX_SPLIT, max_tiles)
        chunks.append((members, s))
        ws = max(ws, a256(t_rows * NP * 4) + (a256(8 * s * src_rows) if s > 1 else 0))
    return chunks, ws


# pair-batch layouts of the pointwise-map cases (target x, source y; V of each shape)
PM_SHAPES = [(10, 20), (13, 31), (40, 75), (16, 16), (9, 15), (30, 41), (20, 20), (11, 12), (25, 60), (8, 16),
             (17, 19), (35, 35)]                                  # V 128 .. 3000


def _pm_pairs(n_shapes=len(PM_SHAPES), P=150, seed=0):
    rs = np.random.RandomState(seed)
    pairs = [(int(a), int(b)) for a, b in zip(rs.randint(n_shapes, size=P), rs.randint(n_shapes, size=P))]
    pairs[5], pairs[70], pairs[140] = (2, 2), (2, 0), (5, 2)      # the duplicated-row shapes as target in every chunk
    return pairs


# at n = 128 (16 Mi floats = 131072 target rows): two ~80k-row targets never share a chunk -> chunks of 1, 3, 1 pairs
BIG_SHAPES = [(280, 286), (281, 285), (10, 20), (13, 31), (8, 16)]
BIG_PAIRS = [(0, 2), (1, 3), (2, 4), (3, 2), (0, 4)]
# a 200k-row target is a chunk of its own, above the limit -> chunks of 2, 1, 1 pairs
HUGE_SHAPES = [(400, 500), (10, 20), (13, 31)]
HUGE_PAIRS = [(1, 2), (2, 1), (0, 1), (0, 2)]
PM_CHUNKS_128 = {"80k targets": [1, 3, 1], "200k target": [2, 1, 1]}


def _layouts():
    return {"150 pairs": ([a * b for a, b in PM_SHAPES], _pm_pairs()),
            "80k targets": ([a * b for a, b in BIG_SHAPES], BIG_PAIRS),
            "200k target": ([a * b for a, b in HUGE_SHAPES], HUGE_PAIRS)}


@pytest.mark.parametrize("n", [3, 5, 12, 30, 50, 128])
def test_pointwise_map_workspace_matches_the_chunk_model(n):
    """Host only: dn_fmap_pointwise_map_batched_workspace_bytes against the chunking model above, and the model's
    chunks are what the GPU tests below rely on (64 + 64 + 22 pairs; a chunk broken on the float limit; one pair over
    it)."""
    lib = dn._lib.load()
    for name, (n_rows, pairs) in _layouts().items():
        chunks, ws = _pm_plan_model(n, pairs, n_rows)
        rb = np.concatenate([[0], np.cumsum([(v + 127) // 128 * 128 for v in n_rows])[:-1]])
        got = lib.dn_fmap_pointwise_map_batched_workspace_bytes(
            n, len(pairs), dn._lib.int_array([a for a, _ in pairs]), dn._lib.int_array([b for _, b in pairs]),
            dn._lib.int_array(rb), dn._lib.int_array(n_rows), len(n_rows))
        assert got == ws, (name, got, ws)
        sizes = [len(m) for m, _ in chunks]
        if name == "150 pairs":
            assert sizes == [64, 64, 22]
        elif n == 128:
            assert sizes == PM_CHUNKS_128[name]


# =====================================================================================================================
# 1. many meshes through forward_batch
# =====================================================================================================================
K1, C1 = 16, 32
FIXED_1 = [(4, 4), (9, 14), (8, 16), (10, 13), (60, 80), (48, 100)]   # V = K, 126, 128, 130, and two of ~5k rows


def _scale_shapes(B, seed=0):
    """B ragged meshes: V from K to a few hundred, the fixed ones spread over the batch (two large meshes near its end,
    so their proportional share of CTAs exceeds one and late tiles look up large mesh indices)."""
    rs = np.random.RandomState(seed)
    out = []
    while len(out) < B - len(FIXED_1):
        a, b = (int(v) for v in rs.randint(3, 21, size=2))
        if a * b >= K1:
            out.append((a, b))
    for pos, s in zip((0, B // 3, B // 2, 2 * B // 3, B - 2, B - 1), FIXED_1):
        out.insert(pos, s)
    return out


_mesh_cache = {}


def _scale_meshes(B):
    if B not in _mesh_cache:
        items = []
        for i, (a, b) in enumerate(_scale_shapes(B)):
            mass, _, evals, evecs, gX, gY = dn.synthetic.structural_operators(a, b, K1, seed=i, device="cuda")
            items.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY))
        _mesh_cache[B] = (items, dn.MeshBatch(items))
    return _mesh_cache[B]


def _csr64(t):
    t = t.coalesce().cpu()
    i = t.indices().numpy()
    return sp.csr_matrix((t.values().numpy().astype(np.float64), (i[0], i[1])), shape=tuple(t.shape))


def _check_plan(mb):
    sm = torch.cuda.get_device_properties(mb.device).multi_processor_count
    ctas, fallback, clamped = _mesh_plan_model(mb.n_rows, sm)
    cb = _np(mb._cta_begin)
    assert np.array_equal(np.diff(cb), ctas)
    tb = _np(mb._tb_rows).reshape(-1, 2)
    for b in range(mb.n_meshes):
        r = tb[cb[b]:cb[b + 1]]
        assert r[0, 0] == mb.row_begin[b] and r[-1, 1] == mb.row_begin[b] + mb.n_rows[b], b
        assert (r[1:, 0] == r[:-1, 1]).all() and (r[:, 1] > r[:, 0]).all(), b
    return ctas, fallback, clamped


@gpu
@pytest.mark.parametrize("B", [300, 1024])
def test_forward_batch_many_meshes_against_fp64(cuda, B):
    """The plan took the one-CTA-per-mesh fallback (and at 1024 meshes the want = 1 clamp); the forward (eval, the
    fused batched block) against O.diffusion_net for every mesh."""
    dn.set_engine("tc3x")
    items, mb = _scale_meshes(B)
    ctas, fallback, clamped = _check_plan(mb)
    assert len(fallback) > B // 2, "the proportional split did not fall back to one CTA per mesh"
    big = [b for b in range(B) if mb.n_rows[b] > 4000]
    if B == 1024:
        assert sum(ctas) == MAX_CTAS and all(c == 1 for c in ctas)
        assert set(big) <= set(clamped), "the want = 1 clamp did not fire"
    else:
        assert not clamped and all(ctas[b] > 1 for b in big)
    net = _net(dn, C1, K1)
    xs, ys = _inputs(items)
    params = {k: _np(v).astype(np.float64) for k, v in net.state_dict().items()}
    net.eval()
    with torch.no_grad():
        outs = net.forward_batch(mb, xs)
    worst = 0.0
    for b, (it, x) in enumerate(zip(items, xs)):
        want = O.diffusion_net(_np(x).astype(np.float64), _np(it["mass"]).astype(np.float64),
                               _np(it["evals"]).astype(np.float64), _np(it["evecs"]).astype(np.float64),
                               _csr64(it["gradX"]), _csr64(it["gradY"]), params, 2)
        e = O.rel_err(_np(outs[b]), want)
        worst = max(worst, e)
        assert e <= 1e-5, (b, mb.n_rows[b], e)
    print("B = {}: {} CTAs, {} meshes at one CTA by fallback, {} clamped; forward worst {:.2e}".format(
        B, sum(ctas), len(fallback), len(clamped), worst))


def _oracle_grads_masked(net, items, xs, ys, rows, masks, NB, engine="tc3x"):
    """test_gpu_batch_train.py::_oracle_grads (fp64 autograd accumulated over the meshes) with every hidden ReLU taken
    under our activation pattern: ``masks[k]`` the batch-layout masks of block k, sliced to each mesh's ``rows``
    (first row, row count).  Checks each mesh's flips with test_gpu_backward.py::_check_kinks for ``engine`` and
    returns (gold, gold_x, [(mesh, block, flips)])."""
    import dn_oracle_torch as T
    d = torch.float64
    prm = {k: v.detach().cpu().to(d).requires_grad_(True) for k, v in net.state_dict().items()}
    xgs = [x.detach().cpu().to(d).requires_grad_(True) for x in xs]
    flipped = []
    for b, (it, xg, y) in enumerate(zip(items, xgs, ys)):
        r0, n = rows[b]
        mass, evals, evecs = (it[k].cpu().to(d) for k in ("mass", "evals", "evecs"))
        h = torch.addmm(prm["first_lin.bias"], xg, prm["first_lin.weight"].t()).unsqueeze(0)
        for k in range(NB):
            bp = {key[len("block_%d." % k):]: v for key, v in prm.items() if key.startswith("block_%d." % k)}
            mk = [m[r0:r0 + n] for m in masks[k]]
            pre = []
            h = T.block_forward(h, mass.unsqueeze(0), evals.unsqueeze(0), evecs.unsqueeze(0), [it["gradX"].cpu().to(d)],
                                [it["gradY"].cpu().to(d)], bp, relu_masks=mk, pre_acts=pre)
            _check_kinks(mk, pre, engine)
            nf = sum(int((m != (p.reshape(m.shape) > 0)).sum()) for m, p in zip(mk, pre))
            if nf:
                flipped.append((b, k, nf))
        logits = torch.addmm(prm["last_lin.bias"], h[0], prm["last_lin.weight"].t())
        torch.nn.functional.cross_entropy(logits, y.cpu()).backward()
    return {k: v.grad for k, v in prm.items()}, [x.grad for x in xgs], flipped


def _rows(mb):
    return [(mb.row_begin[b], mb.n_rows[b]) for b in range(mb.n_meshes)]


def _relu_masks(out, net):
    """Every block's hidden ReLU pattern, read from the MLPFn node ``out`` came through (before its backward)."""
    return {k: [(h > 0).cpu() for h in _mlp_node(out, net.blocks[k].mlp.linears()[0].weight)[0]]
            for k in range(len(net.blocks))}


@gpu
@pytest.mark.parametrize("B", [300, 1024])
def test_forward_batch_many_meshes_gradients_against_fp64(cuda, B):
    """Parameter gradients against fp64 autograd accumulated over all meshes, and every x.grad (train, the
    differentiable batched blocks), at 5e-5.

    ReLU kinks.  The batch holds some 10^6 (B = 300) to 10^7 (B = 1024) hidden pre-activations, and the batched
    to_basis sums each mesh's spectral coefficients in another order than the per-mesh route, so a pre-activation within
    fp32 rounding of zero can land on the other side of the kink from fp64.  That flips one unit's ReLU derivative and
    moves the gradient of its vertex by the unit's whole weight: with these seeds, the 48 x 100 torus at the end of the
    batch gets an x.grad 4.3e-3 from an fp64 gold that takes ReLU on its own pattern, while the per-mesh route (another
    summation order) lands on fp64's side.  A plain fp64 gold therefore does not bound the batch's gradients at 5e-5 at
    this scale.  As test_gpu_backward.py does, the gold takes every ReLU under our pattern (read from the MLPFn node's
    saved activations), and ``_check_kinks`` requires each flip to lie within KINK of zero (1e-5 max|pre-activation|
    for tc3x) and the flips to be few; the 5e-5 bounds then hold unchanged."""
    dn.set_engine("tc3x")
    items, mb = _scale_meshes(B)
    net = _net(dn, C1, K1)
    xs, ys = _inputs(items)
    xg = [x.clone().requires_grad_(True) for x in xs]
    _zero(net)
    outs = net.forward_batch(mb, xg)
    masks = _relu_masks(outs[0], net)
    _batched_loss(outs, ys, "vertices").backward()
    gold, gold_x, flipped = _oracle_grads_masked(net, items, xg, ys, _rows(mb), masks, 2)
    print("B = {}: ReLU flips against fp64 (mesh, block, count): {}".format(B, flipped))
    for name, p_ in net.named_parameters():
        assert O.rel_err(_np(p_.grad), gold[name].numpy()) < 5e-5, name
    for b, (x, gx) in enumerate(zip(xg, gold_x)):
        assert O.rel_err(_np(x.grad), gx.numpy()) < 5e-5, (b, mb.n_rows[b])


@gpu
@pytest.mark.parametrize("B", [300, 1024])
def test_many_meshes_padding_rows_are_isolated(cuda, B):
    """Finite garbage in every mesh's padding rows changes neither an output nor a gradient (as
    test_gpu_batch_train.py::test_padding_rows_are_isolated)."""
    dn.set_engine("tc3x")
    items, mb = _scale_meshes(B)
    assert mb.V > sum(mb.n_rows)
    net = _net(dn, C1, K1)
    xs, ys = _inputs(items)
    clean = mb.pack(xs)
    dirty = clean.clone()
    g = torch.Generator().manual_seed(9)
    for b in range(B):
        r1, end = mb.row_begin[b] + mb.n_rows[b], mb.row_begin[b + 1]
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


@gpu
@pytest.mark.parametrize("B", [300, 1024])
@pytest.mark.parametrize("engine", ["tc1x", "bf16"])
def test_forward_batch_many_meshes_vs_per_mesh(cuda, B, engine):
    """tc1x / bf16: outputs, every x.grad and the parameter gradients against the same engine's per-mesh route,
    DIFF_TOL[engine].

    The two routes round the spectral sums in different orders, so a hidden pre-activation within the engine's rounding
    of zero may take the other side of a ReLU kink in each (see test_forward_batch_many_meshes_gradients_against_fp64):
    that mesh's x.grad then differs by a whole unit's weight, not by rounding.  A mesh whose ReLU patterns agree in
    both routes is held to DIFF_TOL; a mesh whose patterns differ (a few per 1000) is checked against fp64 under the
    batch's own pattern instead, with test_gpu_backward.py's input-gradient bound and kink rule for the engine."""
    dn.set_engine(engine)
    try:
        items, mb = _scale_meshes(B)
        net = _net(dn, C1, K1)
        xs, ys = _inputs(items)
        _zero(net)
        ref_out, ref_x, ref_masks = [], [], []
        for it, x, y in zip(items, xs, ys):
            xr = x.clone().requires_grad_(True)
            out = net(xr, it["mass"], evals=it["evals"], evecs=it["evecs"], gradX=it["gradX"], gradY=it["gradY"])
            ref_masks.append(_relu_masks(out, net))
            torch.nn.functional.cross_entropy(out, y).backward()
            ref_out.append(out.detach())
            ref_x.append(xr.grad)
        ref = _grads(net)
        _zero(net)
        xg = [x.clone().requires_grad_(True) for x in xs]
        outs = net.forward_batch(mb, xg)
        masks = _relu_masks(outs[0], net)
        _batched_loss(outs, ys, "vertices").backward()
        tol = DIFF_TOL[engine]
        rows = _rows(mb)
        differ = []
        for b, (r0, n) in enumerate(rows):
            assert O.rel_err(_np(outs[b]), _np(ref_out[b])) < tol, (b, n)
            if all(torch.equal(ref_masks[b][k][i].reshape(-1), masks[k][i][r0:r0 + n].reshape(-1))
                   for k in masks for i in range(len(masks[k]))):
                assert O.rel_err(_np(xg[b].grad), _np(ref_x[b])) < tol, (b, n)
            else:
                differ.append(b)
        for name, p_ in net.named_parameters():
            assert O.rel_err(_np(p_.grad), _np(ref[name])) < tol, name
    finally:
        dn.set_engine("tc3x")
    print("{} B = {}: meshes whose ReLU pattern differs between the routes: {}".format(engine, B, differ))
    assert len(differ) <= max(1, B // 100)
    if differ:
        sub = [items[b] for b in differ]
        _, gold_x, _ = _oracle_grads_masked(net, sub, [xg[b] for b in differ], [ys[b] for b in differ],
                                            [rows[b] for b in differ], masks, len(net.blocks), engine)
        for b, gx in zip(differ, gold_x):
            assert O.rel_err(_np(xg[b].grad), gx.numpy()) < BWD_TOL[engine][1], (b, rows[b][1])


@gpu
def test_mesh_and_pair_batches_take_1024_and_refuse_1025_before_any_launch(cuda):
    items, mb = _scale_meshes(1024)
    assert mb.n_meshes == 1024
    pb = dn.PairBatch(items, [(0, 1023), (1023, 512)], n_fmap=8)
    assert pb.mesh_batch.n_meshes == 1024 and pb.mesh_batch.row_begin == mb.row_begin
    more = items + items[:1]
    torch.cuda.synchronize()
    l0 = _launches()
    with pytest.raises(RuntimeError, match="unsupported"):
        dn.MeshBatch(more)
    with pytest.raises(ValueError, match="1025 shapes exceed the 1024"):
        dn.PairBatch(more, [(0, 1)], n_fmap=8)
    assert _launches() == l0


# =====================================================================================================================
# 2. project_batched across its envelope
# =====================================================================================================================
RAGGED_5 = [(5, 10), (1, 127), (8, 16), (3, 43), (50, 100)]     # V = 50, 127, 128, 129, 5000 (test_gpu_fmaps_batch.py)
_proj_cache = {}


def _proj_shapes(S, n):
    if S == 5:
        base = RAGGED_5
    else:
        rs = np.random.RandomState(S)
        base = [(int(a), int(b)) for a, b in zip(rs.randint(3, 25, size=S), rs.randint(3, 25, size=S))]
    return [(a, max(b, -(-n // a))) for a, b in base]          # V >= K = n (an M-orthonormal n-column basis)


def _proj_batch(S, n):
    if (S, n) not in _proj_cache:
        items = []
        for i, (a, b) in enumerate(_proj_shapes(S, n)):
            mass, _, evals, evecs, gX, gY = dn.synthetic.structural_operators(a, b, n, seed=7 * i + n, device="cuda")
            items.append({"mass": mass, "evals": evals, "evecs": evecs, "gradX": gX, "gradY": gY})
        _proj_cache[(S, n)] = (items, dn.PairBatch(items, [(0, S - 1)], n_fmap=n))
    return _proj_cache[(S, n)]


@gpu
@pytest.mark.parametrize("S", [5, 300])
@pytest.mark.parametrize("n", [5, 30, 100, 128])
@pytest.mark.parametrize("Cc", [16, 48, 128, 256])
@pytest.mark.parametrize("engine", ["tc3x", "tc1x"])
def test_projection_envelope_against_fp64(cuda, engine, Cc, n, S):
    dn.set_engine(engine)
    try:
        items, pb = _proj_batch(S, n)
        mb = pb.mesh_batch
        assert pb.kp == {5: 8, 30: 32, 100: 104, 128: 128}[n]
        g = torch.Generator().manual_seed(Cc + n + S)
        xs = [torch.randn(it["mass"].shape[0], Cc, generator=g) for it in items]
        feat = mb.pack([x.cuda() for x in xs]).requires_grad_(True)
        out = dn.fmaps.project_batched(feat, pb)
        assert out.shape == (S, pb.kp, Cc)
        G = torch.randn(S, pb.kp, Cc, generator=g)
        out.backward(G.cuda())
        torch.cuda.synchronize()
    finally:
        dn.set_engine("tc3x")
    tol = TB_TOL[engine]
    outn, grad = out.detach().cpu().double().numpy(), feat.grad.cpu().double().numpy()
    assert (outn[:, n:] == 0).all()
    worst = 0.0
    for s, (it, x) in enumerate(zip(items, xs)):
        phi = np.zeros((x.shape[0], pb.kp))
        phi[:, :n] = _np(it["evecs"][:, :n]).astype(np.float64)
        m = _np(it["mass"]).astype(np.float64)
        xd = x.double().numpy() * m[:, None]
        gold, absum = phi.T @ xd, np.abs(phi).T @ np.abs(xd)
        r = np.abs(outn[s] - gold) / (tol * absum + 1e-30)
        Gd = G[s].double().numpy()
        gold_b, absum_b = m[:, None] * (phi @ Gd), m[:, None] * (np.abs(phi) @ np.abs(Gd))
        r0, V = mb.row_begin[s], x.shape[0]
        r_b = np.abs(grad[r0:r0 + V] - gold_b) / (tol * absum_b + 1e-30)
        worst = max(worst, r.max(), r_b.max())
        assert r.max() <= 1.0, (s, V, r.max())
        assert r_b.max() <= 1.0, (s, V, r_b.max())
        assert (grad[r0 + V:mb.row_begin[s + 1]] == 0).all(), s
    print("{} C={} n={} S={}: worst err/bound {:.3e}".format(engine, Cc, n, S, worst))


@gpu
@pytest.mark.parametrize("engine", ["tc3x", "tc1x"])
def test_projection_refuses_a_width_without_a_tensor_core_route(cuda, engine):
    """C = 200 (not a multiple of 16) has no tensor-core to_basis; a mesh batch has no SIMT route, so the call is refused
    before any launch instead of falling back."""
    items, pb = _proj_batch(5, 30)
    feat = torch.randn(pb.mesh_batch.V, 200, device="cuda")
    dn.set_engine(engine)
    try:
        torch.cuda.synchronize()
        l0 = _launches()
        with pytest.raises(RuntimeError, match="unsupported"):
            dn.fmaps.project_batched(feat, pb)
        assert _launches() == l0
    finally:
        dn.set_engine("tc3x")


# =====================================================================================================================
# 3. pointwise maps across chunks and every NP
# =====================================================================================================================
def _pm_items(shapes, seed0, dups=()):
    items = []
    for i, (a, b) in enumerate(shapes):
        mass, _, evals, evecs, gX, gY = dn.synthetic.structural_operators(a, b, 128, seed=seed0 + i, device="cuda")
        items.append({"mass": mass, "evals": evals, "evecs": evecs, "gradX": gX, "gradY": gY})
    for s, lo, hi in dups:                     # duplicate rows: ties in a target must go to the lower index
        items[s]["evecs"][hi] = items[s]["evecs"][lo]
    return items


PM_DUPS = [(2, 7, 2000), (2, 300, 2999), (0, 3, 150), (5, 10, 1200)]


def _run_pointwise(items, pairs, n, seed, sample=None, dups=()):
    pb = dn.PairBatch(items, pairs, n_fmap=n)
    n_rows = [it["mass"].shape[0] for it in items]
    chunks, _ = _pm_plan_model(n, pairs, n_rows)
    g = torch.Generator().manual_seed(seed)
    Cm = (torch.randn(len(pairs), n, n, generator=g) / n ** 0.5).cuda()
    maps = dn.pointwise_map_batch(Cm, pb, n_fmap=n)
    torch.cuda.synchronize()
    l0 = _launches()
    again = dn.pointwise_map_batch(Cm, pb, n_fmap=n)
    torch.cuda.synchronize()
    assert _launches() - l0 == sum(2 + (s > 1) for _, s in chunks), (len(chunks), _launches() - l0)
    assert torch.equal(torch.cat(maps), torch.cat(again))
    hi = {(s, h) for s, _, h in dups}
    fracs = []
    for p, (a, b) in enumerate(pairs):
        ex, ey = items[a]["evecs"], items[b]["evecs"]
        ref = dn.pointwise_map(Cm[p], ex, ey, n_fmap=n)
        assert maps[p].dtype == torch.int64 and torch.equal(maps[p], ref), p
        for s, h in hi:
            if s == a:
                assert not bool((maps[p] == h).any()), (p, h)
        target = dn.fmaps._apply_basis_exact(Cm[p].t().contiguous(), ex[:, :n].contiguous())
        source = ey[:, :n].contiguous()
        rows = None
        if sample is not None and source.shape[0] > sample:
            rows = torch.randperm(source.shape[0], generator=torch.Generator().manual_seed(p))[:sample].cuda()
        # the fp64 brute force in row chunks of about 2^25 distances (the default 64 rows is slow on 80k-row targets)
        fracs.append(_check_nn(maps[p], source, target, rows, n, chunk=max(1, (1 << 25) // target.shape[0])))
    return chunks, fracs


@gpu
@pytest.mark.parametrize("n", [3, 5, 12, 30, 50, 128])
def test_pointwise_map_batch_150_pairs_three_chunks(cuda, n):
    """150 pairs (chunks of 64, 64 and 22), every NP: bitwise the per-pair map and fp64-checked; duplicated target rows
    (far apart, so in different target ranges; their shape a target in every chunk) never map to the higher copy."""
    items = _pm_items(PM_SHAPES, 50, PM_DUPS)
    pairs = _pm_pairs()
    chunks, fracs = _run_pointwise(items, pairs, n, seed=n, dups=PM_DUPS)
    assert [len(m) for m, _ in chunks] == [64, 64, 22]
    print("n = {}: chunk splits {}, certain rows {:.4f}".format(n, [s for _, s in chunks], min(fracs)))
    assert min(fracs) > 0.9


@gpu
def test_pointwise_map_batch_128_pairs_fill_exactly_two_chunks(cuda):
    """128 pairs are exactly two full chunks: the launch count (2 or 3 per chunk) sees a chunk-size change that the
    150-pair batch, three chunks either way, would not."""
    items = _pm_items(PM_SHAPES, 50, PM_DUPS)
    chunks, fracs = _run_pointwise(items, _pm_pairs()[:128], 30, seed=128, dups=PM_DUPS)
    assert [len(m) for m, _ in chunks] == [64, 64]
    assert min(fracs) > 0.9


@gpu
def test_pointwise_map_batch_chunks_break_on_the_float_limit(cuda):
    """n = 128: two ~80k-row targets cannot share a chunk (2 x 80k x 128 floats > 16 Mi); one 200k-row target is a
    chunk of its own above the limit."""
    for name, shapes, pairs in (("80k targets", BIG_SHAPES, BIG_PAIRS), ("200k target", HUGE_SHAPES, HUGE_PAIRS)):
        items = _pm_items(shapes, 80)
        chunks, fracs = _run_pointwise(items, pairs, 128, seed=1, sample=2000)
        assert [len(m) for m, _ in chunks] == PM_CHUNKS_128[name]
        print("chunks {}, certain rows {:.4f}".format([(len(m), s) for m, s in chunks], min(fracs)))
        assert min(fracs) > 0.9
        del items
        torch.cuda.empty_cache()


@gpu
@pytest.mark.parametrize("n", [5, 12, 50])
def test_nearest_neighbor_every_np(cuda, n):
    """dn_nearest_neighbor at NP = 8, 16, 64 (test_gpu_fmaps.py covers NP = 4, 32, 128): fp64 check of a full 5k x 5k
    search, and duplicated target rows far apart take the lowest index."""
    g = torch.Generator().manual_seed(500 + n)
    src, tgt = torch.randn(5000, n, generator=g).cuda(), torch.randn(5000, n, generator=g).cuda()
    idx = dn.fmaps.nearest_neighbor(src, tgt)
    assert idx.dtype == torch.int64 and idx.shape == (5000,)
    assert _check_nn(idx, src, tgt, None, n) > 0.99
    Vt = 20000
    tgt = torch.randn(Vt, n, generator=g)
    for lo, hi in ((5, Vt - 5), (7, 11), (300, 12000)):
        tgt[hi] = tgt[lo]
    for Vs in (50, 5000):
        src = torch.randn(Vs, n, generator=g)
        src[0], src[1], src[2] = tgt[Vt - 5], tgt[11], tgt[12000]
        idx = dn.fmaps.nearest_neighbor(src.cuda(), tgt.cuda())
        assert idx[:3].tolist() == [5, 7, 300]
        assert _check_nn(idx, src.cuda(), tgt.cuda(), None, n) > 0.9


# =====================================================================================================================
# 4. the batched solve at the pair cap
# =====================================================================================================================
@gpu
def test_solve_batched_at_65535_pairs(cuda):
    """P = 65535 pairs of 256 shapes at n = 8, d = 16; shape 0 is in thousands of pairs.  C bitwise the per-pair solve
    on a sample (the first and last pair included) and fp64 per row; the gradients of shapes 0, 1, 2 against fp64 with
    the (tol + m u) bound, m the shape's role count."""
    n, d, S, P = 8, 16, 256, dn.fmaps.MAX_PAIRS
    F, ev = _stack_inputs(S, n, d, seed=65535)
    rs = np.random.RandomState(1)
    px, py = rs.randint(S, size=P), rs.randint(S, size=P)
    px[::13] = 0
    py[5::17] = 0
    px[7], py[7] = 1, 1                                      # a self-pair
    pairs = list(zip(px.tolist(), py.tolist()))
    Ft, evt = torch.from_numpy(F).cuda().requires_grad_(True), torch.from_numpy(ev).cuda()
    pl = dn.fmaps.PairList(pairs, S, "cuda")
    Cb = dn.fmaps.fmap_solve_batched(Ft, evt, pl, n, LAMBDA)
    g = torch.from_numpy(rs.randn(P, n, n).astype(np.float32)).cuda()
    (Cb * g).sum().backward()
    Cb = Cb.detach()
    grad = Ft.grad.cpu().numpy()
    Cn, gn = Cb.cpu().numpy(), g.cpu().numpy()
    fp64_term = 16 * n * (n + d) * EPS64
    sample = sorted(set([0, 7, P - 1] + rs.randint(P, size=200).tolist()))
    for p in sample:
        a, b = pairs[p]
        Cp = dn.fmaps.FmapSolveFn.apply(Ft.detach()[a], Ft.detach()[b], evt[a], evt[b], LAMBDA)
        assert torch.equal(Cp, Cb[p]), p
        gold = OF.solve(F[a], F[b], ev[a], ev[b], LAMBDA)
        kap = _kappa(F[a], ev[a], ev[b], LAMBDA)
        for i in range(n):
            assert np.abs(Cn[p][i].astype(np.float64) - gold[i]).max() <= (U32 + fp64_term * kap[i]) * np.abs(gold[i]).max()
    check = (0, 1, 2)
    gold_acc = {s: np.zeros((n, d)) for s in check}
    mag = {s: 0.0 for s in check}
    terms = {s: 0 for s in check}
    kmax = {s: 0.0 for s in check}
    for p, (a, b) in enumerate(pairs):
        if a not in check and b not in check:
            continue
        dA, dB = OF.solve_adjoint(F[a], F[b], ev[a], ev[b], LAMBDA, gn[p])
        kap = _kappa(F[a], ev[a], ev[b], LAMBDA).max()
        for s, dS in ((a, dA), (b, dB)):
            if s in check:
                gold_acc[s] += dS
                mag[s] += np.abs(dS).max()
                terms[s] += 1
                kmax[s] = max(kmax[s], kap)
    assert terms[0] > 5000 and terms[1] == pl.role_begin[2] - pl.role_begin[1]
    for s in check:
        tol = 4 * U32 + fp64_term * kmax[s]
        err = np.abs(grad[s] - gold_acc[s]).max()
        print("shape {}: {} roles, err / sum max|g_p| = {:.2e}, bound {:.2e}".format(s, terms[s], err / mag[s],
                                                                                    tol + terms[s] * U32))
        assert err <= (tol + terms[s] * U32) * mag[s], (s, err / mag[s])
    # one pair over the cap: refused by the pair list and by the C-ABI before any launch
    with pytest.raises(ValueError, match="at most 65535 pairs"):
        dn.fmaps.PairList(pairs + [(0, 0)], S, "cuda")
    torch.cuda.synchronize()
    l0 = _launches()
    rc = dn._lib.load().dn_fmap_solve_fwd_batched(Ft.data_ptr(), n * d, evt.data_ptr(), n, S, pl.pair_x.data_ptr(),
                                                  pl.pair_y.data_ptr(), P + 1, n, d, LAMBDA, Cb.data_ptr(),
                                                  dn.ops._stream())
    assert rc != 0 and "unsupported" in dn._lib.load().dn_error_string(rc).decode().lower()
    assert _launches() == l0


# =====================================================================================================================
# 5. operators of ~150 small meshes
# =====================================================================================================================
def _ops_meshes():
    S = dn.synthetic
    rs = np.random.RandomState(5)
    out = []
    for i in range(150):
        kind = i % 3
        if kind == 0:
            a, b = (int(v) for v in rs.randint(10, 25, size=2))
            out.append(S.torus_mesh(a, b, seed=i))
        elif kind == 1:
            a, b = (int(v) for v in rs.randint(10, 25, size=2))
            out.append(S.patch_mesh(a, b, seed=i))
        else:
            out.append(S.icosphere_mesh(2, seed=i))               # V = 162
    return out


@gpu
def test_compute_operators_batch_150_meshes_against_oracle(cuda, monkeypatch):
    """k = 16 over 150 tori, patches and icospheres of 100-625 vertices: every mesh against the fp64 oracle with
    _check_against's bounds, and the same list twice bitwise equal.  The iteration at which each mesh leaves the active
    set is recorded: the mask must shrink over several iterations."""
    k = 16
    meshes = _ops_meshes()
    assert all(100 <= v.shape[0] <= 625 for v, _ in meshes)
    masks = []
    orig = dn.eigen._BatchSolver.set_active

    def spy(self, flags):
        masks.append([bool(f) for f in flags])
        return orig(self, flags)

    monkeypatch.setattr(dn.eigen._BatchSolver, "set_active", spy)
    st = {}
    vl, fl = [v for v, _ in meshes], [f for _, f in meshes]
    first = dn.geometry.compute_operators_batch(vl, fl, k, device=cuda, stats=st)
    n_masks = len(masks)
    second = dn.geometry.compute_operators_batch(vl, fl, k, device=cuda)
    assert len(masks) == 2 * n_masks and masks[:n_masks] == masks[n_masks:]
    assert st["groups"] == 1 and st["eig"][0]["n_stacked"] == len(meshes)
    for a, b in zip(first, second):
        for x, y in zip(a, b):
            if x.is_sparse:
                assert torch.equal(x.indices(), y.indices()) and torch.equal(x.values(), y.values())
            else:
                assert torch.equal(x, y)
    # last iteration each mesh was still filtered (the outer iterations are 1-based; 0: converged before any filter)
    left = [max([i + 1 for i, m in enumerate(masks[:n_masks]) if m[b]], default=0) for b in range(len(meshes))]
    print("iterations: {}; meshes leaving the active set per iteration: {}".format(
        n_masks, np.bincount(left).tolist()))
    assert len(set(left)) > 2
    for b, ((v, f), out) in enumerate(zip(meshes, first)):
        g = OO.compute_operators(v.numpy(), f.numpy(), k + 1)
        gold = (g[0].astype(np.float64), g[1], g[2], g[3][:k], g[4][:, :k], g[5], g[6])
        _check_against(out, gold, k, g[3])
