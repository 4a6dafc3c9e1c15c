"""Every backward kernel against fp64 autograd on the CPU, at the shapes where its dispatch changes.

Gold: ``oracle/dn_oracle_torch.block_forward`` for blocks and nets (pinned to the live reference by test_oracle.py);
plain torch float64 expressions of the same operations for the single autograd Functions.  The loss is sum(out * R)
with a seeded R, the metric max|ours - gold| / max|gold| (``O.rel_err``).

Cases (V = n x m, K eigenpairs, C channels) and the route each one reaches:

  tiny   5 x 10,  K 40,  C 16   V below one 128-row tile; tensor-core to_basis with <= 4 partials -> serial spectral_bwd
  k12   23 x 31,  K 12,  C 48   K % 8 = 4: to_basis on tensor cores, from_basis and its dX on SIMT; generic gather G = 8
  k160  40 x 50,  K 160, C 96   K > 128: to_basis on SIMT, from_basis on tensor cores; generic gather G = 16
  c40   30 x 41,  K 64,  C 40   C off the 16 grid: every dense layer and weight gradient on SIMT under tc3x
  c256  60 x 83,  K 128, C 256  two-slice to_basis, P / Q split, 256-wide layers, SIMT weight gradients, gather NH = 2
  full 400 x 500, K 128, C 128  200k-row weight / bias / time-gradient reductions, ~132 split-V partials

``test_dispatch_routes_under_strict_tc`` runs the same cases in a DN_STRICT_TC=1 subprocess so that none of them drifts
to the other side of the dispatch it is named after.

Bounds.  simt and tc3x: 1e-5 on outputs, 2e-5 on input gradients, 5e-5 on parameter gradients (the suite's fp32
bounds).  tc1x rounds every tensor-core operand to TF32 (unit roundoff u = 2^-11) and bf16 to bf16 (u = 2^-8).  A
product of two rounded operands is off by up to 2u.  A block's deepest gradient, that of A_re / A_im, sits behind
eight rounded contractions in series: to_basis, from_basis and the [P|Q] layer in the forward, three MiniMLP dX layers
and the weight-gradient contraction in the backward.  So both engines state 16u for outputs and gradients alike:
TC1X_TOL = 7.8e-3, BF16_GRAD_TOL = 6.25e-2 (bf16 outputs keep the suite's BF16_TOL = 2e-2).

ReLU kinks: the gradient of ReLU is discontinuous at 0.  Our activation pattern (read from the MLPFn node's saved
hidden tensors) may differ from the fp64 one only where the fp64 pre-activation lies within the engine's rounding of
zero, and the gradients are compared under our pattern (``_check_kinks``)."""
import json
import os
import subprocess
import sys

import pytest
import torch

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle as O  # noqa: E402  (checker only)
import dn_oracle_torch as T  # noqa: E402  (checker only)

pytestmark = pytest.mark.gpu

D = torch.float64
FP32_TOL = (1e-5, 2e-5, 5e-5)                 # (output, input gradient, parameter gradient)
TC1X_TOL = 16 * 2.0 ** -11
BF16_GRAD_TOL = 16 * 2.0 ** -8
TOL = {"simt": FP32_TOL, "tc3x": FP32_TOL, "tc1x": (TC1X_TOL,) * 3,
       "bf16": (2e-2, BF16_GRAD_TOL, BF16_GRAD_TOL)}  # bf16 outputs: the suite's BF16_TOL (test_gpu_parity.py)
ENGINES = ["simt", "tc3x"]
# a flip of the ReLU pattern is allowed where |fp64 pre-activation| < KINK * max|pre-activation|: 1e-5 for the fp32
# engines (the config-2 test's allowance), scaled by the engine's parameter-gradient bound for the others
KINK = {e: 1e-5 * TOL[e][2] / FP32_TOL[2] for e in TOL}
# the fp32 floor: where a bound is missed by a formula's own fp32 rounding, an fp32 torch evaluation of the same sums
# misses it too; a check given a floor is held to max(bound, FLOOR_FACTOR[engine] * that evaluation's error).  tc3x
# drops the low x low product of its split operands, so each of its products is off by up to 2^-22, four times fp32's
# unit roundoff
FLOOR_FACTOR = {"simt": 2.0, "tc3x": 8.0}

CASES = {"tiny": (5, 10, 40, 16), "k12": (23, 31, 12, 48), "k160": (40, 50, 160, 96), "c40": (30, 41, 64, 40),
         "c256": (60, 83, 128, 256), "full": (400, 500, 128, 128)}
T_UNDERFLOW = 100.0     # exp(-lambda_k t) is 0 in fp32 for every k >= 1 (lambda_1 = 200 / K >= 1.25 here)


@pytest.fixture(scope="module")
def dn():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import diffusion_net_b200 as d
    d._lib.load()
    yield d
    d.set_engine("tc3x")


class Checker:
    """Collects every comparison of a test, prints it, and fails at the end with all the misses listed."""

    def __init__(self, label):
        self.label, self.misses = label, []
        self.floor_factor = FLOOR_FACTOR.get(label.rsplit("/", 1)[-1])

    def __call__(self, what, ours, gold, tol, floor=None):
        ours = ours.detach().cpu().double().numpy() if torch.is_tensor(ours) else ours
        gold = gold.detach().cpu().double().numpy() if torch.is_tensor(gold) else gold
        err = O.rel_err(ours, gold)
        bound = tol
        if floor is not None:
            f_err = O.rel_err(floor.detach().cpu().double().numpy(), gold)
            bound = max(tol, self.floor_factor * f_err)
            print("[measured] {} {} err={:.3e} fp32-floor={:.3e} bound={:.1e}".format(self.label, what, err, f_err,
                                                                                    bound))
        else:
            print("[measured] {} {} err={:.3e} bound={:.1e}".format(self.label, what, err, bound))
        if not err < bound:
            self.misses.append("{}: {:.3e} >= {:.1e}".format(what, err, bound))

    def done(self):
        assert not self.misses, "{}: {}".format(self.label, "; ".join(self.misses))


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _case_ops(dn, case, seed=0, **kw):
    n, m, K, C = CASES[case]
    return dn.synthetic.structural_operators(n, m, K, seed=seed, device="cuda", **kw)


def _mlp_node(out, weight0):
    """The MLPFn autograd node whose first weight is ``weight0``: (hidden activations, dropout masks) it saved."""
    seen, stack = {}, [out.grad_fn]
    while stack:
        f = stack.pop()
        if f is None or id(f) in seen:
            continue
        seen[id(f)] = f                 # keeps the node alive: a freed wrapper's id may be reused
        if "MLPFn" in type(f).__name__:
            n_src, n_layers = f.meta[0], f.meta[1]
            sv = f.saved_tensors
            if sv[n_src].data_ptr() == weight0.data_ptr():
                h0 = n_src + n_layers
                return list(sv[h0:h0 + f.n_hidden]), list(sv[h0 + f.n_hidden:])
        stack.extend(nf for nf, _ in f.next_functions)
    raise AssertionError("no MLPFn node with this first weight")


def _check_kinks(masks, pre, engine, keep=None):
    """Our ReLU pattern may differ from fp64's only within the engine's rounding of zero.  ``keep``: where a dropout
    mask keeps the element (a dropped element has no pattern)."""
    for i, (mk, pa) in enumerate(zip(masks, pre)):
        pa = pa.reshape(mk.shape)
        flips = mk != (pa > 0)
        if keep is not None:
            flips &= keep[i]
        cap = 8 * max(1, -(-mk.numel() // 1_000_000)) * TOL[engine][2] / FP32_TOL[2]
        assert int(flips.sum()) <= cap, (i, int(flips.sum()))
        worst = float(pa[flips].abs().max()) if flips.any() else 0.0
        assert worst < KINK[engine] * float(pa.abs().max()), (i, worst)


# ---- a. single autograd Functions ------------------------------------------------------------------------------
def _diffusion_gold(x, t, mass, evals, evecs):
    spec = evecs.t() @ (x * mass.unsqueeze(-1))
    return evecs @ (torch.exp(-evals.unsqueeze(-1) * t.unsqueeze(0)) * spec)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case", list(CASES))
def test_diffusion_fn(dn, engine, case):
    """grad_x and grad_time of DiffusionFn; the time vector includes -0.1, 0 and 1e-9 (clamped to 1e-8 in place, the
    gradient taken at the clamped value as the reference's clamp of ``.data`` does) and one t where every exp(-lambda
    t) but the first underflows."""
    dn.set_engine(engine)
    chk = Checker("diffusion/{}/{}".format(case, engine))
    mass, L, evals, evecs, gX, gY = _case_ops(dn, case, seed=1)
    V, C = mass.shape[0], CASES[case][3]
    g = _gen(11)
    x, R = torch.randn(V, C, generator=g), torch.randn(V, C, generator=g)
    t0 = torch.rand(C, generator=g) * 0.3
    t0[:4] = torch.tensor([-0.1, 0.0, 1e-9, T_UNDERFLOW])
    xg = x.cuda().requires_grad_(True)
    t = t0.cuda().requires_grad_(True)
    out = dn.ops.DiffusionFn.apply(xg, t, mass, evals, evecs)
    (out * R.cuda()).sum().backward()
    assert torch.equal(t.detach().cpu(), t0.clamp(min=1e-8))
    x64 = x.to(D).requires_grad_(True)
    t64 = t0.to(D).clamp(min=1e-8).requires_grad_(True)
    gold = _diffusion_gold(x64, t64, mass.cpu().to(D), evals.cpu().to(D), evecs.cpu().to(D))
    (gold * R.to(D)).sum().backward()
    tol = TOL[engine]
    chk("out", out, gold, tol[0])
    chk("grad_x", xg.grad, x64.grad, tol[1])
    chk("grad_time", t.grad, t64.grad, tol[2])
    chk.done()


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case", list(CASES))
def test_to_from_basis_fn(dn, engine, case):
    dn.set_engine(engine)
    chk = Checker("basis/{}/{}".format(case, engine))
    mass, L, evals, evecs, gX, gY = _case_ops(dn, case, seed=2)
    V, K, C = mass.shape[0], evecs.shape[1], CASES[case][3]
    g = _gen(12)
    v, Rk = torch.randn(V, C, generator=g), torch.randn(K, C, generator=g)
    s, Rv = torch.randn(K, C, generator=g), torch.randn(V, C, generator=g)
    vg, sg = v.cuda().requires_grad_(True), s.cuda().requires_grad_(True)
    spec = dn.ops.to_basis(vg, evecs, mass)
    back = dn.ops.from_basis(sg, evecs)
    ((spec * Rk.cuda()).sum() + (back * Rv.cuda()).sum()).backward()
    E, M = evecs.cpu().to(D), mass.cpu().to(D)
    v64, s64 = v.to(D).requires_grad_(True), s.to(D).requires_grad_(True)
    spec64, back64 = T.to_basis(v64, E, M), T.from_basis(s64, E)
    ((spec64 * Rk.to(D)).sum() + (back64 * Rv.to(D)).sum()).backward()
    tol = TOL[engine]
    chk("to_basis", spec, spec64, tol[0])
    chk("from_basis", back, back64, tol[0])
    chk("to_basis grad", vg.grad, v64.grad, tol[1])
    chk("from_basis grad", sg.grad, s64.grad, tol[1])
    chk.done()


def _features_arg(xd, gX, gY, A_re, A_im):
    vx, vy = torch.sparse.mm(gX, xd), torch.sparse.mm(gY, xd)
    if A_im is None:
        b_re, b_im = vx @ A_re.t(), vy @ A_re.t()
    else:
        b_re = vx @ A_re.t() - vy @ A_im.t()
        b_im = vy @ A_re.t() + vx @ A_im.t()
    return vx * b_re + vy * b_im


def _features_gold(xd, gX, gY, A_re, A_im):
    return torch.tanh(_features_arg(xd, gX, gY, A_re, A_im))


def _run_features(dn, gops, gX, gY, C, rot, seed, chk, engine):
    """GradFeaturesFn forward + backward on ``gops`` against fp64; returns our gradients.  Held to the fp32 floor of
    the formula (DESIGN §2): an fp32 torch evaluation of the same sums misses 1e-5 on its own at C = 256 and V = 200k."""
    V = gX.shape[0]
    g = _gen(seed)
    xd, R = torch.randn(V, C, generator=g), torch.randn(V, C, generator=g)
    A_re = torch.randn(C, C, generator=g) / C ** 0.5
    A_im = torch.randn(C, C, generator=g) / C ** 0.5 if rot else None
    sx, sy = gX.coalesce().cpu(), gY.coalesce().cpu()
    # scale xd so that the tanh argument has unit rms, as in a block (x_diffuse is smooth): white noise through these
    # operators gives arguments of ~1e3 whose cancellations near tanh's zero are an fp32 floor of any evaluation
    arg = _features_arg(xd.to(D), sx.to(D), sy.to(D), A_re.to(D), None if A_im is None else A_im.to(D))
    xd =(xd.to(D) / float(arg.square().mean().sqrt()) ** 0.5).float()
    leaves = [t.cuda().requires_grad_(True) if t is not None else None for t in (xd, A_re, A_im)]
    out = dn.ops.GradFeaturesFn.apply(leaves[0], leaves[1], leaves[2], gops)
    (out * R.cuda()).sum().backward()

    def evaluate(dt):
        ls = [t.to(dt).requires_grad_(True) if t is not None else None for t in (xd, A_re, A_im)]
        res = _features_gold(ls[0], sx.to(dt), sy.to(dt), ls[1], ls[2])
        (res * R.to(dt)).sum().backward()
        return res, ls

    gold, l64 = evaluate(D)
    f32, l32 = evaluate(torch.float32)
    tol = TOL[engine]
    chk("features", out, gold, tol[0], f32)
    chk("grad_xd", leaves[0].grad, l64[0].grad, tol[1], l32[0].grad)
    chk("grad_A_re", leaves[1].grad, l64[1].grad, tol[2], l32[1].grad)
    if rot:
        chk("grad_A_im", leaves[2].grad, l64[2].grad, tol[2], l32[2].grad)
    return [t.grad.clone() for t in leaves if t is not None]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("rot", [True, False])
@pytest.mark.parametrize("case", list(CASES))
def test_gradient_features_fn(dn, engine, rot, case):
    dn.set_engine(engine)
    chk = Checker("features/{}/rot={}/{}".format(case, rot, engine))
    mass, L, evals, evecs, gX, gY = _case_ops(dn, case, seed=3)
    _run_features(dn, dn.ops.GradOperators(gX, gY), gX, gY, CASES[case][3], rot, 13, chk, engine)
    chk.done()


def _coo(rows, cols, vals, V):
    return torch.sparse_coo_tensor(torch.stack((rows, cols)), vals, (V, V)).coalesce()


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("C", [48, 128])
def test_gradient_features_union_pattern_empty_row_and_column(dn, engine, C):
    """gradX / gradY with different patterns; row 7 has no entry in either (an empty forward row) and column 11 is
    never referenced (an empty row of the transposed CSR)."""
    dn.set_engine(engine)
    chk = Checker("features/union/C={}/{}".format(C, engine))
    n, m = 23, 31
    V = n * m
    rows, cols = (torch.from_numpy(a) for a in dn.synthetic.torus_pattern(n, m))
    g = _gen(14)
    keep_x = (rows != 7) & (cols != 11)
    keep_y = keep_x & (torch.rand(rows.shape[0], generator=g) < 0.7)
    gX = _coo(rows[keep_x], cols[keep_x], torch.randn(int(keep_x.sum()), generator=g) * 3, V).cuda()
    gY = _coo(rows[keep_y], cols[keep_y], torch.randn(int(keep_y.sum()), generator=g) * 3, V).cuda()
    gops = dn.ops.GradOperators(gX, gY)
    rp = gops.csr_t[1].cpu()
    assert int(rp[12] - rp[11]) == 0 and int(gops.csr[1][8] - gops.csr[1][7]) == 0
    for rot in (True, False):
        _run_features(dn, gops, gX, gY, C, rot, 15, chk, engine)
    chk.done()


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("C", [128, 256])
def test_gradient_features_long_rows(dn, engine, C):
    """Rows 64..66 (one 64-row block of spmm_features_blk_kernel) and row 3001 carry ~300 entries each: the block
    stages more than GB_NNZ = 1024 entries and reads the rest from global memory; the backward walks long rows of the
    transposed CSR."""
    dn.set_engine(engine)
    chk = Checker("features/long_rows/C={}/{}".format(C, engine))
    n, m = 60, 83
    V = n * m
    rows, cols = (torch.from_numpy(a) for a in dn.synthetic.torus_pattern(n, m))
    g = _gen(16)
    extra_r = torch.tensor([64, 65, 66, 3001]).repeat_interleave(300)
    extra_c = torch.randint(0, V, (extra_r.shape[0],), generator=g)
    r, c = torch.cat((rows, extra_r)), torch.cat((cols, extra_c))
    gX = _coo(r, c, torch.randn(r.shape[0], generator=g) * 3, V).cuda()
    gY = _coo(r, c, torch.randn(r.shape[0], generator=g) * 3, V).cuda()
    gops = dn.ops.GradOperators(gX, gY)
    rp = gops.csr[1].cpu()
    assert int(rp[67] - rp[64]) > 800 and int(rp[128] - rp[64]) > 1024
    for rot in (True, False):
        _run_features(dn, gops, gX, gY, C, rot, 17, chk, engine)
    chk.done()


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("rot", [True, False])
def test_gradient_features_patched_permuted_mesh(dn, engine, rot):
    """A permuted mesh with ``dn_patches`` built: the forward takes the patched gather; its output and gradients are
    bitwise equal to the plain operators' and within the bounds of fp64."""
    dn.set_engine(engine)
    chk = Checker("features/patched/rot={}/{}".format(rot, engine))
    C = 128
    mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(60, 70, 32, seed=4, device="cuda", permute=True)
    plain = dn.ops.GradOperators(gX, gY)
    patched = dn.ops.GradOperators(gX, gY).build_patches()
    assert patched._patches
    g_plain = _run_features(dn, plain, gX, gY, C, rot, 18, chk, engine)
    g_patch = _run_features(dn, patched, gX, gY, C, rot, 18, chk, engine)
    for a, b in zip(g_plain, g_patch):
        assert torch.equal(a, b)
    chk.done()


# MiniMLP variants: (name, C, V, hidden widths, which bias slots are None, dropout, residual)
MLP_CASES = [
    ("chain_64_32", 128, 7056, [64, 32], (), False, True),      # a fused chain whose N varies
    ("hidden_256", 128, 7056, [256], (), False, True),          # 256-wide hidden layer: layer by layer, SIMT atb
    ("hidden_40", 48, 713, [40], (), False, True),              # hidden width off the 16 grid
    ("bias_none", 96, 2000, [96, 96], (1,), False, True),       # a None bias slot inside the chain
    ("dropout", 96, 2000, [96, 96], (), True, True),            # dropout masks in the dX epilogue
    ("no_residual", 128, 7056, [128, 128], (), False, False),
    ("full", 128, 200000, [128, 128], (), False, True),         # 200k-row weight / bias reductions
]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name,C,V,hidden,no_bias,dropout,res", MLP_CASES, ids=[c[0] for c in MLP_CASES])
def test_mini_mlp_fn(dn, engine, name, C, V, hidden, no_bias, dropout, res):
    dn.set_engine(engine)
    chk = Checker("mlp/{}/{}".format(name, engine))
    g = _gen(19)
    dims = [3 * C] + hidden + [C]
    srcs = [torch.randn(V, C, generator=g) for _ in range(3)]
    Ws = [(torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5 for i in range(len(dims) - 1)]
    bs = [None if i in no_bias else (torch.rand(dims[i + 1], generator=g) * 2 - 1) / dims[i] ** 0.5
          for i in range(len(dims) - 1)]
    resid = torch.randn(V, C, generator=g) if res else None
    R = torch.randn(V, C, generator=g)
    cu = lambda ts: [t.cuda().requires_grad_(True) if t is not None else None for t in ts]
    s_c, w_c, b_c = cu(srcs), cu(Ws), cu(bs)
    r_c = resid.cuda().requires_grad_(True) if res else None
    torch.manual_seed(1234)
    out = dn.ops.mlp_apply(s_c, w_c, b_c, residual=r_c, drop_p=0.5 if dropout else 0.0)
    hid, _ = _mlp_node(out, w_c[0])
    masks = [(h > 0).cpu() for h in hid]
    (out * R.cuda()).sum().backward()
    drops = None
    if dropout:   # replay the mask draws (same order / shapes as ops.MLPFn.forward)
        torch.manual_seed(1234)
        drops = [torch.empty(V, dims[l + 1], device="cuda").bernoulli_(0.5).mul_(2.0).cpu()
                 for l in range(len(dims) - 2)]
    l64 = lambda ts: [t.to(D).requires_grad_(True) if t is not None else None for t in ts]
    s6, w6, b6 = l64(srcs), l64(Ws), l64(bs)
    r6 = resid.to(D).requires_grad_(True) if res else None
    h, pre = torch.cat(s6, -1), []
    for i in range(len(w6)):
        h = h @ w6[i].t() + (b6[i] if b6[i] is not None else 0.0)
        if i + 1 < len(w6):
            pre.append(h.detach())
            h = h * masks[i].to(D) * (drops[i].to(D) if dropout else 1.0)
    if res:
        h = h + r6
    (h * R.to(D)).sum().backward()
    _check_kinks(masks, pre, engine, keep=[d != 0 for d in drops] if dropout else None)
    tol = TOL[engine]
    chk("out", out, h, tol[0])
    for i, (a, b) in enumerate(zip(s_c, s6)):
        chk("grad_src%d" % i, a.grad, b.grad, tol[1])
    for i in range(len(w6)):
        chk("grad_W%d" % i, w_c[i].grad, w6[i].grad, tol[2])
        if b6[i] is not None:
            chk("grad_b%d" % i, b_c[i].grad, b6[i].grad, tol[2])
        else:
            assert b_c[i] is None
    if res:
        chk("grad_residual", r_c.grad, r6.grad, tol[1])
    chk.done()


def test_mini_mlp_single_layer_without_bias(dn):
    """The standalone SpatialGradientFeatures route: one layer, one source, bias None."""
    for engine in ENGINES:
        dn.set_engine(engine)
        chk = Checker("mlp/single_no_bias/{}".format(engine))
        g = _gen(20)
        V, C = 3000, 96
        x, W, R = torch.randn(V, C, generator=g), torch.randn(C, C, generator=g) / C ** 0.5, torch.randn(V, C, generator=g)
        xc, Wc = x.cuda().requires_grad_(True), W.cuda().requires_grad_(True)
        out = dn.ops.mlp_apply([xc], [Wc], [None])
        (out * R.cuda()).sum().backward()
        x6, W6 = x.to(D).requires_grad_(True), W.to(D).requires_grad_(True)
        ((x6 @ W6.t()) * R.to(D)).sum().backward()
        chk("out", out, x6 @ W6.t(), TOL[engine][0])
        chk("grad_x", xc.grad, x6.grad, TOL[engine][1])
        chk("grad_W", Wc.grad, W6.grad, TOL[engine][2])
        chk.done()


# ---- b. blocks and nets ----------------------------------------------------------------------------------------
BLOCK_CASES = {   # name: (n, m, K, C, block keyword arguments)
    "c256": (60, 83, 128, 256, {}),
    "k160": (40, 50, 160, 96, {}),
    "k12": (23, 31, 12, 48, {}),
    "norot": (84, 84, 128, 128, {"with_gradient_rotations": False}),
    "nograd": (84, 84, 128, 128, {"with_gradient_features": False}),
    "tiny": (5, 10, 40, 16, {}),
    "full": (400, 500, 128, 128, {}),
    "config2": (84, 84, 128, 128, {}),
    # C % 4 != 0: the scalar-lane feature gather and its two backward kernels
    "c1": (20, 25, 64, 1, {}), "c3": (20, 25, 64, 3, {}), "c6": (20, 25, 64, 6, {}), "c30": (20, 25, 64, 30, {}),
    # a MiniMLP deeper than one fused chain (8 layers): layer by layer, forward and backward
    "mlp9": (20, 25, 64, 64, {"mlp_hidden_dims": [64] * 8}), "mlp12": (20, 25, 64, 64, {"mlp_hidden_dims": [64] * 11}),
}


def _block_run(dn, engine, name, chk, floor=False):
    n, m, K, C, kw = BLOCK_CASES[name]
    kw = dict(kw)
    hid = kw.pop("mlp_hidden_dims", [C, C])
    V = n * m
    mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=5, device="cuda")
    params = dn.synthetic.block_weights(C, seed=5, mlp_hidden_dims=hid, **kw)
    g = _gen(21)
    x, R = torch.randn(V, C, generator=g), torch.randn(V, C, generator=g)
    blk = dn.DiffusionNetBlock(C_width=C, mlp_hidden_dims=hid, dropout=False, **kw)
    blk.load_state_dict(params, strict=True)
    blk = blk.cuda().train()
    xg = x.cuda().unsqueeze(0).requires_grad_(True)
    u = lambda t: t.unsqueeze(0)
    out = blk(xg, u(mass), None, u(evals), u(evecs), [gX], [gY])
    hid, _ = _mlp_node(out, blk.mlp.linears()[0].weight)
    masks = [(h > 0).cpu() for h in hid]
    (out[0] * R.cuda()).sum().backward()
    ops64 = (mass.cpu().to(D).unsqueeze(0), evals.cpu().to(D).unsqueeze(0), evecs.cpu().to(D).unsqueeze(0),
             [gX.cpu().to(D)], [gY.cpu().to(D)])

    def evaluate(dt):
        prm = {k: v.to(dt).requires_grad_(True) for k, v in params.items()}
        xx = x.to(dt).unsqueeze(0).requires_grad_(True)
        pre = []
        ops_dt = [o.to(dt) if torch.is_tensor(o) else [s.to(dt) for s in o] for o in ops64]
        res = T.block_forward(xx, *ops_dt, prm, with_gradient_features=kw.get("with_gradient_features", True),
                              relu_masks=masks, pre_acts=pre)
        (res[0] * R.to(dt)).sum().backward()
        return res, xx, prm, pre

    gold, x64, prm, pre = evaluate(D)
    _check_kinks(masks, pre, engine)
    f32 = evaluate(torch.float32) if floor else None
    tol = TOL[engine]
    chk("out", out[0], gold[0], tol[0], f32[0][0] if floor else None)
    chk("grad_x", xg.grad[0], x64.grad[0], tol[1], f32[1].grad[0] if floor else None)
    for pname, p_ in blk.named_parameters():
        assert p_.grad is not None, pname
        if C == 1 and pname.endswith("A_im.weight"):
            # one channel: g0 b_re + g1 b_im = A_re (g0^2 + g1^2), A_im cancels and its gradient is 0 in exact arithmetic;
            # ours is rounding, held to the bound relative to A_re's gradient
            scale = prm[pname.replace("A_im", "A_re")].grad.abs().max().item()
            err = (p_.grad.detach().cpu().double() - prm[pname].grad).abs().max().item() / scale
            print("[measured] {} grad {} err={:.3e} (of max|grad A_re|)".format(chk.label, pname, err))
            if not err < tol[2]:
                chk.misses.append("grad {}: {:.3e} >= {:.1e}".format(pname, err, tol[2]))
            continue
        chk("grad " + pname, p_.grad, prm[pname].grad, tol[2], f32[2][pname].grad if floor else None)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", [n for n in BLOCK_CASES if n != "config2"])
def test_block_backward_vs_fp64(dn, engine, name):
    """DiffusionNetBlock in train mode (dropout off), forward and backward, against fp64 autograd of the torch oracle:
    x_in and every parameter gradient.  (config 2's shape under simt / tc3x is test_gpu_parity's own test.)"""
    dn.set_engine(engine)
    chk = Checker("block/{}/{}".format(name, engine))
    _block_run(dn, engine, name, chk, floor=name == "full")
    chk.done()


@pytest.mark.parametrize("engine", ["tc1x", "bf16"])
@pytest.mark.parametrize("name", ["config2", "c256"])
def test_block_backward_low_precision_engines(dn, engine, name):
    """tc1x and bf16 gradients against fp64 under their stated bounds (TC1X_TOL, BF16_GRAD_TOL)."""
    dn.set_engine(engine)
    chk = Checker("block/{}/{}".format(name, engine))
    try:
        _block_run(dn, engine, name, chk)
    finally:
        dn.set_engine("tc3x")
    chk.done()


@pytest.mark.parametrize("engine", ENGINES)
def test_net_on_computed_operators_vs_fp64(dn, engine):
    """A 2-block DiffusionNet (C_in = 3, xyz in) on a torus whose operators come from geometry.compute_operators (the
    real data path: its transposed CSR is built by dn_csr_transpose), against the fp64 composition of the oracle."""
    dn.set_engine(engine)
    chk = Checker("net/computed_ops/{}".format(engine))
    C, K, C_out, NB = 64, 64, 5, 2
    verts, faces = dn.synthetic.torus_mesh(30, 40, seed=6)
    frames, mass, L, evals, evecs, gX, gY = dn.geometry.compute_operators(verts, faces, K, device="cuda")
    V = verts.shape[0]
    torch.manual_seed(6)
    net = dn.DiffusionNet(C_in=3, C_out=C_out, C_width=C, N_block=NB, dropout=False).cuda().train()
    with torch.no_grad():
        for n_, p_ in net.named_parameters():
            if n_.endswith("diffusion_time"):
                p_.uniform_(1e-3, 0.3)
    R = torch.randn(V, C_out, generator=_gen(22))
    x = verts.cuda().requires_grad_(True)
    out = net(x, mass, L=L, evals=evals, evecs=evecs, gradX=gX, gradY=gY)
    masks = {b: [(h > 0).cpu() for h in _mlp_node(out, net.blocks[b].mlp.linears()[0].weight)[0]] for b in range(NB)}
    (out * R.cuda()).sum().backward()
    prm = {k: v.detach().cpu().to(D).requires_grad_(True) for k, v in net.state_dict().items()}
    x64 = verts.to(D).requires_grad_(True)
    m64, e64, v64 = (t.cpu().to(D).unsqueeze(0) for t in (mass, evals, evecs))
    h = torch.addmm(prm["first_lin.bias"], x64, prm["first_lin.weight"].t()).unsqueeze(0)
    for b in range(NB):
        bp = {k[len("block_%d." % b):]: v for k, v in prm.items() if k.startswith("block_%d." % b)}
        pre = []
        h = T.block_forward(h, m64, e64, v64, [gX.cpu().to(D)], [gY.cpu().to(D)], bp, relu_masks=masks[b],
                            pre_acts=pre)
        _check_kinks(masks[b], pre, engine)
    gold = torch.addmm(prm["last_lin.bias"], h[0], prm["last_lin.weight"].t())
    (gold * R.to(D)).sum().backward()
    tol = TOL[engine]
    chk("out", out, gold, tol[0])
    chk("grad_x", x.grad, x64.grad, tol[1])
    for name, p_ in net.named_parameters():
        chk("grad " + name, p_.grad, prm[name].grad, tol[2])
    chk.done()


# ---- c. every case reaches the route it is named after -----------------------------------------------------------
# True: stays on tensor cores under tc3x; False: meant to reach a SIMT fallback ("unsupported" under DN_STRICT_TC=1)
ROUTES = {
    "tiny/block": True, "full/block": True, "config2/block": True, "norot/block": True, "nograd/block": True,
    "k12/to_basis": True, "k12/from_basis": False, "k12/block": False,
    "k160/to_basis": False, "k160/from_basis": True, "k160/block": False,
    "c40/block": False,
    "c256/to_basis": True, "c256/block": False,
    "mlp/chain_64_32": True, "mlp/hidden_256": False, "mlp/hidden_40": False, "mlp/bias_none": True,
    "mlp/dropout": True, "mlp/no_residual": True,
}


def _route_report():
    """Run in a DN_STRICT_TC=1 subprocess: each route's forward + backward under tc3x; prints one JSON line."""
    import diffusion_net_b200 as dn
    dn.set_engine("tc3x")
    res = {}
    for key in ROUTES:
        case, what = key.split("/")
        try:
            if case == "mlp":
                _, C, V, hidden, no_bias, dropout, res_ = next(c for c in MLP_CASES if c[0] == what)
                dims = [3 * C] + hidden + [C]
                srcs = [torch.randn(V, C, device="cuda", requires_grad=True) for _ in range(3)]
                Ws = [torch.randn(dims[i + 1], dims[i], device="cuda", requires_grad=True) for i in range(len(dims) - 1)]
                bs = [None if i in no_bias else torch.zeros(dims[i + 1], device="cuda", requires_grad=True)
                      for i in range(len(dims) - 1)]
                out = dn.ops.mlp_apply(srcs, Ws, bs, residual=srcs[0] if res_ else None, drop_p=0.5 if dropout else 0)
            elif what == "block":
                n, m, K, C, kw = BLOCK_CASES[case] if case in BLOCK_CASES else CASES[case] + ({},)
                mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, device="cuda")
                blk = dn.DiffusionNetBlock(C_width=C, mlp_hidden_dims=[C, C], dropout=False, **kw).cuda().train()
                x = torch.randn(1, n * m, C, device="cuda", requires_grad=True)
                u = lambda t: t.unsqueeze(0)
                out = blk(x, u(mass), None, u(evals), u(evecs), [gX], [gY])
            else:   # one contraction alone (the backward of each is the other)
                mass, L, evals, evecs, gX, gY = _case_ops(dn, case)
                V, K, C = mass.shape[0], evecs.shape[1], CASES[case][3]
                if what == "to_basis":
                    dn.ops.to_basis_raw(torch.randn(V, C, device="cuda"), evecs, mass)
                else:
                    dn.ops.from_basis_raw(torch.randn(K, C, device="cuda"), evecs)
                torch.cuda.synchronize()
                res[key] = "ok"
                continue
            out.square().sum().backward()
            torch.cuda.synchronize()
            res[key] = "ok"
        except RuntimeError as e:
            res[key] = "unsupported" if "unsupported" in str(e) else "error: " + str(e)
    print(json.dumps(res))


def test_dispatch_routes_under_strict_tc(dn):
    tests_dir = os.path.join(ROOT, "tests")
    env = dict(os.environ, DN_STRICT_TC="1")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", "import sys; sys.path[:0] = [{!r}, {!r}]; import test_gpu_backward as t; t._route_report()".format(
            tests_dir, ROOT)]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    want = {k: "ok" if v else "unsupported" for k, v in ROUTES.items()}
    assert got == want, {k: (got.get(k), want[k]) for k in want if got.get(k) != want[k]}


# ---- d. reproducibility ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("engine,C", [("tc3x", 128), ("simt", 128), ("tc3x", 256)])
def test_two_passes_give_bitwise_equal_gradients(dn, engine, C):
    """Two forward + backward passes of a 2-block net at V = 7056: every parameter and input gradient is bitwise
    equal.  Every gradient reduction (weights, biases, diffusion times) runs in a fixed order."""
    dn.set_engine(engine)
    K = 128
    mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(84, 84, K, seed=7, device="cuda")
    V = mass.shape[0]
    torch.manual_seed(7)
    net = dn.DiffusionNet(C_in=16, C_out=8, C_width=C, N_block=2, dropout=False).cuda().train()
    with torch.no_grad():
        for n_, p_ in net.named_parameters():
            if n_.endswith("diffusion_time"):
                p_.uniform_(1e-3, 0.3)
    g = _gen(23)
    x0, R = torch.randn(V, 16, generator=g).cuda(), torch.randn(V, 8, generator=g).cuda()
    runs = []
    for _ in range(2):
        for p_ in net.parameters():
            p_.grad = None
        x = x0.clone().requires_grad_(True)
        (net(x, mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY) * R).sum().backward()
        runs.append(({n_: p_.grad.clone() for n_, p_ in net.named_parameters()}, x.grad.clone()))
    (g0, x0g), (g1, x1g) = runs
    differ = [n_ for n_ in g0 if not torch.equal(g0[n_], g1[n_])]
    assert not differ, differ
    assert torch.equal(x0g, x1g)
