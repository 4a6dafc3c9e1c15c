"""Whole-shape classification (outputs_at='global_mean'): the mass-weighted segmented mean (ops.global_mean_pool), the
fused head with label smoothing (ops.linear_nll(..., label_smoothing)) and DiffusionNet.forward_global_nll /
forward_batch_global_nll, against fp64 torch.

Pool bound.  The kernel sums a segment of n rows as a tree: one CTA sums a run of at most 256 rows (at most 256
additions per lane, then a fold of at most 128 row groups), and a segment's runs (at most ceil(n / 256) + 1) are summed
over at most 128 slices, then folded.  Every term m_v x_v (one rounded product) therefore passes through at most
d = min(n, 1024 + ceil(n / 256)) + 1 roundings, and a sum of depth d is off by at most gamma_d sum |a| (gamma_d =
d u / (1 - d u), u = 2^-24).  With A = sum m |x| and M = sum m, the numerator is off by gamma_d A, the mass sum by
gamma_d M, and the quotient rounds once more:
  |pooled - pooled_64| <= (2 gamma_d + u) A / M         (to first order)
  |grad_x - grad_x_64| <= (gamma_d + 2 u) m |g| / M     (m / M_fp32, then one product)
both times a safety factor 2.

Head bound with smoothing.  With s' = s / (n_class - 1) the row loss is (1 - s - s') nll + s' sum_j (lse - z_j); the
kernel forms sum_j (lse - z_j) as sum_j (m - z_j) + n_class log(sum-exp) (m the row max).  On top of the plain nll
bound of test_gpu_linear_nll.py (scaled by |1 - s - s'|), the smoothed term is off by s' times: n_class e_r (the logit
errors), (n_class + 2 ceil(n_class / 128) + 8) u sum_j (m - z_j) (the fp32 running sum of non-negative terms and its
rescales), n_class ((n_class + 8) u) (the log of the fp32 sum-exp) and u |sum_j (lse - z_j)|; plus u |loss| for the
final combination.  The logit gradient is g (P - t) with t rounded to fp32: the plain bound's D gains u g t."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle_torch as T  # noqa: E402  (checker only)

pytestmark = pytest.mark.gpu

D = torch.float64
U = 2.0 ** -24
U_PROD = {"tc3x": 2.0 ** -22, "tc1x": 2.0 ** -11, "bf16": 2.0 ** -8}
TC_ENGINES = ["tc3x", "tc1x", "bf16"]
SAFETY = 2.0


@pytest.fixture(scope="module")
def dn():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import diffusion_net_b200 as dn_
    yield dn_
    dn_.set_engine("tc3x")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ---- 1. the pool against fp64 ---------------------------------------------------------------------------------------
def _ragged(n_seg=40, seed=0):
    """n_seg segment lengths: a 1-row segment, one shorter than a tile, lengths across tile edges; the last one is not
    padded, so V is not a multiple of 128."""
    g = _gen(seed)
    rows = [1, 77, 128, 129, 300] + [int(v) for v in torch.randint(1, 700, (n_seg - 6,), generator=g)] + [555]
    begin, r0 = [], 0
    for n in rows:
        begin.append(r0)
        r0 += (n + 127) // 128 * 128
    V = begin[-1] + rows[-1]
    assert V % 128 != 0 and len(rows) == n_seg
    return begin, rows, V


LAYOUTS = {"ragged40": _ragged(), "single200k": ([0], [200000], 200000)}


def _pool_inputs(V, C, seed):
    g = _gen(seed)
    x = torch.randn(V, C, generator=g)
    mass = torch.rand(V, generator=g) + 0.25
    return x.cuda(), mass.cuda()


def _pool_gold(x, mass, begin, rows, g):
    """fp64 pooled rows, gradient and the ingredients of the bounds (on the GPU)."""
    x64, m64, g64 = x.to(D), mass.to(D), g.to(D)
    pooled, A, M, gx = [], [], [], torch.zeros_like(x64)
    for b, (r0, n) in enumerate(zip(begin, rows)):
        xs, ms = x64[r0:r0 + n], m64[r0:r0 + n]
        Mb = ms.sum()
        pooled.append((ms[:, None] * xs).sum(0) / Mb)
        A.append((ms[:, None] * xs.abs()).sum(0))
        M.append(Mb)
        gx[r0:r0 + n] = ms[:, None] / Mb * g64[b]
    return torch.stack(pooled), torch.stack(A), torch.stack(M), gx


def _pad_mask(begin, rows, V):
    pad = torch.ones(V, dtype=torch.bool, device="cuda")
    for r0, n in zip(begin, rows):
        pad[r0:r0 + n] = False
    return pad


@pytest.mark.parametrize("C", [16, 64, 128, 256])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_pool_vs_fp64(dn, layout, C):
    begin, rows, V = LAYOUTS[layout]
    seg = dn.ops.Segments(begin, rows, V, "cuda")
    x, mass = _pool_inputs(V, C, seed=C + V)
    xg = x.clone().requires_grad_(True)
    pooled = dn.ops.global_mean_pool(xg, mass, seg)
    g = torch.randn(len(rows), C, generator=_gen(C)).cuda()
    pooled.backward(g)
    torch.cuda.synchronize()
    P64, A, M, gx64 = _pool_gold(x, mass, begin, rows, g)
    d = torch.tensor([min(n, 1024 + math.ceil(n / 256)) + 1 for n in rows], dtype=D, device="cuda")
    gam = d * U / (1 - d * U)
    bound = SAFETY * (2 * gam + U)[:, None] * A / M[:, None]
    err = (pooled.detach().to(D) - P64).abs()
    assert bool((err <= bound).all()), "pooled: worst err/bound {:.3g}".format(float((err / bound).max()))
    # gradient: per-row bound from the row's segment
    seg_of = torch.full((V,), -1, dtype=torch.int64, device="cuda")
    for b, (r0, n) in enumerate(zip(begin, rows)):
        seg_of[r0:r0 + n] = b
    pad = seg_of < 0
    s_of = seg_of.clamp(min=0)
    bg = SAFETY * (gam[s_of] + 2 * U)[:, None] * mass.to(D)[:, None] * g.to(D)[s_of].abs() / M[s_of][:, None]
    err = (xg.grad.to(D) - gx64).abs()
    assert bool((err[~pad] <= bg[~pad] + 1e-30).all()), "grad_x: worst err/bound {:.3g}".format(
        float((err[~pad] / (bg[~pad] + 1e-30)).max()))
    if pad.any():
        assert not xg.grad[pad].any()                    # exactly 0 on padding rows
        # padding rows are never read: 1e3 or NaN there changes no output bit
        for fill in (1e3, float("nan")):
            x2, m2 = x.clone(), mass.clone()
            x2[pad], m2[pad] = fill, fill
            p2 = dn.ops.global_mean_pool(x2, m2, seg)
            assert torch.equal(p2, pooled.detach()), fill


def test_pool_single_mesh_default_segment(dn):
    """segments=None is one segment [0, V), built once per V."""
    x, mass = _pool_inputs(1000, 64, seed=3)
    p = dn.ops.global_mean_pool(x, mass)
    assert p.shape == (1, 64)
    assert dn.ops.single_segment(1000, x.device) is dn.ops.single_segment(1000, x.device)
    ref = (mass.to(D)[:, None] * x.to(D)).sum(0) / mass.to(D).sum()
    assert torch.allclose(p[0].to(D), ref, rtol=0, atol=1e-5)
    with pytest.raises(RuntimeError):                   # mass is data: no gradient
        dn.ops.global_mean_pool(x, mass.clone().requires_grad_(True))


# ---- 2. the head with label smoothing against fp64 ------------------------------------------------------------------
def _head_inputs(R, C, n, seed):
    g = _gen(seed)
    x = torch.randn(R, C, generator=g)
    w = torch.randn(n, C, generator=g) / C ** 0.5
    b = torch.randn(n, generator=g) * 0.1
    lab = torch.randint(0, n, (R,), generator=g)
    if R > 7:
        lab[::7] = -100
    gr = torch.rand(R, generator=g) + 0.5
    return x, w, b, lab, gr


def _smooth_target(lab, n, s, dtype=D):
    """The reference's label_smoothing_log_loss target per row (rows with an ignored label: 0)."""
    ok = lab != -100
    t = torch.full((lab.shape[0], n), s / (n - 1), dtype=dtype)
    t[ok] = t[ok].scatter(1, lab[ok][:, None], 1.0 - s)
    t[~ok] = 0
    return t


def _head_gold(x, w, b, lab, gr, s):
    x64, w64, b64 = (t.to(D).requires_grad_(True) for t in (x, w, b))
    z = x64 @ w64.t() + b64
    logp = torch.log_softmax(z, dim=-1)
    n = w.shape[0]
    t = _smooth_target(lab, n, s)
    loss = -(t * logp).sum(-1)
    (loss * gr.to(D)).sum().backward()
    with torch.no_grad():
        keep = (lab != -100).to(D)
        P = logp.exp()
        lse = torch.logsumexp(z, 1)
        m = z.max(1).values
        zl = z.gather(1, lab.clamp(min=0)[:, None])[:, 0] * keep
        ax = (x64.abs() @ w64.abs().t() + b64.abs()).max(dim=1).values
        top = torch.topk(z, min(2, n), dim=1).values
        gap = top[:, 0] - top[:, 1] if n > 1 else torch.full_like(m, float("inf"))
    return dict(loss=loss.detach(), gx=x64.grad, gw=w64.grad, gb=b64.grad, P=P, t=t, lse=lse, m=m, zl=zl, ax=ax,
                z=z.detach(), gap=gap, argmax=z.detach().argmax(1), x=x64.detach(), w=w64.detach(),
                gr=gr.to(D) * keep)


def _head_check(engine, G, s, loss, pred, gx, gw, gb, what):
    up = U_PROD[engine]
    R, C = G["x"].shape
    n = G["w"].shape[0]
    off = s / (n - 1)
    e = (2 * up + (C + 1) * U) * G["ax"]
    b_plain = 2 * e + (n + 8) * U + 2 * U * (G["lse"].abs() + G["zl"].abs())
    dsum = (G["m"][:, None] - G["z"]).sum(1)
    tot = (G["lse"][:, None] - G["z"]).sum(1)
    b_smooth = off * (n * e + (n + 2 * math.ceil(n / 128) + 8) * U * dsum + n * (n + 8) * U + U * tot.abs())
    keep = G["gr"] != 0
    bound = SAFETY * (abs(1 - s - off) * b_plain + b_smooth + U * G["loss"].abs()) * keep
    err = (loss.cpu().to(D) - G["loss"]).abs()
    assert bool((err <= bound).all()), "{} loss: worst err/bound {:.3g}".format(what, float((err / (bound + 1e-300)).max()))
    sure = G["gap"] > 4 * e
    assert bool((pred.cpu()[sure] == G["argmax"][sure]).all()), "{} argmax".format(what)
    Dm = G["gr"][:, None] * (G["P"] * torch.expm1(2 * e + (n + 12) * U)[:, None] + U * G["t"])
    dz = G["gr"][:, None] * (G["P"] - G["t"])
    A = dz.abs() + Dm
    b_gx = SAFETY * (Dm @ G["w"].abs() + (2 * up + (n + 1) * U) * (A @ G["w"].abs()))
    b_gw = SAFETY * (Dm.t() @ G["x"].abs() + (2 * up + (R + 1) * U) * (A.t() @ G["x"].abs()))
    b_gb = SAFETY * (Dm.sum(0) + (2 * up + (R + 1) * U) * A.sum(0))
    for name, ours, gold, bnd in (("grad_x", gx, G["gx"], b_gx), ("grad_w", gw, G["gw"], b_gw),
                                  ("grad_b", gb, G["gb"], b_gb)):
        err = (ours.cpu().to(D) - gold).abs()
        bnd = bnd + 1e-30
        assert bool((err <= bnd).all()), "{} {}: worst err/bound {:.3g}".format(what, name, float((err / bnd).max()))


def _head_run(dn, x, w, b, lab, gr, s):
    xc, wc, bc = (t.cuda().requires_grad_(True) for t in (x, w, b))
    loss, pred = dn.ops.linear_nll(xc, wc, bc, lab.cuda(), -100, label_smoothing=s)
    (loss * gr.cuda()).sum().backward()
    torch.cuda.synchronize()
    return loss.detach(), pred, xc.grad, wc.grad, bc.grad


@pytest.mark.parametrize("R", [1, 129, 300])
@pytest.mark.parametrize("n", [2, 8, 30, 129, 260])
@pytest.mark.parametrize("s", [0.2, 1.0])
@pytest.mark.parametrize("engine", TC_ENGINES)
def test_linear_nll_smoothing_vs_fp64(dn, engine, s, n, R):
    dn.set_engine(engine)
    args = _head_inputs(R, 64, n, seed=R + n)
    G = _head_gold(*args, s)
    _head_check(engine, G, s, *_head_run(dn, *args, s), "{} s={} n={} R={}".format(engine, s, n, R))


def _raw_head(dn, x, w, b, lab, g, s, entry):
    """Forward and backward through the plain (entry 'old') or the smoothing (entry 'ls') C-ABI entries."""
    lib = dn._lib.load()
    R, C = x.shape
    n = w.shape[0]
    P = lambda t: t.data_ptr()  # noqa: E731
    nll, lse = torch.empty(R, device="cuda"), torch.empty(R, device="cuda")
    am = torch.empty(R, dtype=torch.int64, device="cuda")
    fwd = (P(x), P(w), P(b), P(lab), R, C, n, -100, P(nll), P(am), P(lse), dn._lib.ENGINE_TC3X, None)
    rc = lib.dn_linear_nll_fwd(*fwd) if entry == "old" else lib.dn_linear_nll_ls_fwd(*fwd, s)
    assert rc == 0
    need = lib.dn_linear_nll_workspace_bytes(R, C, n)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    gx, gw, gb = torch.empty_like(x), torch.empty_like(w), torch.empty_like(b)
    bwd = (P(x), P(w), P(b), P(lab), P(lse), P(g), R, C, n, -100, P(gx), P(gw), P(gb), P(ws), need,
           dn._lib.ENGINE_TC3X, None)
    rc = lib.dn_linear_nll_bwd(*bwd) if entry == "old" else lib.dn_linear_nll_ls_bwd(*bwd, s)
    assert rc == 0
    torch.cuda.synchronize()
    return nll, lse, am, gx, gw, gb


def test_smoothing_zero_is_the_plain_head_bitwise(dn):
    for (R, C, n) in [(300, 64, 30), (6890, 128, 260)]:
        x, w, b, lab, gr = (t.cuda() for t in _head_inputs(R, C, n, seed=R))
        old = _raw_head(dn, x, w, b, lab, gr, 0.0, "old")
        new = _raw_head(dn, x, w, b, lab, gr, 0.0, "ls")
        for a, b_ in zip(old, new):
            assert torch.equal(a, b_)


def test_simt_engine_composes_the_smoothed_target(dn):
    args = _head_inputs(300, 48, 30, seed=12)
    G = _head_gold(*args, 0.2)
    dn.set_engine("simt")
    try:
        loss, pred, gx, gw, gb = _head_run(dn, *args, 0.2)
    finally:
        dn.set_engine("tc3x")
    err = (loss.cpu().to(D) - G["loss"]).abs().max().item()
    assert err <= 1e-5 * G["loss"].abs().max().item()
    for ours, gold in ((gx, G["gx"]), (gw, G["gw"]), (gb, G["gb"])):
        assert (ours.cpu().to(D) - gold).abs().max().item() <= 1e-5 * gold.abs().max().item()


# ---- 3. forward_global_nll against the fp64 oracle composition ------------------------------------------------------
def label_smoothing_log_loss(pred, labels, smoothing=0.0):
    """The reference's loss of the classification experiment (utils.py), on one mesh's 1-D prediction."""
    n_class = pred.shape[-1]
    one_hot = torch.zeros_like(pred)
    one_hot[labels] = 1.
    one_hot = one_hot * (1 - smoothing) + (1 - one_hot) * smoothing / (n_class - 1)
    return -(one_hot * pred).sum(dim=-1).mean()


def _net(dn, K, n_class=30, C=64, N_block=4, outputs_at="global_mean", seed=0):
    """The SHREC11 classifier: C_in 16, C_width 64, 4 blocks, 30 classes, global mean, log_softmax."""
    torch.manual_seed(seed)
    net = dn.DiffusionNet(C_in=16, C_out=n_class, C_width=C, N_block=N_block, dropout=False, outputs_at=outputs_at,
                          last_activation=lambda x: F.log_softmax(x, dim=-1)).cuda().train()
    with torch.no_grad():
        for n_, p_ in net.named_parameters():
            if n_.endswith("diffusion_time"):
                p_.uniform_(1e-3, 0.3)
    return net


def _gold_global(net, x, mass, evals, evecs, gX, gY, label, s, N_block):
    prm = {k: v.detach().cpu().to(D).requires_grad_(True) for k, v in net.state_dict().items()}
    m64, e64, v64 = (t.cpu().to(D).unsqueeze(0) for t in (mass, evals, evecs))
    h = torch.addmm(prm["first_lin.bias"], x.cpu().to(D), prm["first_lin.weight"].t()).unsqueeze(0)
    for b in range(N_block):
        bp = {k[len("block_%d." % b):]: v for k, v in prm.items() if k.startswith("block_%d." % b)}
        h = T.block_forward(h, m64, e64, v64, [gX.cpu().to(D)], [gY.cpu().to(D)], bp)
    z = torch.addmm(prm["last_lin.bias"], h[0], prm["last_lin.weight"].t())
    pooled = (z * m64[0][:, None]).sum(0) / m64[0].sum()
    loss = label_smoothing_log_loss(F.log_softmax(pooled, -1), label.cpu(), s)
    loss.backward()
    return loss.detach(), pooled.detach(), prm


@pytest.mark.parametrize("s", [0.0, 0.2])
def test_forward_global_nll_vs_fp64(dn, s):
    dn.set_engine("tc3x")
    n, m, K = 20, 24, 128
    mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=2, device="cuda")
    net = _net(dn, K)
    x = torch.randn(mass.shape[0], 16, generator=_gen(4)).cuda()
    label = torch.tensor([7]).cuda()
    loss, pred = net.forward_global_nll(x, mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY, labels=label,
                                        label_smoothing=s)
    assert loss.dim() == 0 and pred.dim() == 0 and pred.dtype == torch.int64
    loss.backward()
    grads = {k: p_.grad.clone() for k, p_ in net.named_parameters()}
    gold, pooled, prm = _gold_global(net, x, mass, evals, evecs, gX, gY, label, s, 4)
    # test_gpu_backward.py's fp32 bounds: 1e-5 on outputs, 5e-5 on parameter gradients (relative to the largest)
    assert abs(loss.item() - gold.item()) <= 1e-5 * abs(gold.item())
    for k, p_ in prm.items():
        if k not in grads:
            continue
        err = (grads[k].cpu().to(D) - p_.grad).abs().max().item()
        assert err <= 5e-5 * p_.grad.abs().max().item() + 1e-12, (k, err)
    top = torch.topk(pooled, 2).values
    if top[0] - top[1] > 1e-4:
        assert pred.item() == int(pooled.argmax())
    # the same net's forward (reference order: last_lin, mean, log_softmax) agrees
    with torch.no_grad():
        out = net(x, mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY)
    ref = label_smoothing_log_loss(out, label, s)
    assert abs(ref.item() - loss.item()) <= 1e-5 * abs(gold.item())


# ---- 4. the batch route equals the per-mesh loop --------------------------------------------------------------------
SHAPES = [(9, 11), (14, 10), (7, 8), (20, 13), (6, 7)]    # 99, 140, 56, 260, 42 vertices


def _meshes(dn, shapes, K):
    out = []
    for i, (n, m) in enumerate(shapes):
        mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=i, device="cuda")
        out.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY))
    return out


def _single(net, it, x, label, s):
    return net.forward_global_nll(x, it["mass"], evals=it["evals"], evecs=it["evecs"], gradX=it["gradX"],
                                  gradY=it["gradY"], labels=label, label_smoothing=s)


def test_forward_batch_global_nll_matches_per_mesh(dn):
    dn.set_engine("tc3x")
    K, s = 32, 0.2
    meshes = _meshes(dn, SHAPES, K)
    mb = dn.MeshBatch(meshes)
    net = _net(dn, K)
    xs = [torch.randn(it["mass"].shape[0], 16, generator=_gen(20 + i)).cuda() for i, it in enumerate(meshes)]
    labs = [torch.tensor([i * 5 % 30]).cuda() for i in range(len(meshes))]
    net.zero_grad()
    losses, preds = net.forward_batch_global_nll(mb, xs, labs, label_smoothing=s)
    assert losses.shape == (len(meshes),) and preds.shape == (len(meshes),)
    losses.sum().backward()
    gb = {k: p_.grad.clone() for k, p_ in net.named_parameters()}
    net.zero_grad()
    for i, it in enumerate(meshes):
        l1, p1 = _single(net, it, xs[i], labs[i], s)
        assert abs(l1.item() - losses[i].item()) <= 1e-5 * abs(l1.item()), i
        assert p1.item() == preds[i].item(), i
        l1.backward()
    for k, p_ in net.named_parameters():
        err = (p_.grad - gb[k]).abs().max().item()
        assert err <= 5e-5 * p_.grad.abs().max().item() + 1e-12, (k, err)
    # labels as one (n_meshes,) tensor; the padding rows of the batch layout are never read
    x_lay = mb.pack(xs)
    pad = _pad_mask(mb.row_begin[:-1], mb.n_rows, mb.V)
    assert pad.any()
    x2 = x_lay.clone()
    x2[pad] = 1e3
    with torch.no_grad():
        a, pa = net.forward_batch_global_nll(mb, x_lay, torch.cat(labs), label_smoothing=s)
        b_, pb = net.forward_batch_global_nll(mb, x2, torch.cat(labs), label_smoothing=s)
    assert torch.equal(a, b_) and torch.equal(pa, pb)


# ---- 5. CUDA graphs -------------------------------------------------------------------------------------------------
def test_graphed_train_steps(dn):
    dn.set_engine("tc3x")
    K, s = 32, 0.2
    meshes = _meshes(dn, SHAPES[:3], K)
    mb = dn.MeshBatch(meshes)
    net = _net(dn, K)
    xs = [torch.randn(it["mass"].shape[0], 16, generator=_gen(40 + i)).cuda() for i, it in enumerate(meshes)]
    labs = torch.tensor([3, 17, 29]).cuda()
    it = meshes[0]

    def single(net_, x_, l_):
        return _single(net_, it, x_, l_, s)[0]

    def batched(net_, xs_, l_):
        return net_.forward_batch_global_nll(mb, xs_, l_, label_smoothing=s)[0].sum()

    for fn, inputs in ((single, (xs[0], labs[:1])), (batched, (xs, labs))):
        net.zero_grad()
        fn(net, *inputs).backward()
        ref = {k: p_.grad.clone() for k, p_ in net.named_parameters()}
        step = dn.graphs.GraphedTrainStep(net, fn, inputs)
        dn.graphs.GraphedTrainStep.zero_grads(net)
        step.replay()
        torch.cuda.synchronize()
        for k, p_ in net.named_parameters():
            assert torch.equal(p_.grad, ref[k]), (fn.__name__, k)


# ---- 6. determinism and launch counts -------------------------------------------------------------------------------
def test_deterministic_and_launch_counts(dn):
    dn.set_engine("tc3x")
    lib = dn._lib.load()
    pool_counts = {}
    for name, (begin, rows, V) in (("one", ([0], [5000], 5000)), ("forty", LAYOUTS["ragged40"])):
        seg = dn.ops.Segments(begin, rows, V, "cuda")
        x, mass = _pool_inputs(V, 64, seed=1)
        g = torch.randn(len(rows), 64, generator=_gen(2)).cuda()
        runs = []
        for _ in range(2):
            xg = x.clone().requires_grad_(True)
            c0 = lib.dn_kernel_launch_count()
            p = dn.ops.global_mean_pool(xg, mass, seg)
            c1 = lib.dn_kernel_launch_count()
            p.backward(g)
            c2 = lib.dn_kernel_launch_count()
            pool_counts.setdefault(name, set()).add((c1 - c0, c2 - c1))
            runs.append((p.detach(), xg.grad))
        assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    assert pool_counts == {"one": {(2, 1)}, "forty": {(2, 1)}}, pool_counts
    # the smoothed head: 1 forward and 3 backward launches, bitwise reproducible
    x, w, b, lab, gr = _head_inputs(1000, 64, 30, seed=5)
    runs, counts = [], set()
    for _ in range(2):
        xc, wc, bc = (t.cuda().requires_grad_(True) for t in (x, w, b))
        c0 = lib.dn_kernel_launch_count()
        loss, pred = dn.ops.linear_nll(xc, wc, bc, lab.cuda(), label_smoothing=0.2)
        c1 = lib.dn_kernel_launch_count()
        (loss * gr.cuda()).sum().backward()
        counts.add((c1 - c0, lib.dn_kernel_launch_count() - c1))
        runs.append((loss.detach(), pred, xc.grad, wc.grad, bc.grad))
    assert counts == {(1, 3)}, counts
    assert all(torch.equal(a, b_) for a, b_ in zip(*runs))


# ---- 7. refusals ----------------------------------------------------------------------------------------------------
def test_c_abi_refusals_enqueue_nothing(dn):
    lib = dn._lib.load()
    P = lambda t: t.data_ptr()  # noqa: E731
    V, C = 1000, 64
    seg = dn.ops.Segments([0], [V], V, "cuda")
    x, mass = _pool_inputs(V, 260, seed=0)
    out, msum = torch.empty(1, 260, device="cuda"), torch.empty(1, device="cuda")
    need = lib.dn_global_mean_workspace_bytes(V, C)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    tabs = (P(seg.begin), P(seg.rows), P(seg.tile_seg), 1)
    c0 = lib.dn_kernel_launch_count()
    for CC in (6, 260):
        rc = lib.dn_global_mean_fwd(P(x), P(mass), V, CC, *tabs, P(out), P(msum), P(ws), 1 << 30, None)
        assert rc == -2, (CC, rc)
        rc = lib.dn_global_mean_bwd(P(out), P(mass), P(msum), V, CC, *tabs, P(x), None)
        assert rc == -2, (CC, rc)
    rc = lib.dn_global_mean_fwd(P(x), P(mass), V, C, *tabs, P(out), P(msum), P(ws), need - 4, None)
    assert rc == -3
    R, n = 300, 30
    hx, hw, hb, lab, gr = (t.cuda() for t in _head_inputs(R, C, n, seed=13))
    nll = torch.empty(R, device="cuda")
    am = torch.empty(R, dtype=torch.int64, device="cuda")
    hneed = lib.dn_linear_nll_workspace_bytes(R, C, n)
    hws = torch.empty(hneed, dtype=torch.uint8, device="cuda")
    gx, gw, gbias = torch.empty_like(hx), torch.empty_like(hw), torch.empty_like(hb)
    tc = dn._lib.ENGINE_TC3X
    for s, nn_ in ((-0.1, n), (1.5, n), (float("nan"), n), (0.2, 1)):
        rc = lib.dn_linear_nll_ls_fwd(P(hx), P(hw), P(hb), P(lab), R, C, nn_, -100, P(nll), P(am), P(nll), tc, None, s)
        assert rc == -1, (s, nn_, rc)
        rc = lib.dn_linear_nll_ls_bwd(P(hx), P(hw), P(hb), P(lab), P(nll), P(gr), R, C, nn_, -100, P(gx), P(gw),
                                      P(gbias), P(hws), hneed, tc, None, s)
        assert rc == -1, (s, nn_, rc)
    rc = lib.dn_linear_nll_ls_bwd(P(hx), P(hw), P(hb), P(lab), P(nll), P(gr), R, C, n, -100, P(gx), P(gw), P(gbias),
                                  P(hws), hneed - 8, tc, None, 0.2)
    assert rc == -3
    assert lib.dn_kernel_launch_count() == c0


def test_python_refusals(dn):
    K = 32
    meshes = _meshes(dn, SHAPES[:2], K)
    mb = dn.MeshBatch(meshes)
    it = meshes[0]
    x = torch.randn(it["mass"].shape[0], 16).cuda()
    kw = dict(evals=it["evals"], evecs=it["evecs"], gradX=it["gradX"], gradY=it["gradY"])
    seg_net = _net(dn, K, N_block=1, outputs_at="vertices")
    with pytest.raises(ValueError):
        seg_net.forward_global_nll(x, it["mass"], labels=torch.tensor([1]).cuda(), **kw)
    with pytest.raises(ValueError):
        seg_net.forward_batch_global_nll(mb, [x, x], torch.tensor([1, 2]).cuda())
    net = _net(dn, K, N_block=1)
    with pytest.raises(ValueError):        # forward_nll has no global_mean route
        net.forward_nll(x, it["mass"], labels=torch.tensor([1]).cuda(), **kw)
    with pytest.raises(ValueError):        # two labels for one mesh
        net.forward_global_nll(x, it["mass"], labels=torch.tensor([1, 2]).cuda(), **kw)
    with pytest.raises(ValueError):        # not int64
        net.forward_global_nll(x, it["mass"], labels=torch.tensor([1.0]).cuda(), **kw)
    xs = [torch.randn(m["mass"].shape[0], 16).cuda() for m in meshes]
    with pytest.raises(ValueError):        # one label for two meshes
        net.forward_batch_global_nll(mb, xs, torch.tensor([1]).cuda())
    with pytest.raises(ValueError):
        net.forward_batch_global_nll(mb, xs, [torch.tensor([1]).cuda()])
    with pytest.raises(ValueError):        # a label tensor of two elements
        net.forward_batch_global_nll(mb, xs, [torch.tensor([1, 2]).cuda(), torch.tensor([1]).cuda()])
    with pytest.raises(ValueError):
        net.forward_global_nll(x, it["mass"], labels=torch.tensor([1]).cuda(), label_smoothing=1.5, **kw)
