"""The functional-map head on the GPU: ``dn_fmap_solve_fwd`` / ``_bwd``, ``dn_nearest_neighbor`` and the model built on
them (diffusion_net_b200/fmaps.py), against fp64 golds.

Bounds (u = 2^-24, the fp32 unit roundoff; eps = 2^-53, fp64's):
  * solve: each row is computed in fp64 and rounded once to fp32, so
      max_j |C[i][j] - C_gold[i][j]| <= (u + 16 n (n + d) kappa(S_i) eps) max_j |C_gold[i][j]|,
    the second term covering the fp64 Gram / Cholesky / substitution error of both our solve and scipy's.  dA and dB are
    two fp64 solves and an fp64 contraction away from their fp32 rounding: rel_err <= 4u + 16 n (n + d) kappa_max eps.
  * nearest neighbour: each distance is one fp32 chain over n terms of rounded differences, so the computed distance is
    within tau = (n + 2) u / (1 - (n + 2) u) of the exact distance of the fp32 inputs (relative; all terms are >= 0).
    Hence the chosen target's exact squared distance is at most d_min (1 + tau) / (1 - tau), and wherever the
    second-best exact distance exceeds that, the index is the exact argmin.
"""
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle as O  # noqa: E402
import dn_oracle_fmaps as OF  # noqa: E402
import dn_oracle_torch as T  # noqa: E402

import diffusion_net_b200 as dn  # noqa: E402

gpu = pytest.mark.gpu
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
U32, EPS64 = 2.0 ** -24, 2.0 ** -53
N = 30
LAMBDA = 1e-3


@pytest.mark.skipif(shutil.which(NVCC) is None and not os.path.exists(NVCC), reason="nvcc not found")
def test_fmap_kernels_do_not_spill(tmp_path):
    flags = [f for f in dn._lib.NVCC_FLAGS if f != "-shared"]
    cmd = [NVCC] + flags + ["-Xptxas", "-v", "-c", os.path.join(dn._lib._CSRC, "dn_fmap.cu"), "-o",
                            str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [l for l in (r.stdout + r.stderr).splitlines() if "spill stores" in l]
    assert len(lines) == 9      # row solve, gradient, 6 nearest-neighbour widths, combine
    for l in lines:
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", l)
        assert m and m.group(1) == "0" and m.group(2) == "0", l


def _launches():
    return dn._lib.load().dn_kernel_launch_count()


def _solve_inputs(n, d, seed=0):
    rs = np.random.RandomState(seed)
    A = rs.randn(n, d).astype(np.float32)
    B = rs.randn(n, d).astype(np.float32)
    ex = np.sort(rs.rand(n) * 40).astype(np.float32)
    ey = np.sort(rs.rand(n) * 40).astype(np.float32)
    ey[0] = ex[0]                      # D[0][0] = 0: row 0 has one unregularised entry
    return A, B, ex, ey


def _kappas(A, ex, ey, lam):
    A = A.astype(np.float64)
    AAt = A @ A.T
    D = (ex.astype(np.float64)[None, :] - ey.astype(np.float64)[:, None]) ** 2
    return np.array([np.linalg.cond(AAt + lam * np.diag(D[i])) for i in range(A.shape[0])])


def _cuda(*arrs):
    return [torch.from_numpy(a).cuda() for a in arrs]


def _torch_solve(A, B, ex, ey, lam):
    """float64 torch restatement of fmaps_model.py:26-38."""
    D = (ex[None, :] - ey[:, None]) ** 2
    AAt, BAt = A @ A.T, B @ A.T
    return torch.stack([torch.linalg.solve(AAt + lam * torch.diag(D[i]), BAt[i]) for i in range(A.shape[0])])


WORST = {}


@gpu
@pytest.mark.parametrize("n", [1, 8, 30, 128])
@pytest.mark.parametrize("d", [16, 128, 200])
def test_solve_against_oracle(n, d):
    A, B, ex, ey = _solve_inputs(n, d, seed=n * 1000 + d)
    At, Bt, ext, eyt = _cuda(A, B, ex, ey)
    At.requires_grad_(True)
    Bt.requires_grad_(True)
    C = dn.fmaps.fmap_solve(At, Bt, ext, eyt, LAMBDA)
    gold = OF.solve(A, B, ex, ey, LAMBDA)
    kap = _kappas(A, ex, ey, LAMBDA)
    Cn = C.detach().cpu().numpy().astype(np.float64)
    fp64_term = 16 * n * (n + d) * EPS64
    for i in range(n):
        scale = np.abs(gold[i]).max()
        err = np.abs(Cn[i] - gold[i]).max()
        assert err <= (U32 + fp64_term * kap[i]) * scale, (i, err / scale, kap[i])
    WORST["C", n, d] = float((np.abs(Cn - gold).max(axis=1) / np.abs(gold).max(axis=1)).max())
    g = np.random.RandomState(7).randn(n, n).astype(np.float32)
    (C * torch.from_numpy(g).cuda()).sum().backward()
    A64, B64 = torch.tensor(A, dtype=torch.float64, requires_grad=True), torch.tensor(B, dtype=torch.float64,
                                                                                     requires_grad=True)
    (_torch_solve(A64, B64, torch.tensor(ex, dtype=torch.float64), torch.tensor(ey, dtype=torch.float64), LAMBDA)
     * torch.tensor(g, dtype=torch.float64)).sum().backward()
    tol = 4 * U32 + fp64_term * kap.max()
    eA, eB = O.rel_err(At.grad.cpu().numpy(), A64.grad.numpy()), O.rel_err(Bt.grad.cpu().numpy(), B64.grad.numpy())
    assert eA <= tol and eB <= tol, (eA, eB, tol)
    dA_o, dB_o = OF.solve_adjoint(A, B, ex, ey, LAMBDA, g)
    assert O.rel_err(At.grad.cpu().numpy(), dA_o) <= tol and O.rel_err(Bt.grad.cpu().numpy(), dB_o) <= tol
    print("fmap solve n={} d={}: C {:.2e}, dA {:.2e}, dB {:.2e}, kappa_max {:.1e}".format(n, d, WORST["C", n, d], eA,
                                                                                        eB, kap.max()))


@gpu
def test_solve_is_deterministic_with_one_forward_and_two_backward_launches():
    A, B, ex, ey = _solve_inputs(N, 128, seed=3)
    At, Bt, ext, eyt = _cuda(A, B, ex, ey)
    g = torch.randn(N, N, generator=torch.Generator().manual_seed(1)).cuda()
    outs = []
    for _ in range(2):
        a, b = At.clone().requires_grad_(True), Bt.clone().requires_grad_(True)
        torch.cuda.synchronize()
        n0 = _launches()
        C = dn.fmaps.FmapSolveFn.apply(a, b, ext, eyt, LAMBDA)
        n1 = _launches()
        C.backward(g)
        torch.cuda.synchronize()
        n2 = _launches()
        assert n1 - n0 == 1 and n2 - n1 <= 2, (n1 - n0, n2 - n1)
        outs.append((C.detach().clone(), a.grad.clone(), b.grad.clone()))
    for x, y in zip(*outs):
        assert torch.equal(x, y)


@gpu
def test_singular_rows_are_nan_without_sync():
    n, d = 8, 16
    A, B, ex, ey = _solve_inputs(n, d, seed=11)
    A[3] = 0.0                           # A A^T has a zero row / column 3
    ey[5] = ex[3]                        # ... and row 5's regulariser is 0 there: S_5 is singular
    At, Bt, ext, eyt = _cuda(A, B, ex, ey)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        C = dn.fmaps.fmap_solve(At, Bt, ext, eyt, LAMBDA)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    Cn = C.cpu().numpy()
    bad = ~np.isfinite(Cn).all(axis=1)
    assert bad.tolist() == [i == 5 for i in range(n)]
    assert np.isnan(Cn[5]).all()


# ---- the fixture model -------------------------------------------------------------------------------------------
def _shape(fx, tag):
    f = lambda k: fx[tag + ":" + k]
    V = f("mass").shape[0]
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    gX = torch.sparse_coo_tensor(cu(f("gradX_idx")), cu(f("gradX_vals")), (V, V)).coalesce()
    gY = torch.sparse_coo_tensor(cu(f("gradY_idx")), cu(f("gradY_vals")), (V, V)).coalesce()
    return [cu(f("verts")), cu(f("faces")), None, cu(f("mass")), None, cu(f("evals")), cu(f("evecs")), gX, gY, None,
            torch.arange(V, device="cuda")]


def _fixture_model(fx):
    m = dn.FunctionalMapCorrespondenceWithDiffusionNetFeatures(n_feat=128, input_features="xyz")
    sd = {k[2:]: torch.from_numpy(v.astype(np.float32)) for k, v in fx.items() if k.startswith("p:")}
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


@gpu
def test_fixture_model_matches_reference():
    fx = load_golden("fmaps_small")
    dn.set_engine("tc3x")
    m = _fixture_model(fx)
    s1, s2 = _shape(fx, "x"), _shape(fx, "y")
    C_pred, f1, f2 = m(s1, s2)
    assert C_pred.shape == (1, N, N)
    for mine, key in ((C_pred[0], "C"), (f1, "feat1"), (f2, "feat2")):
        tol = max(1e-5, 4 * float(fx["err32:" + key]))
        err = O.rel_err(mine.detach().cpu().numpy(), fx["C64" if key == "C" else key + "_64"])
        print("fixture {}: {:.2e} (tol {:.2e})".format(key, err, tol))
        assert err <= tol, (key, err, tol)
    # Gold: fp64 autograd of dn_oracle_fmaps.model_torch, pinned to the reference's fp64 run by test_fmaps_oracle.py.
    # The loss is mean((C_pred - C_gt)^2), whose upstream gradient G = 2 (C_pred - C_gt) / n^2 is taken at the fp64 C.
    # An fp32 C (ours or the reference's own, 2.6e-5 .. 3.2e-5 off) perturbs G by about 1e-4 relative: that is the
    # loss's conditioning, not the backward's.  So the backward is fed the same G.  What remains is the fp32 floor of
    # the backward through the solve and both nets; the fixture records the reference's own fp32 error under the same G
    # (``gradfloor:``, up to 6e-5), and the bound is max(5e-5, 4 x that floor), as for C above.
    C64, _, _, prm = OF.fixture_model_gold(fx, n=N, lam=LAMBDA)
    G64 = 2 * (C64.detach() - torch.from_numpy(fx["C_gt"])) / N ** 2
    (C64 * G64).sum().backward()
    (C_pred[0] * G64.float().cuda()).sum().backward()
    worst = 0.0
    for k, p in m.named_parameters():
        e = O.rel_err(p.grad.cpu().numpy(), prm[k].grad.numpy())
        worst = max(worst, e)
        assert e <= max(5e-5, 4 * float(fx["gradfloor:" + k])), (k, e, float(fx["gradfloor:" + k]))
    print("fixture parameter gradients: worst {:.2e}".format(worst))
    # the pointwise map from the reference's own C, against its KD-tree map under the gap rule
    Cref = torch.from_numpy(fx["C32"]).cuda()
    idx = dn.pointwise_map(Cref, s1[6], s2[6], n_fmap=N).cpu().numpy()
    phi, C64 = fx["x:evecs"][:, :N].astype(np.float64), fx["C32"].astype(np.float64)
    eps_row = np.sqrt(((2 * N * U32 / (1 - N * U32) * (np.abs(phi) @ np.abs(C64).T)) ** 2).sum(1)).max()
    tau = (N + 2) * U32 / (1 - (N + 2) * U32)
    r1, r2 = np.sqrt(fx["map_d1"]), np.sqrt(fx["map_d2"])
    sure = (r2 - r1) > 2 * eps_row + tau * r2
    assert sure.mean() > 0.9, sure.mean()
    assert np.array_equal(idx[sure], fx["map"][sure])


def _strict_report():
    """Run in a DN_STRICT_TC=1 subprocess: both spectral projections of the model, forward and backward, under tc3x."""
    fx = load_golden("fmaps_small")
    dn.set_engine("tc3x")
    m = _fixture_model(fx)
    m.train(False)
    res = {}
    try:
        C_pred, _, _ = m(_shape(fx, "x"), _shape(fx, "y"))
        C_pred.square().sum().backward()
        torch.cuda.synchronize()
        res["model"] = "ok"
    except RuntimeError as e:
        res["model"] = "unsupported" if "unsupported" in str(e) else "error: " + str(e)
    s = _shape(fx, "x")
    feat = torch.randn(s[3].shape[0], 128, device="cuda", requires_grad=True)
    for name, k in (("padded", 32), ("unpadded", 30)):
        try:
            basis = torch.zeros(s[6].shape[0], k, device="cuda")
            basis[:, :N] = s[6][:, :N]
            dn.ops.to_basis(feat, basis, s[3]).square().sum().backward()
            torch.cuda.synchronize()
            res[name] = "ok"
        except RuntimeError as e:
            res[name] = "unsupported" if "unsupported" in str(e) else "error: " + str(e)
    print(json.dumps(res))


@gpu
def test_projection_runs_on_tensor_cores_under_strict_tc():
    """The model's only dense projections (to_basis at K = 30 padded to 32, and its backward) stay on the tc3x kernels;
    unpadded K = 30 would not."""
    tests_dir = os.path.join(ROOT, "tests")
    env = dict(os.environ, DN_STRICT_TC="1")
    code = "import sys; sys.path[:0] = [{!r}, {!r}]; import test_gpu_fmaps as t; t._strict_report()".format(tests_dir,
                                                                                                          ROOT)
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    assert got["padded"] == "ok" and got["unpadded"] == "unsupported", got
    assert got["model"] in ("ok", "unsupported"), got      # other layers of the net may take SIMT routes by design


# ---- compute_correspondence --------------------------------------------------------------------------------------
@gpu
def test_compute_correspondence_drop_in():
    V, d = 3000, 128
    g = torch.Generator().manual_seed(2)
    fx_, fy_ = torch.randn(V, d, generator=g), torch.randn(V, d, generator=g)
    etx, ety = torch.randn(N, V, generator=g) / V ** 0.5, torch.randn(N, V, generator=g) / V ** 0.5
    ex, ey = torch.sort(torch.rand(N, generator=g) * 40)[0], torch.sort(torch.rand(N, generator=g) * 40)[0]
    a, b = fx_.cuda().requires_grad_(True), fy_.cuda().requires_grad_(True)
    C = dn.compute_correspondence(a, b, ex.cuda(), ey.cuda(), etx.cuda(), ety.cuda(), lambda_param=LAMBDA)
    assert C.shape == (1, N, N)
    R = torch.randn(1, N, N, generator=g)
    (C * R.cuda()).sum().backward()
    D = torch.float64
    a64, b64 = fx_.to(D).requires_grad_(True), fy_.to(D).requires_grad_(True)
    gold = _torch_solve(etx.to(D) @ a64, ety.to(D) @ b64, ex.to(D), ey.to(D), LAMBDA)
    (gold * R[0].to(D)).sum().backward()
    e = [O.rel_err(C[0].detach().cpu().numpy(), gold.detach().numpy()), O.rel_err(a.grad.cpu().numpy(), a64.grad.numpy()),
         O.rel_err(b.grad.cpu().numpy(), b64.grad.numpy())]
    print("compute_correspondence: C {:.2e}, d feat_x {:.2e}, d feat_y {:.2e}".format(*e))
    assert max(e) <= 1e-4, e


# ---- large V ------------------------------------------------------------------------------------------------------
def _net_fp64(net, x, mass, evals, evecs, gX, gY):
    """dn_oracle_torch's block restatement in float64 on the CPU, through first_lin / blocks / last_lin."""
    D = torch.float64
    sd = {k: v.detach().cpu().to(D) for k, v in net.state_dict().items()}
    h = torch.addmm(sd["first_lin.bias"], x.to(D), sd["first_lin.weight"].t())
    for b in range(net.N_block):
        pre = "block_{}.".format(b)
        bp = {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}
        h = T.block_forward(h[None], mass[None].to(D), evals[None].to(D), evecs[None].to(D), [gX.to(D)], [gY.to(D)],
                            bp)[0]
    return torch.addmm(sd["last_lin.bias"], h, sd["last_lin.weight"].t())


@gpu
def test_large_pair_at_200k():
    torch.manual_seed(0)
    m = dn.FunctionalMapCorrespondenceWithDiffusionNetFeatures(n_feat=128, input_features="xyz").cuda().eval()
    shapes, cpu_ops = [], []
    for seed in (0, 1):
        mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(400, 500, 128, seed=seed, device="cuda")
        x = torch.randn(400 * 500, 3, generator=torch.Generator().manual_seed(10 + seed)).cuda()
        shapes.append([x, None, None, mass, None, evals, evecs, gX, gY, None, None])
        cpu_ops.append((x.cpu(), mass.cpu(), evals.cpu(), evecs.cpu(), gX.cpu(), gY.cpu()))
    C_pred, f1, f2 = m(shapes[0], shapes[1])
    C_pred.square().sum().backward()
    torch.cuda.synchronize()
    assert all(torch.isfinite(p.grad).all() for p in m.parameters())
    feats64 = [_net_fp64(m.feature_extractor, *o) for o in cpu_ops]
    e_feat = max(O.rel_err(f.detach().cpu().numpy(), g.numpy()) for f, g in zip((f1, f2), feats64))
    spec = lambda f, o: OF.spectral(f, o[3].numpy(), o[1].numpy(), N)
    gold = OF.solve(spec(feats64[0].numpy(), cpu_ops[0]), spec(feats64[1].numpy(), cpu_ops[1]),
                    cpu_ops[0][2][:N].numpy(), cpu_ops[1][2][:N].numpy(), LAMBDA)
    # the same solve from OUR fp32 features: what the fp32 feature error alone does to C
    own = OF.solve(spec(f1.detach().cpu().numpy(), cpu_ops[0]), spec(f2.detach().cpu().numpy(), cpu_ops[1]),
                   cpu_ops[0][2][:N].numpy(), cpu_ops[1][2][:N].numpy(), LAMBDA)
    e_c, e_own, e_prop = (O.rel_err(C_pred[0].detach().cpu().numpy(), gold), O.rel_err(C_pred[0].detach().cpu().numpy(), own),
                          O.rel_err(own, gold))
    print("200k pair: features {:.2e}, C vs fp64 {:.2e}, C vs solve of our features {:.2e}, propagated {:.2e}".format(
        e_feat, e_c, e_own, e_prop))
    assert e_feat <= 1e-5
    assert e_own <= 1e-5
    assert e_c <= 1e-5 + 2 * e_prop


# ---- graph capture -----------------------------------------------------------------------------------------------
@gpu
def test_graphed_pair_step_matches_eager_bitwise():
    fx = load_golden("fmaps_small")
    dn.set_engine("tc3x")
    m = _fixture_model(fx)          # eval(): dropout off, GraphedTrainStep's documented limit
    s1, s2 = _shape(fx, "x"), _shape(fx, "y")
    C_gt = torch.from_numpy(fx["C_gt"]).float().cuda()

    def loss_fn(net, a, b, c):
        C_pred, _, _ = net(a, b)
        return torch.mean(torch.square(C_pred.squeeze(0) - c))

    for p in m.parameters():
        p.grad = None
    loss_e = loss_fn(m, s1, s2, C_gt)
    loss_e.backward()
    # keep the value only: the eager graph's gradient accumulators were made on the default stream, and a capture that
    # reused them would make the legacy stream wait on the capturing one
    loss_e = loss_e.detach()
    eager = [p.grad.clone() for p in m.parameters()]
    step = dn.graphs.GraphedTrainStep(m, loss_fn, (s1, s2, C_gt))
    step.zero_grads(m)
    loss_g = step.replay()
    torch.cuda.synchronize()
    assert torch.equal(loss_g, loss_e)
    for g, p in zip(eager, m.parameters()):
        assert torch.equal(g, p.grad)


# ---- nearest neighbour -------------------------------------------------------------------------------------------
def _nn_fp64(source, target, rows=None, chunk=64):
    """fp64 brute force on the device (checker): argmin, best and second-best squared distance of each source row."""
    s = source.to(torch.float64) if rows is None else source[rows].to(torch.float64)
    t = target.to(torch.float64)
    idx, d1, d2 = [], [], []
    for a in range(0, s.shape[0], chunk):
        q = s[a:a + chunk]
        d = torch.zeros(q.shape[0], t.shape[0], dtype=torch.float64, device=t.device)
        for k in range(s.shape[1]):
            d += (q[:, k:k + 1] - t[:, k][None, :]) ** 2
        v, i = torch.topk(d, 2, dim=1, largest=False, sorted=True)
        idx.append(i[:, 0])
        d1.append(v[:, 0])
        d2.append(v[:, 1])
    return torch.cat(idx), torch.cat(d1), torch.cat(d2)


def _check_nn(idx, source, target, rows, n, chunk=64):
    gi, d1, d2 = _nn_fp64(source, target, rows, chunk=chunk)
    tau = (n + 2) * U32 / (1 - (n + 2) * U32)
    lim = d1 * (1 + tau) / (1 - tau)
    q = source.to(torch.float64) if rows is None else source[rows].to(torch.float64)
    mine = idx if rows is None else idx[rows]
    dm = ((q - target[mine].to(torch.float64)) ** 2).sum(1)
    assert bool((dm <= lim).all()), float((dm - lim).max())
    sure = d2 > lim
    assert bool((mine[sure] == gi[sure]).all()), int((mine[sure] != gi[sure]).sum())
    return float(sure.float().mean())


@gpu
@pytest.mark.parametrize("n", [3, 30, 128])
def test_nearest_neighbor_5k_full(n):
    g = torch.Generator().manual_seed(n)
    src, tgt = torch.randn(5000, n, generator=g).cuda(), torch.randn(5000, n, generator=g).cuda()
    idx = dn.fmaps.nearest_neighbor(src, tgt)
    assert idx.dtype == torch.int64 and idx.shape == (5000,)
    frac = _check_nn(idx, src, tgt, None, n)
    assert frac > 0.99
    assert torch.equal(idx, dn.fmaps.nearest_neighbor(src, tgt))


@gpu
@pytest.mark.parametrize("n", [3, 30, 128])
def test_nearest_neighbor_200k_sampled(n):
    g = torch.Generator().manual_seed(100 + n)
    V = 200_000
    src, tgt = torch.randn(V, n, generator=g).cuda(), torch.randn(V, n, generator=g).cuda()
    idx = dn.fmaps.nearest_neighbor(src, tgt)
    rows = torch.randperm(V, generator=g)[:2000].cuda()
    frac = _check_nn(idx, src, tgt, rows, n)
    assert frac > 0.99


@gpu
@pytest.mark.parametrize("Vs", [50, 5000])
def test_nearest_neighbor_duplicates_take_lowest_index(Vs):
    """Duplicated target rows, far apart (so that a split search sees them in different ranges when Vs is small)."""
    g = torch.Generator().manual_seed(Vs)
    n, Vt = 30, 20000
    tgt = torch.randn(Vt, n, generator=g)
    for lo, hi in ((5, Vt - 5), (7, 11), (300, 12000)):
        tgt[hi] = tgt[lo]
    src = torch.randn(Vs, n, generator=g)
    src[0], src[1], src[2] = tgt[Vt - 5], tgt[11], tgt[12000]
    idx = dn.fmaps.nearest_neighbor(src.cuda(), tgt.cuda()).cpu()
    assert idx[:3].tolist() == [5, 7, 300]


@gpu
def test_refusals():
    A = torch.randn(8, 16)
    e = torch.arange(8, dtype=torch.float32)
    with pytest.raises(RuntimeError):
        dn.fmaps.fmap_solve(A, A, e, e)
    with pytest.raises(RuntimeError):
        dn.fmaps.nearest_neighbor(A, A)
    with pytest.raises(RuntimeError):
        dn.compute_correspondence(A, A, e, e, torch.randn(8, 8), torch.randn(8, 8))
    Ab = torch.randn(129, 16, device="cuda")
    eb = torch.arange(129, dtype=torch.float32, device="cuda")
    with pytest.raises(RuntimeError, match="128"):
        dn.fmaps.fmap_solve(Ab, Ab, eb, eb)
    with pytest.raises(RuntimeError, match="128"):
        dn.fmaps.nearest_neighbor(torch.randn(10, 129, device="cuda"), torch.randn(10, 129, device="cuda"))
    Ac = A.cuda()
    with pytest.raises(ValueError):
        dn.fmaps.fmap_solve(Ac, Ac[:, :8], e.cuda(), e.cuda())
    with pytest.raises(ValueError):
        dn.fmaps.fmap_solve(Ac, Ac, e[:4].cuda(), e.cuda())
    with pytest.raises(ValueError):
        dn.fmaps.nearest_neighbor(torch.randn(10, 3, device="cuda"), torch.randn(10, 4, device="cuda"))
    with pytest.raises(ValueError):
        dn.compute_correspondence(torch.randn(20, 16, device="cuda"), torch.randn(20, 16, device="cuda"), e.cuda(),
                                  e[:4].cuda(), torch.randn(8, 20, device="cuda"), torch.randn(8, 20, device="cuda"))
    with pytest.raises(ValueError):
        dn.pointwise_map(torch.randn(1, 8, 8, device="cuda"), torch.randn(20, 8, device="cuda"),
                         torch.randn(20, 8, device="cuda"), n_fmap=30)
    # the C-ABI itself refuses n > 128 before enqueuing anything
    assert dn._lib.load().dn_fmap_solve_fwd(Ab.data_ptr(), Ab.data_ptr(), eb.data_ptr(), eb.data_ptr(), 129, 16, 1e-3,
                                            Ab.data_ptr(), None) == -2
