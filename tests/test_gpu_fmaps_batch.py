"""The functional-map head over a pair batch (diffusion_net_b200/fmaps.py: PairBatch, project_batched,
fmap_solve_batched, forward_pairs, pointwise_map_batch) against the per-pair calls and fp64 golds.

Bounds (u = 2^-24, eps = 2^-53):
  * solve: each pair's C is bitwise the per-pair ``fmap_solve``; against fp64 the per-row bound of test_gpu_fmaps.py,
    (u + 16 n (n + d) kappa(S_i) eps) max_j |C_gold[i][j]|.  The per-shape gradient is bitwise the per-pair
    ``dn_fmap_solve_bwd`` outputs summed in fp32 in the stated order; against fp64 each summand carries test_gpu_fmaps.py's
    relative error tol = 4u + 16 n (n + d) kappa_max eps of its own magnitude, and each of the m additions one more u of
    the running sum: |ours - gold| <= (tol + m u) sum_p max|g_p|, normalised by max|gold| as rel_err is.
  * projection: test_gpu_to_basis.py's componentwise tc3x bound, 2^-13 sum_v |Phi[v][k] m[v] x[v][c]|; the adjoint
    m[v] sum_k Phi[v][k] G[k][c] runs on the 3xTF32 from_basis chain, bounded the same way over its K terms.
  * model: the fixture's existing C tolerance max(1e-5, 4 err32:C) for pair (x, y), and its gradient bound
    max(5e-5, 4 gradfloor:k) scaled by the 4 pairs of the loss (each pair's backward contributes its own fp32 floor).
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
TB_TOL = 2.0 ** -13


def _launches():
    return dn._lib.load().dn_kernel_launch_count()


def model_torch_pairs(params, shapes, pairs, n=30, lam=1e-3):
    """fp64 gold of a pair batch: ``dn_oracle_fmaps.model_torch`` (fmaps_model.py:62-83) for every pair (x, y) of
    ``pairs``, indices into ``shapes`` (each ``(x, mass, evals, evecs, gradX, gradY)``), with each shape's features
    computed once, as ``forward_pairs`` runs them.  Returns (C (P, n, n), feats), feats the per-shape feature list;
    float64 torch on the CPU, differentiable in ``params``."""
    pre = "feature_extractor."
    p = {k[len(pre):]: v for k, v in params.items() if k.startswith(pre)}
    n_block = len([k for k in p if k.endswith("diffusion.diffusion_time")])
    feats, specs = [], []
    for x, mass, evals, evecs, gX, gY in shapes:
        h = torch.addmm(p["first_lin.bias"], x, p["first_lin.weight"].t())
        for b in range(n_block):
            bp = {k[len("block_%d." % b):]: v for k, v in p.items() if k.startswith("block_%d." % b)}
            h = T.block_forward(h[None], mass[None], evals[None], evecs[None], [gX], [gY], bp)[0]
        f = torch.addmm(p["last_lin.bias"], h, p["last_lin.weight"].t())
        feats.append(f)
        specs.append(evecs[:, :n].t() @ (mass[:, None] * f))
    Cs = []
    for a, b in pairs:
        A, B = specs[a], specs[b]
        ex, ey = shapes[a][2][:n], shapes[b][2][:n]
        D = (ex[None, :] - ey[:, None]) ** 2
        AAt, BAt = A @ A.t(), B @ A.t()
        Cs.append(torch.stack([torch.linalg.solve(AAt + lam * torch.diag(D[i]), BAt[i]) for i in range(n)]))
    return torch.stack(Cs), feats


# ---- host -----------------------------------------------------------------------------------------------------------
def test_role_csr_self_pairs_repeats_and_unused_shape():
    pairs = [(0, 1), (1, 0), (2, 2), (0, 1), (1, 2)]
    begin, ent = dn.fmaps.role_csr(pairs, 4)
    assert begin == [0, 3, 7, 10, 10]
    assert ent[0:3] == [0, 3, 6]                  # shape 0: x of pairs 0, 3; y of pair 1
    assert ent[3:7] == [1, 2, 7, 8]               # shape 1: y of 0, x of 1, y of 3, x of 4
    assert ent[7:10] == [4, 5, 9]                 # shape 2: x then y of the self-pair 2, y of 4
    assert begin[4] - begin[3] == 0               # shape 3 is in no pair


def _cpu_item(V=40, K=32):
    return {"mass": torch.ones(V), "evals": torch.arange(K, dtype=torch.float32), "evecs": torch.zeros(V, K),
            "gradX": None, "gradY": None}


def test_pair_batch_refusals():
    items = [_cpu_item(), _cpu_item()]
    with pytest.raises(ValueError, match="at least one pair"):
        dn.PairBatch(items, [])
    with pytest.raises(ValueError, match=r"pair 1 = \(0, 2\) indexes a shape outside \[0, 2\)"):
        dn.PairBatch(items, [(0, 1), (0, 2)])
    with pytest.raises(ValueError, match="outside"):
        dn.PairBatch(items, [(-1, 0)])
    with pytest.raises(ValueError, match="K = 32 eigenpairs is fewer than n_fmap = 40"):
        dn.PairBatch(items, [(0, 1)], n_fmap=40)
    with pytest.raises(RuntimeError, match="n = 129 exceeds the supported maximum of 128"):
        dn.PairBatch([_cpu_item(K=160)] * 2, [(0, 1)], n_fmap=129)
    with pytest.raises(ValueError, match="1025 shapes exceed the 1024"):
        dn.PairBatch([_cpu_item()] * 1025, [(0, 1)])
    with pytest.raises(ValueError, match="at most 65535 pairs"):
        dn.fmaps.PairList([(0, 0)] * 65536, 1, "cpu")
    with pytest.raises(ValueError, match=r"pair 0 = \(0, 3\)"):
        dn.fmaps.PairList([(0, 3)], 3, "cpu")


def _fixture_shapes64(fx):
    d = torch.float64

    def shape(tag):
        f = lambda k: torch.from_numpy(np.asarray(fx[tag + ":" + k]))
        V = f("mass").shape[0]
        sp = lambda i, v: torch.sparse_coo_tensor(f(i), f(v).to(d), (V, V)).coalesce()
        return (f("verts").to(d), f("mass").to(d), f("evals").to(d), f("evecs").to(d), sp("gradX_idx", "gradX_vals"),
                sp("gradY_idx", "gradY_vals"))
    return [shape("x"), shape("y")]


def test_model_torch_pairs_matches_per_pair_loop():
    fx = load_golden("fmaps_small")
    params = {k[2:]: torch.from_numpy(v.astype(np.float64)) for k, v in fx.items() if k.startswith("p:")}
    shapes = _fixture_shapes64(fx)
    pairs = [(0, 1), (1, 0), (0, 0), (1, 1)]
    C, feats = model_torch_pairs(params, shapes, pairs, n=N, lam=LAMBDA)
    assert C.shape == (4, N, N) and len(feats) == 2
    for p, (a, b) in enumerate(pairs):
        Cl, fa, fb = OF.model_torch(params, shapes[a], shapes[b], n=N, lam=LAMBDA)
        assert O.rel_err(C[p].numpy(), Cl.numpy()) <= 1e-12
        assert O.rel_err(feats[a].numpy(), fa.numpy()) <= 1e-12 and O.rel_err(feats[b].numpy(), fb.numpy()) <= 1e-12


@pytest.mark.skipif(shutil.which(NVCC) is None and not os.path.exists(NVCC), reason="nvcc not found")
def test_fmap_batch_kernels_and_partial_reduction_do_not_spill(tmp_path):
    """The pair-batch kernels, the single-pair kernels whose bodies they share, and the split-V partial reduction that
    sums each mesh's to_basis partials (one kernel for single meshes and mesh batches)."""
    flags = [f for f in dn._lib.NVCC_FLAGS if f != "-shared"]
    expect = {"dn_fmap_batch.cu": 16, "dn_fmap.cu": 9, "dn_simt.cu": None}
    for src, count in expect.items():
        cmd = [NVCC] + flags + ["-Xptxas", "-v", "-c", os.path.join(dn._lib._CSRC, src), "-o", str(tmp_path / "x.o")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        out = (r.stdout + r.stderr).splitlines()
        pairs = []
        for i, l in enumerate(out):
            if "Compiling entry function" in l:
                nxt = [x for x in out[i + 1:i + 4] if "spill stores" in x]
                assert nxt, (src, l)
                pairs.append((l, nxt[0]))
        if count is None:
            pairs = [p for p in pairs if "reduce_partials_kernel" in p[0]]
            assert len(pairs) == 1, src
        else:
            assert len(pairs) == count, (src, len(pairs))
        for name, l in pairs:
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", l)
            assert m and m.group(1) == "0" and m.group(2) == "0", (name, l)


# ---- solve ----------------------------------------------------------------------------------------------------------
SOLVE_PAIRS = [(0, 1), (1, 0), (0, 0), (2, 1), (0, 1), (1, 2), (2, 2)]   # shape 3 is in no pair


def _stack_inputs(S, n, d, seed):
    rs = np.random.RandomState(seed)
    F = rs.randn(S, n, d).astype(np.float32)
    ev = np.sort(rs.rand(S, n) * 40, axis=1).astype(np.float32)
    ev[1, 0] = ev[0, 0]
    return F, ev


def _kappa(A, ex, ey, lam):
    A = A.astype(np.float64)
    D = (ex.astype(np.float64)[None, :] - ey.astype(np.float64)[:, None]) ** 2
    return np.array([np.linalg.cond(A @ A.T + lam * np.diag(D[i])) for i in range(A.shape[0])])


@gpu
@pytest.mark.parametrize("n", [1, 8, 30, 128])
@pytest.mark.parametrize("d", [16, 128, 200])
def test_solve_batched_matches_per_pair_bitwise_and_fp64(n, d):
    S, pairs = 4, SOLVE_PAIRS
    P = len(pairs)
    F, ev = _stack_inputs(S, n, d, seed=n * 1000 + d)
    Ft, evt = torch.from_numpy(F).cuda().requires_grad_(True), torch.from_numpy(ev).cuda()
    pl = dn.fmaps.PairList(pairs, S, "cuda")
    C = dn.fmaps.fmap_solve_batched(Ft, evt, pl, n, LAMBDA)
    g = torch.from_numpy(np.random.RandomState(7).randn(P, n, n).astype(np.float32)).cuda()
    (C * g).sum().backward()
    C2 = dn.fmaps.fmap_solve_batched(Ft.detach(), evt, pl, n, LAMBDA)
    assert torch.equal(C.detach(), C2)
    acc = [torch.zeros(n, d, device="cuda") for _ in range(S)]
    fp64_term = 16 * n * (n + d) * EPS64
    gold_acc = [np.zeros((n, d)) for _ in range(S)]
    mag = [0.0] * S
    terms = [0] * S
    kmax = 0.0
    for p, (a, b) in enumerate(pairs):
        A = Ft.detach()[a].clone().requires_grad_(True)
        B = Ft.detach()[b].clone().requires_grad_(True)
        Cp = dn.fmaps.FmapSolveFn.apply(A, B, evt[a], evt[b], LAMBDA)
        assert torch.equal(Cp.detach(), C[p].detach()), p
        Cp.backward(g[p])
        acc[a] = acc[a] + A.grad            # role x before role y, increasing p
        acc[b] = acc[b] + B.grad
        gold = OF.solve(F[a], F[b], ev[a], ev[b], LAMBDA)
        kap = _kappa(F[a], ev[a], ev[b], LAMBDA)
        kmax = max(kmax, kap.max())
        Cn = C[p].detach().cpu().numpy().astype(np.float64)
        for i in range(n):
            scale = np.abs(gold[i]).max()
            assert np.abs(Cn[i] - gold[i]).max() <= (U32 + fp64_term * kap[i]) * scale, (p, i)
        dA, dB = OF.solve_adjoint(F[a], F[b], ev[a], ev[b], LAMBDA, g[p].cpu().numpy())
        gold_acc[a] += dA
        gold_acc[b] += dB
        mag[a] += np.abs(dA).max()
        mag[b] += np.abs(dB).max()
        terms[a] += 1
        terms[b] += 1
    grad = Ft.grad
    for s in range(S):
        assert torch.equal(grad[s], acc[s]), s
    assert bool((grad[3] == 0).all())
    tol = 4 * U32 + fp64_term * kmax
    for s in range(3):
        err = np.abs(grad[s].cpu().numpy() - gold_acc[s]).max()
        assert err <= (tol + terms[s] * U32) * mag[s], (s, err / mag[s], tol)


@gpu
def test_solve_batched_singular_row_stays_in_its_pair_and_runs_without_sync():
    n, d, S = 8, 16, 3
    F, ev = _stack_inputs(S, n, d, seed=11)
    F[0, 3] = 0.0                       # shape 0's A A^T has a zero row / column 3 ...
    ev[1, 5] = ev[0, 3]                 # ... and row 5 of pair (0, 1) has no regulariser there
    Ft, evt = torch.from_numpy(F).cuda(), torch.from_numpy(ev).cuda()
    pl = dn.fmaps.PairList([(1, 2), (0, 1), (2, 0)], S, "cuda")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        C = dn.fmaps.fmap_solve_batched(Ft, evt, pl, n, LAMBDA)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    Cn = C.cpu().numpy()
    bad = ~np.isfinite(Cn).all(axis=2)
    assert bad[1].tolist() == [i == 5 for i in range(n)] and np.isnan(Cn[1, 5]).all()
    assert not bad[0].any() and not bad[2].any()


@gpu
def test_solve_batched_launch_counts_do_not_depend_on_pairs():
    n, d, S = N, 128, 6
    F, ev = _stack_inputs(S, n, d, seed=5)
    counts = []
    for P in (2, 64):
        pairs = [(p % S, (3 * p + 1) % S) for p in range(P)]
        pl = dn.fmaps.PairList(pairs, S, "cuda")
        Ft = torch.from_numpy(F).cuda().requires_grad_(True)
        torch.cuda.synchronize()
        n0 = _launches()
        C = dn.fmaps.fmap_solve_batched(Ft, torch.from_numpy(ev).cuda(), pl, n, LAMBDA)
        n1 = _launches()
        C.square().sum().backward()
        torch.cuda.synchronize()
        counts.append((n1 - n0, _launches() - n1))
    assert counts[0] == counts[1] and counts[0][0] == 1 and counts[0][1] <= 3, counts


# ---- projection -----------------------------------------------------------------------------------------------------
RAGGED = [(5, 10), (1, 127), (8, 16), (3, 43), (50, 100)]    # V = 50, 127, 128, 129, 5000


def _synthetic_items(shapes, K, seed0=0):
    items = []
    for i, (a, b) in enumerate(shapes):
        mass, _, evals, evecs, gX, gY = dn.synthetic.structural_operators(a, b, K, seed=seed0 + i, device="cuda")
        items.append({"mass": mass, "evals": evals, "evecs": evecs, "gradX": gX, "gradY": gY})
    return items


def _projection_pb(shapes=RAGGED, K=48):
    items = _synthetic_items(shapes, K)
    return dn.PairBatch(items, [(0, 1)], n_fmap=N), items


@gpu
def test_projection_forward_and_adjoint_against_fp64():
    dn.set_engine("tc3x")
    pb, items = _projection_pb()
    mb = pb.mesh_batch
    Cc = 128
    g = torch.Generator().manual_seed(3)
    xs = [torch.randn(it["mass"].shape[0], Cc, generator=g) for it in items]
    feat = mb.pack([x.cuda() for x in xs]).requires_grad_(True)
    out = dn.fmaps.project_batched(feat, pb)
    assert out.shape == (len(items), pb.kp, Cc)
    G = torch.randn(len(items), pb.kp, Cc, generator=g)
    out.backward(G.cuda())
    grad = feat.grad.cpu().double().numpy()
    for s, (it, x) in enumerate(zip(items, xs)):
        phi = np.zeros((x.shape[0], pb.kp))
        phi[:, :N] = it["evecs"][:, :N].cpu().double().numpy()
        m = it["mass"].cpu().double().numpy()
        xd = x.double().numpy() * m[:, None]
        gold, absum = phi.T @ xd, np.abs(phi).T @ np.abs(xd)
        err = np.abs(out[s].detach().cpu().double().numpy() - gold)
        assert (err <= TB_TOL * absum + 1e-30).all(), (s, (err / (TB_TOL * absum + 1e-30)).max())
        Gd = G[s].double().numpy()
        gold_b, absum_b = m[:, None] * (phi @ Gd), m[:, None] * (np.abs(phi) @ np.abs(Gd))
        r0 = mb.row_begin[s]
        err_b = np.abs(grad[r0:r0 + x.shape[0]] - gold_b)
        assert (err_b <= TB_TOL * absum_b + 1e-30).all(), (s, (err_b / (TB_TOL * absum_b + 1e-30)).max())
        pad_end = mb.row_begin[s + 1]
        assert (grad[r0 + x.shape[0]:pad_end] == 0).all(), s
    assert (out[:, N:].detach() == 0).all()


@gpu
def test_projection_launch_counts_do_not_depend_on_shapes():
    dn.set_engine("tc3x")
    counts = []
    for shapes in (RAGGED[:2], RAGGED * 3):
        pb, _ = _projection_pb(shapes)
        feat = torch.randn(pb.mesh_batch.V, 128, device="cuda", requires_grad=True)
        torch.cuda.synchronize()
        n0 = _launches()
        out = dn.fmaps.project_batched(feat, pb)
        n1 = _launches()
        out.square().sum().backward()
        torch.cuda.synchronize()
        counts.append((n1 - n0, _launches() - n1))
    assert counts[0] == counts[1] == (2, 2), counts


@gpu
def test_projection_refuses_simt():
    pb, _ = _projection_pb(RAGGED[:2])
    feat = torch.randn(pb.mesh_batch.V, 128, device="cuda")
    dn.set_engine("simt")
    try:
        with pytest.raises(RuntimeError, match="unsupported"):
            dn.fmaps.project_batched(feat, pb)
        with pytest.raises(RuntimeError, match="unsupported"):
            dn.fmaps.ProjectBatchedFn.backward(type("Ctx", (), {"pb": pb})(),
                                               torch.randn(2, pb.kp, 128, device="cuda"))
    finally:
        dn.set_engine("tc3x")


def _strict_report():
    """Run in a DN_STRICT_TC=1 subprocess: both directions of the batched projection under tc3x."""
    dn.set_engine("tc3x")
    pb, _ = _projection_pb(RAGGED[:3])
    feat = torch.randn(pb.mesh_batch.V, 128, device="cuda", requires_grad=True)
    try:
        dn.fmaps.project_batched(feat, pb).square().sum().backward()
        torch.cuda.synchronize()
        res = "ok"
    except RuntimeError as e:
        res = "error: " + str(e)
    print(json.dumps({"projection": res}))


@gpu
def test_projection_stays_on_tensor_cores_under_strict_tc():
    tests_dir = os.path.join(ROOT, "tests")
    env = dict(os.environ, DN_STRICT_TC="1")
    code = "import sys; sys.path[:0] = [{!r}, {!r}]; import test_gpu_fmaps_batch as t; t._strict_report()".format(
        tests_dir, ROOT)
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    assert json.loads(r.stdout.strip().splitlines()[-1]) == {"projection": "ok"}
    assert "outside the tensor-core kernels' envelope" not in r.stderr


# ---- model ----------------------------------------------------------------------------------------------------------
def _fixture_items(fx):
    items, xs = [], []
    for tag in ("x", "y"):
        f = lambda k: torch.from_numpy(np.ascontiguousarray(fx[tag + ":" + k])).cuda()
        V = f("mass").shape[0]
        gX = torch.sparse_coo_tensor(f("gradX_idx"), f("gradX_vals"), (V, V)).coalesce()
        gY = torch.sparse_coo_tensor(f("gradY_idx"), f("gradY_vals"), (V, V)).coalesce()
        items.append({"mass": f("mass"), "evals": f("evals"), "evecs": f("evecs"), "gradX": gX, "gradY": gY,
                      "faces": f("faces")})
        xs.append(f("verts"))
    return items, xs


def _fixture_model(fx):
    m = dn.FunctionalMapCorrespondenceWithDiffusionNetFeatures(n_feat=128, input_features="xyz")
    sd = {k[2:]: torch.from_numpy(v.astype(np.float32)) for k, v in fx.items() if k.startswith("p:")}
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


@gpu
def test_fixture_pairs_match_fp64_gold_with_gradients():
    fx = load_golden("fmaps_small")
    dn.set_engine("tc3x")
    m = _fixture_model(fx)
    items, xs = _fixture_items(fx)
    pairs = [(0, 1), (1, 0), (0, 0), (1, 1)]
    pb = dn.PairBatch(items, pairs)
    C_pred, feats = m.forward_pairs(pb, xs)
    assert C_pred.shape == (4, N, N) and len(feats) == 2
    tol_c = max(1e-5, 4 * float(fx["err32:C"]))
    assert O.rel_err(C_pred[0].detach().cpu().numpy(), fx["C64"]) <= tol_c
    params = {k[2:]: torch.from_numpy(v.astype(np.float64)).requires_grad_(True) for k, v in fx.items()
              if k.startswith("p:")}
    C64, f64 = model_torch_pairs(params, _fixture_shapes64(fx), pairs, n=N, lam=LAMBDA)
    for p in range(4):
        e = O.rel_err(C_pred[p].detach().cpu().numpy(), C64[p].detach().numpy())
        print("pair {}: C {:.2e} (tol {:.2e})".format(pairs[p], e, tol_c))
        assert e <= tol_c, (p, e)
    for s in range(2):
        assert O.rel_err(feats[s].detach().cpu().numpy(), f64[s].detach().numpy()) <= max(
            1e-5, 4 * float(fx["err32:feat%d" % (s + 1)]))
    C_gt = torch.from_numpy(fx["C_gt"])
    G64 = torch.stack([2 * (C64[p].detach() - C_gt) / N ** 2 for p in range(4)])
    (C64 * G64).sum().backward()
    (C_pred * G64.float().cuda()).sum().backward()
    worst = 0.0
    for k, prm in m.named_parameters():
        e = O.rel_err(prm.grad.cpu().numpy(), params[k].grad.numpy())
        worst = max(worst, e)
        assert e <= 4 * max(5e-5, 4 * float(fx["gradfloor:" + k])), (k, e)
    print("fixture pair batch parameter gradients: worst {:.2e}".format(worst))


def _ragged_model_setup(shapes, pairs, seed=0):
    torch.manual_seed(seed)
    m = dn.FunctionalMapCorrespondenceWithDiffusionNetFeatures(n_feat=128, input_features="xyz").cuda().eval()
    items = _synthetic_items(shapes, 64, seed0=20)
    g = torch.Generator().manual_seed(seed + 1)
    xs = [torch.randn(it["mass"].shape[0], 3, generator=g).cuda() for it in items]
    return m, items, xs, dn.PairBatch(items, pairs)


RAGGED_MODEL = [(10, 30), (13, 41), (20, 50), (8, 64), (31, 33)]
RAGGED_PAIRS = [(0, 1), (1, 2), (2, 0), (3, 3), (4, 1), (1, 4), (0, 1), (2, 3), (3, 0), (4, 4)]


@gpu
def test_ragged_pairs_agree_with_per_pair_forward():
    dn.set_engine("tc3x")
    m, items, xs, pb = _ragged_model_setup(RAGGED_MODEL, RAGGED_PAIRS)
    with torch.no_grad():
        C_pred, feats = m.forward_pairs(pb, xs)
    sh = lambda s: [xs[s], None, None, items[s]["mass"], None, items[s]["evals"], items[s]["evecs"], items[s]["gradX"],
                    items[s]["gradY"], None, None]
    worst_c, worst_f = 0.0, 0.0
    for p, (a, b) in enumerate(RAGGED_PAIRS):
        with torch.no_grad():
            C1, f1, f2 = m(sh(a), sh(b))
        worst_f = max(worst_f, O.rel_err(feats[a].cpu().numpy(), f1.cpu().numpy()),
                      O.rel_err(feats[b].cpu().numpy(), f2.cpu().numpy()))
        # what the features' own fp32 difference does to C: the solve of the per-pair features, bitwise the per-pair C
        worst_c = max(worst_c, O.rel_err(C_pred[p].cpu().numpy(), C1[0].cpu().numpy()))
    print("ragged pairs: features {:.2e}, C {:.2e}".format(worst_f, worst_c))
    assert worst_f <= 1e-5
    assert worst_c <= 1e-3


@gpu
def test_graphed_pair_batch_step_matches_eager_bitwise_and_launches_do_not_depend_on_pairs():
    dn.set_engine("tc3x")
    m, items, xs, pb = _ragged_model_setup(RAGGED_MODEL[:3], [(0, 1), (2, 1)])
    C_gt = torch.randn(N, N, generator=torch.Generator().manual_seed(4)).cuda() * 0.1

    def loss_fn(net, pair_batch, inputs, c):
        C_pred, _ = net.forward_pairs(pair_batch, inputs)
        return torch.mean(torch.square(C_pred - c))

    counts = []
    for pairs in ([(0, 1), (2, 1)], [(i % 3, (i * 2 + 1) % 3) for i in range(12)]):
        pbp = dn.PairBatch(items, pairs)
        loss_fn(m, pbp, xs, C_gt).backward()          # warm caches
        torch.cuda.synchronize()
        n0 = _launches()
        loss_fn(m, pbp, xs, C_gt).backward()
        torch.cuda.synchronize()
        counts.append(_launches() - n0)
    assert counts[0] == counts[1], counts
    for p in m.parameters():
        p.grad = None
    loss_e = loss_fn(m, pb, xs, C_gt)
    loss_e.backward()
    loss_e = loss_e.detach()
    eager = [p.grad.clone() for p in m.parameters()]
    step = dn.graphs.GraphedTrainStep(m, loss_fn, (pb, xs, C_gt))
    step.zero_grads(m)
    loss_g = step.replay()
    torch.cuda.synchronize()
    assert torch.equal(loss_g, loss_e)
    for g, p in zip(eager, m.parameters()):
        assert torch.equal(g, p.grad)


# ---- pointwise maps -------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("n", [3, 30, 128])
def test_pointwise_map_batch_bitwise_per_pair(n):
    shapes = [(10, 20), (13, 31), (40, 75), (16, 16)]
    items = _synthetic_items(shapes, 128, seed0=50)
    # duplicate rows inside a shape: ties in the target must go to the lowest index
    ev = items[2]["evecs"]
    ev[2000] = ev[7]
    ev[2999] = ev[300]
    items[0]["evecs"][150] = items[0]["evecs"][3]
    pairs = [(0, 1), (1, 0), (2, 2), (2, 0), (3, 2), (0, 0), (1, 3)]
    pb = dn.PairBatch(items, pairs, n_fmap=n)
    g = torch.Generator().manual_seed(n)
    C = (torch.randn(len(pairs), n, n, generator=g) / n ** 0.5).cuda()
    maps = dn.pointwise_map_batch(C, pb, n_fmap=n)
    assert len(maps) == len(pairs)
    for p, (a, b) in enumerate(pairs):
        ref = dn.pointwise_map(C[p], items[a]["evecs"], items[b]["evecs"], n_fmap=n)
        assert maps[p].dtype == torch.int64 and torch.equal(maps[p], ref), p
    assert torch.equal(torch.cat(maps), torch.cat(dn.pointwise_map_batch(C, pb, n_fmap=n)))


@gpu
def test_pointwise_map_batch_launch_count_does_not_depend_on_pairs():
    items = _synthetic_items([(10, 20), (13, 31), (20, 50)], 64, seed0=60)
    counts = []
    for P in (2, 12):
        pairs = [(p % 3, (p + 1) % 3) for p in range(P)]
        pb = dn.PairBatch(items, pairs)
        C = torch.randn(P, N, N, generator=torch.Generator().manual_seed(P)).cuda()
        dn.pointwise_map_batch(C, pb)
        torch.cuda.synchronize()
        n0 = _launches()
        dn.pointwise_map_batch(C, pb)
        torch.cuda.synchronize()
        counts.append(_launches() - n0)
    assert counts[0] == counts[1] and counts[0] <= 3, counts
