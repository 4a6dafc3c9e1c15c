"""Shuffled shape pairs of a device-resident dataset (fmaps.PairDataset / PairSlot): the ground-truth functional maps
(dn_fmap_ground_truth) against an fp64 numpy restatement of faust_scape_dataset.py:186-190, the per-mesh rotations
(dn_rotate_rows, batch.random_rotations), and the pair slot's training step against the eager pair-batch routes and
in a CUDA graph.

Bounds: the ground truth is an fp64 solve of the normal equations on the exactly promoted fp32 rows, so against
``np.linalg.lstsq`` it differs by the fp64 error kappa(A)^2 eps (kappa(A) < 1e3 here) plus the fp32 rounding of the
output: max|delta| / max|gold| <= 1e-5.  A rotated row is three fp32 products summed, within 2 u of the fp64 value
per unit of |x| |R| (1e-6 here)."""
import copy
import itertools
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import diffusion_net_b200 as dn

gpu = pytest.mark.gpu
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def test_new_kernels_do_not_spill(tmp_path):
    if shutil.which(NVCC) is None and not os.path.exists(NVCC):
        pytest.skip("needs nvcc")
    flags = [f for f in dn._lib.NVCC_FLAGS if f != "-shared"]
    seen = {}
    for src, names in (("dn_fmap_gt.cu", ("gt_partial_kernel", "gt_solve_kernel")),
                       ("dn_batch_rotate.cu", ("rotate_rows_kernel",))):
        cmd = [NVCC] + flags + ["-Xptxas", "-v", "-c", os.path.join(dn._lib._CSRC, src), "-o", str(tmp_path / "x.o")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        cur = None
        for line in (r.stdout + r.stderr).splitlines():
            m = re.search(r"Compiling entry function '(\w+)'", line)
            if m:
                cur = next((n for n in names if n in m.group(1)), None)
            elif cur and "spill stores" in line:
                seen[cur] = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                                      line).groups()
    assert set(seen) == {"gt_partial_kernel", "gt_solve_kernel", "rotate_rows_kernel"}, seen
    assert all(v == ("0", "0", "0") for v in seen.values()), seen


# ---- helpers -------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    dn._lib.load()
    dn.set_engine("tc3x")
    yield torch.device("cuda")
    dn.set_engine("tc3x")


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int32 if t.dtype == torch.float32 else t.dtype)


def _eq(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def _items(shapes, K, seed0=0):
    items = []
    for i, (a, b) in enumerate(shapes):
        mass, _, evals, evecs, gX, gY = dn.synthetic.structural_operators(a, b, K, seed=seed0 + i, device="cuda")
        items.append({"mass": mass, "evals": evals, "evecs": evecs, "gradX": gX, "gradY": gY})
    return items


def _vts(items, ms, seed=0, distinct=None):
    """Random correspondences with repeats: m_s vertices of mesh s drawn with replacement (from its first
    ``distinct[s]`` vertices when given)."""
    rs = np.random.RandomState(seed)
    out = []
    for s, (it, m) in enumerate(zip(items, ms)):
        hi = it["mass"].shape[0] if distinct is None or distinct[s] is None else distinct[s]
        out.append(torch.from_numpy(rs.randint(0, hi, m).astype(np.int64)))
    return out


def _gold_gt(items, vts, a, b, n):
    """faust_scape_dataset.py:186-190 in fp64 numpy: C_gt = lstsq(Phi_x[vts_x, :n], Phi_y[vts_y, :n]).T"""
    A = items[a]["evecs"].cpu().numpy().astype(np.float64)[vts[a].numpy(), :n]
    B = items[b]["evecs"].cpu().numpy().astype(np.float64)[vts[b].numpy(), :n]
    return np.linalg.lstsq(A, B, rcond=None)[0].T


# ---- ground truth ----------------------------------------------------------------------------------------------------------
GT_SHAPES = [(12, 15), (12, 12), (20, 30), (24, 25), (50, 100), (40, 120)]     # 144 .. 5000 vertices
GT_M = [40, 40, 700, 700, 7000, 7000]                                         # m = 40 .. 7000, with repeats


@gpu
@pytest.mark.parametrize("K,n", [(32, 8), (32, 30), (128, 8), (128, 30)])
def test_ground_truth_matches_lstsq_and_is_bitwise_independent_of_the_draw(cuda, K, n):
    items = _items(GT_SHAPES, K, seed0=K + n)
    vts = _vts(items, GT_M, seed=n)
    ds = dn.MeshDataset(items)
    pairs = [(a, b) for g in ((0, 1), (2, 3), (4, 5)) for a, b in itertools.product(g, g)]
    pds = dn.PairDataset(ds, vts, pairs, n_fmap=n)
    assert pds.max_m == 7000
    C = pds.ground_truth(list(range(len(pairs))))
    worst = 0.0
    for p, (a, b) in enumerate(pairs):
        e = _rel(C[p].cpu().numpy(), _gold_gt(items, vts, a, b, n))
        worst = max(worst, e)
        assert e <= 1e-5, (p, a, b, e)
    print(json.dumps({"K": K, "n": n, "ground_truth_rel_err_vs_lstsq": worst}))
    # one pair alone, and at position 17 of 64 drawn pairs (device ids), bitwise
    rs = np.random.RandomState(K)
    for p in (1, 8, 11):
        ids = torch.from_numpy(rs.randint(0, len(pairs), 64)).cuda()
        ids[17] = p
        many = pds.ground_truth(ids)
        alone = pds.ground_truth([p])
        assert _eq(many[17], alone[0]) and _eq(alone[0], C[p])
    pds.check()


@gpu
def test_ground_truth_singular_pair_and_bad_index(cuda):
    """Correspondences of the source shape on 5 distinct vertices cannot determine an 8 x 8 map: NaN and a status that
    check() raises; the other pairs of the call (the same shape as target included) are unaffected.  A bad device pair
    index: NaN, IndexError."""
    items = _items([(10, 12), (12, 12), (9, 14)], 32, seed0=3)
    vts = _vts(items, [50, 50, 50], seed=1, distinct=[None, None, 5])
    ds = dn.MeshDataset(items)
    pds = dn.PairDataset(ds, vts, [(0, 1), (1, 2), (2, 0)], n_fmap=8)
    C = pds.ground_truth(torch.tensor([0, 1, 2, 0], device="cuda"))
    assert torch.isnan(C[2]).all()
    assert torch.isfinite(C[0]).all() and torch.isfinite(C[1]).all() and _eq(C[0], C[3])
    with pytest.raises(RuntimeError, match="singular"):
        pds.check()
    pds.check()                                              # cleared
    C = pds.ground_truth(torch.tensor([0, 3], device="cuda"))
    assert torch.isnan(C[1]).all() and torch.isfinite(C[0]).all()
    with pytest.raises(IndexError, match="pair index 3 at position 1"):
        pds.check()
    with pytest.raises(IndexError, match="pair index -1 at position 0"):
        pds.ground_truth([-1])
    with pytest.raises(ValueError, match="40 and 50 correspondences"):
        dn.PairDataset(ds, [vts[0], vts[1][:40], vts[2]], [(1, 0)], n_fmap=8)
    with pytest.raises(IndexError, match="outside the mesh"):
        dn.PairDataset(ds, [vts[0], vts[1], vts[2] + 1000], [(0, 1)], n_fmap=8)
    with pytest.raises(ValueError, match="fewer than n_fmap"):
        dn.PairDataset(ds, vts, [(0, 1)], n_fmap=33)


# ---- rotations -------------------------------------------------------------------------------------------------------------
@gpu
def test_rotate_rows_batch_and_slot(cuda):
    items = _items([(8, 15), (30, 30), (5, 7), (12, 11)], 16, seed0=9)
    ds = dn.MeshDataset(items)
    X = torch.randn(ds.V, 3, generator=torch.Generator().manual_seed(0)).cuda()
    slot = ds.slot(3)
    for ids in ([1, 3, 0], [2, 2, 1]):
        b = ds.batch(ids)
        R = dn.batch.random_rotations(3, device="cuda")
        x = ds.pack(X, b, rotations=R)
        plain = ds.pack(X, b)
        assert _eq(dn.batch.rotate_rows(plain, b, R), x)
        real = torch.zeros(b.V, dtype=torch.bool, device="cuda")
        for k, (r0, nr, i) in enumerate(zip(b.row_begin, b.n_rows, ids)):
            real[r0:r0 + nr] = True
            x0 = X[ds.row_begin[i]:ds.row_begin[i] + nr].double()
            gold = (x0 @ R[k].double()).cpu().numpy()
            assert np.abs(x[r0:r0 + nr].cpu().numpy() - gold).max() <= 1e-6 * max(1.0, np.abs(x0.cpu().numpy()).max())
        assert not x[~real].any()
        slot.fill(torch.tensor(ids, device="cuda"))
        xs = slot.pack(X, rotations=R)
        assert _eq(xs[:b.V], x) and not xs[b.V:].any()
        assert _eq(slot.pack(X)[:b.V], plain)                # the unrotated buffer is a different one
    y = dn.batch.random_rotations(3, axis="y", device="cuda")
    assert (y[:, 1, 1] == 1).all()
    with pytest.raises(ValueError, match="float32 \\(V_total, 3\\)"):
        slot.pack(torch.randn(ds.V, 4, device="cuda"), rotations=R)
    with pytest.raises(ValueError, match="\\(3, 3, 3\\)"):
        slot.pack(X, rotations=R[:2])


# ---- the pair slot against the eager routes ---------------------------------------------------------------------------------
MODEL_SHAPES = [(10, 30), (13, 41), (20, 50), (8, 64), (31, 33)]
M_CORR = 60


def _model_setup(seed=0):
    torch.manual_seed(seed)
    m = dn.FunctionalMapCorrespondenceWithDiffusionNetFeatures(n_feat=128, input_features="xyz").cuda()
    items = _items(MODEL_SHAPES, 64, seed0=20)
    ds = dn.MeshDataset(items)
    X = torch.randn(ds.V, 3, generator=torch.Generator().manual_seed(seed + 1)).cuda()
    vts = _vts(items, [M_CORR] * len(items), seed=seed + 2)
    pds = dn.PairDataset(ds, vts, list(itertools.permutations(range(len(items)), 2)))
    return m, items, ds, X, pds


def _loss(model, pb, x, C_gt):
    C_pred, _ = model.forward_pairs(pb, x)
    return C_pred, (C_pred - C_gt).square().mean()


@gpu
def test_pair_slot_matches_pair_batch_and_per_pair_forward(cuda):
    """forward_pairs on a PairSlot against forward_pairs on pds.batch(ids) for the same draws, dropout off: C_pred,
    the features on the batch's rows and the loss bitwise.  Parameter gradients are held to 1e-4 (max relative
    difference), not bitwise: their weight reductions run over the slot's V_cap rows instead of the batch's V, so the
    fp32 partial sums are grouped differently, as for BatchSlot (tests/test_gpu_batch_slot.py); whether they happen to
    agree bitwise is printed.  Every pair's C_pred against the single-pair model forward as well."""
    m, items, ds, X, pds = _model_setup()
    m.eval()                                                       # dropout off; gradients still flow
    P = 3
    slot = pds.slot(P)
    rs = np.random.RandomState(5)
    worst_grad, worst_c, bitwise_grads = 0.0, 0.0, True
    for draw in range(3):
        ids = rs.randint(0, len(pds), P).tolist()
        slot.fill(torch.tensor(ids, device="cuda"))
        pb = pds.batch(ids)
        gt = slot.ground_truth()
        assert _eq(gt, pds.ground_truth(ids))
        with torch.no_grad():
            C_s, feat = m.forward_pairs(slot, slot.pack(X))
            C_b, _ = m.forward_pairs(pb, ds.pack(X, pb.mesh_batch))
        assert feat.shape == (slot.mesh_batch.V, 128)
        assert _eq(C_s, C_b)
        res = []
        for route, x in ((slot, slot.pack(X)), (pb, ds.pack(X, pb.mesh_batch))):
            m.zero_grad(set_to_none=True)
            C, loss = _loss(m, route, x, gt)
            loss.backward()
            res.append((C.detach(), loss.detach(), {k: p.grad.clone() for k, p in m.named_parameters()}))
        assert _eq(res[0][0], res[1][0]) and _eq(res[0][1], res[1][1])
        for k in res[0][2]:
            bitwise_grads &= _eq(res[0][2][k], res[1][2][k])
            e = _rel(res[0][2][k].cpu().numpy(), res[1][2][k].cpu().numpy())
            worst_grad = max(worst_grad, e)
            assert e < 1e-4, (draw, k, e)
        # every pair against the single-pair model forward
        sh = lambda s: [X[ds.row_begin[s]:ds.row_begin[s + 1]], None, None, items[s]["mass"], None, items[s]["evals"],
                        items[s]["evecs"], items[s]["gradX"], items[s]["gradY"], None, None]
        for p, i in enumerate(ids):
            with torch.no_grad():
                C1, _, _ = m(sh(pds.pair_x_host[i]), sh(pds.pair_y_host[i]))
            worst_c = max(worst_c, _rel(C_s[p].cpu().numpy(), C1[0].cpu().numpy()))
    slot.check()
    print(json.dumps({"param_grad_rel_err_slot_vs_pair_batch": worst_grad, "param_grads_bitwise": bitwise_grads,
                      "C_rel_err_vs_per_pair_forward": worst_c}))
    assert worst_c <= 1e-3


@gpu
def test_pair_slot_step_does_not_synchronise(cuda):
    m, items, ds, X, pds = _model_setup(seed=1)
    m.train()
    P = 2
    slot = pds.slot(P)
    ids = torch.tensor([0, 7], device="cuda")

    def step():
        slot.fill(ids)
        x = slot.pack(X, rotations=dn.batch.random_rotations(2 * P, device="cuda"))
        C_pred, _ = m.forward_pairs(slot, x)
        loss = (C_pred - slot.ground_truth()).square().mean()
        loss.backward()
        return loss

    step()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ids.fill_(3)
        loss = step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(loss)
    slot.check()


@gpu
def test_graphed_pair_step_with_rotations_and_dropout(cuda):
    """Rotations and dropout on: a replay after torch.cuda.manual_seed(s) computes bitwise what the eager slot step
    computes after the same seed (CUDA graphs replay torch's generator from its current seed and offset); replays
    draw new rotations and masks; an invalid pair index gives a NaN loss and IndexError, and the next fill recovers."""
    m, items, ds, X, pds = _model_setup(seed=2)
    m.train()
    P = 2
    slot = pds.slot(P)
    ids = torch.zeros(P, dtype=torch.int64, device="cuda")
    seen = {}

    def step(model, ids_):
        slot.fill(ids_)
        x = slot.pack(X, rotations=dn.batch.random_rotations(2 * P, device="cuda"))
        seen["x"] = x
        C_pred, _ = model.forward_pairs(slot, x)
        return (C_pred - slot.ground_truth()).square().mean()

    gs = dn.graphs.GraphedTrainStep(m, step, (ids,))
    x_buf = seen["x"]
    eager = copy.deepcopy(m)
    for s, draw in ((11, [3, 15]), (12, [8, 8])):
        ids.copy_(torch.tensor(draw, device="cuda"))
        torch.cuda.manual_seed(s)
        eager.zero_grad(set_to_none=True)
        le = step(eager, ids)
        le.backward()
        x_eager = seen["x"].clone()
        torch.cuda.manual_seed(s)
        gs.zero_grads(m)
        lg = gs.replay().clone()
        torch.cuda.synchronize()
        assert _eq(x_buf, x_eager)
        assert _eq(lg, le.detach()), (lg, le)
        for (k, p), q in zip(m.named_parameters(), eager.parameters()):
            assert _eq(p.grad, q.grad), k
    # consecutive replays: new rotations (and masks)
    xs, losses = [], []
    for _ in range(2):
        gs.zero_grads(m)
        losses.append(gs.replay().clone())
        xs.append(x_buf.clone())
    assert not torch.equal(xs[0], xs[1]) and not torch.equal(losses[0], losses[1])
    slot.check()
    # the masks alone: a second graph whose rotations are a fixed tensor; its only random draws are dropout's
    R_fixed = dn.batch.random_rotations(2 * P, device="cuda")

    def step_fixed(model, ids_):
        slot.fill(ids_)
        x = slot.pack(X, rotations=R_fixed)
        seen["x_fixed"] = x
        C_pred, _ = model.forward_pairs(slot, x)
        return (C_pred - slot.ground_truth()).square().mean()

    gf = dn.graphs.GraphedTrainStep(m, step_fixed, (ids,))
    xs, losses = [], []
    for _ in range(2):
        gf.zero_grads(m)
        losses.append(gf.replay().clone())
        xs.append(seen["x_fixed"].clone())
    assert _eq(xs[0], xs[1]) and not torch.equal(losses[0], losses[1])
    slot.check()
    # an invalid pair index, then recovery
    ids.copy_(torch.tensor([1, len(pds) + 4], device="cuda"))
    gs.zero_grads(m)
    assert torch.isnan(gs.replay()).item()
    with pytest.raises(IndexError, match="position 1"):
        slot.check()
    slot.check()
    ids.copy_(torch.tensor([1, 2], device="cuda"))
    gs.zero_grads(m)
    assert torch.isfinite(gs.replay()).item()
    assert all(torch.isfinite(p.grad).all() for p in m.parameters())
    slot.check()


@gpu
def test_pair_slot_check_reports_singular_ground_truth_and_over_capacity(cuda):
    """PairSlot.check() merges its ground-truth status with its BatchSlot's: a singular pair raises RuntimeError (its
    C_gt NaN), a draw past an explicit small capacity raises ValueError; each clears, and the next valid draw is clean."""
    items = _items([(10, 12), (12, 12), (9, 14), (30, 40)], 32, seed0=5)
    vts = _vts(items, [50] * 4, seed=3, distinct=[None, None, 5, None])
    ds = dn.MeshDataset(items)
    pds = dn.PairDataset(ds, vts, [(0, 1), (2, 0), (3, 3), (1, 0)], n_fmap=8)
    slot = pds.slot(2)
    slot.fill(torch.tensor([1, 0], device="cuda"))
    gt = slot.ground_truth()
    assert torch.isnan(gt[0]).all() and torch.isfinite(gt[1]).all()
    with pytest.raises(RuntimeError, match="pair 1 at position 0: the ground-truth system A\\^T A is singular"):
        slot.check()
    slot.check()                                             # cleared
    small = pds.slot(2, max_rows=1024)                       # pairs 2 and 0 need 2944 rows, pair 0 twice 768
    small.fill(torch.tensor([2, 0], device="cuda"))
    gt = small.ground_truth()
    assert torch.isfinite(gt).all()                          # the ground truth reads the dataset, not the slot
    with pytest.raises(ValueError, match="capacity of 1024 rows"):
        small.check()
    small.check()
    small.fill(torch.tensor([0, 0], device="cuda"))
    small.ground_truth()
    small.check()
    assert _eq(small.ground_truth(), pds.ground_truth([0, 0]))
