"""The training forward's entry points dn_learned_time_diffusion_fwd (and _batched, dn_to_basis_batched,
dn_from_basis_batched), dn_gradient_features_fwd, dn_mini_mlp_fwd and dn_compute_hks, called through the C-ABI on every
engine with exact fp32 inputs the test chooses, against the engine-emulating fp64 gold of
oracle/dn_oracle_engines_fwd.py under its componentwise bound: |ours - gold| <= bound element by element.

Every stage is checked on the fp32 intermediates the call itself wrote and the next stage read: x_diffuse on its
x_spec_out, the features on its pq_out, MiniMLP layer l on its hidden_out[l - 1].  Output buffers have NAN_ROWS extra
rows prefilled with NaN that must stay NaN.

``test_feat_tanh_sweep`` measures dn_feat_tanh over 2^27 arguments in every binade from 2^-40 to 16 against its
derived error bound.  ``test_routes_under_strict_tc`` runs every case in a DN_STRICT_TC=1 subprocess: a call succeeds
there iff the oracle's route table keeps each of its layers on tensor cores."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from test_gpu_backward_engines import (BATCH_CASES, DIFF_CASES, ENGINE_ID, FEAT_CASES, MLP_CASES, SEED, Report,  # noqa: F401
                                       _dev, _nan_buf, _sm, _stream, _ws, diffusion_inputs, lib, mlp_inputs)

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle_engines_bwd as B  # noqa: E402  (checker only)
import dn_oracle_engines_fwd as F  # noqa: E402  (checker only)

ENGINES = B.ENGINES
TC_ENGINES = ("tc3x", "tc1x", "bf16")


def diffusion_fwd_inputs(V, K, C, seed=SEED):
    """The backward's diffusion inputs, its grad_out as x: (x, mass, evals, evecs, time)."""
    g, mass, evals, evecs, time, _ = diffusion_inputs(V, K, C, seed)
    return g, mass, evals, evecs, time


def run_diffusion_fwd(lib, engine, x, mass, evals, evecs, time):
    V, C = x.shape
    K = evecs.shape[1]
    xd = _nan_buf(V, C)
    xs = torch.full((K, C), float("nan"), device="cuda")
    ins = [_dev(a) for a in (x, mass, evals, evecs, time)]
    ws = _ws(V, C)
    rc = lib.dn_learned_time_diffusion_fwd(*[t.data_ptr() for t in ins], V, K, C, xd.data_ptr(), xs.data_ptr(),
                                           ws.data_ptr(), ws.numel(), ENGINE_ID[engine], _stream())
    torch.cuda.synchronize()
    return rc, xd, xs, ins[4]


FLIPS = {}   # engine -> [elements of S, elements with a rounding boundary in their band]


def _flip(engine, st):
    f = FLIPS.setdefault(engine, [0, 0])
    f[0] += st.n
    f[1] += st.flip


def _check_time(rep, what, got, want):
    if not np.array_equal(got.cpu().numpy().view(np.int32), want.view(np.int32)):
        rep.misses.append("{}: time after the call is not max(t, 1e-8f) bitwise".format(what))


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(DIFF_CASES))
def test_diffusion_fwd(lib, case):
    """x_spec_out = Phi^T fl32(m x) (to_basis + spectral_scale's 4-slice tree), time clamped in place, x_diffuse =
    Phi (exp(-lambda t) x_spec_out) with S's band spread through the packed operand."""
    V, K, C = DIFF_CASES[case]
    sm = _sm(lib)
    a = diffusion_fwd_inputs(V, K, C)
    rep = Report("diffusion_fwd/{}".format(case))
    cache = {}
    for engine in ENGINES:
        rc, xd, xs, t = run_diffusion_fwd(lib, engine, *a)
        assert rc == 0, (engine, rc)
        st = B.Stats()
        gold = F.diffusion_fwd(*a, engine, x_spec_out=xs.cpu().numpy(), sm=sm, stats=st, cache=cache)
        _flip(engine, st)
        rep(engine + " x_spec", xs, gold["x_spec"])
        _check_time(rep, engine, t, gold["time"])
        rep(engine + " x_diffuse", xd[:V], gold["x_diffuse"])
        rep.nan_rows(engine + " x_diffuse", xd, V)
    rep.done()


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(BATCH_CASES))
def test_diffusion_fwd_batched(lib, case):
    """dn_learned_time_diffusion_fwd_batched (pack kernel's 8-slice tree), dn_to_basis_batched and
    dn_from_basis_batched on a ragged MeshBatch against each mesh's gold; padding rows of x_diffuse are exactly 0."""
    import diffusion_net_b200 as d
    rows, K, C = BATCH_CASES[case]
    sm = _sm(lib)
    meshes = [diffusion_fwd_inputs(v, K, C, seed=SEED + i) for i, v in enumerate(rows)]
    time = meshes[0][4]
    eye = lambda v: torch.sparse_coo_tensor(torch.arange(v).repeat(2, 1), torch.ones(v), (v, v)).cuda()
    items = [dict(mass=_dev(mi[1]), evals=_dev(mi[2]), evecs=_dev(mi[3]), gradX=eye(v), gradY=eye(v))
             for mi, v in zip(meshes, rows)]
    mb = d.MeshBatch(items)
    tb = mb._tb_rows.cpu().numpy().reshape(-1, 2)
    split = (len(tb), int((tb[:, 1] - tb[:, 0]).max()))    # every CTA of the plan, its longest row range
    V, nb = mb.V, len(rows)
    x = mb.pack([torch.from_numpy(mi[0]).cuda() for mi in meshes])
    G = np.random.RandomState(7).randn(nb * K, C).astype(np.float32)
    rep = Report("diffusion_fwd_batched/{}".format(case))
    for engine in TC_ENGINES:
        t = _dev(time)
        xd = torch.full((V, C), float("nan"), device="cuda")
        xs = torch.full((nb * K, C), float("nan"), device="cuda")
        tbo = torch.full((nb * K, C), float("nan"), device="cuda")
        fbo = torch.full((V, C), float("nan"), device="cuda")
        ws = _ws(V, 2 * C)
        args = (ctypes.byref(mb.desc), V, K, C)
        rc = lib.dn_learned_time_diffusion_fwd_batched(x.data_ptr(), mb.mass.data_ptr(), mb.evals.data_ptr(),
                                                       mb.evecs.data_ptr(), t.data_ptr(), *args, xd.data_ptr(),
                                                       xs.data_ptr(), ws.data_ptr(), ws.numel(), ENGINE_ID[engine],
                                                       _stream())
        assert rc == 0, (engine, rc)
        rc = lib.dn_to_basis_batched(x.data_ptr(), mb.evecs.data_ptr(), mb.mass.data_ptr(), *args, tbo.data_ptr(),
                                     ws.data_ptr(), ws.numel(), ENGINE_ID[engine], _stream())
        assert rc == 0, (engine, rc)
        g = _dev(G)
        rc = lib.dn_from_basis_batched(g.data_ptr(), mb.evecs.data_ptr(), mb.mass.data_ptr(), *args, fbo.data_ptr(),
                                       ws.data_ptr(), ws.numel(), ENGINE_ID[engine], _stream())
        assert rc == 0, (engine, rc)
        torch.cuda.synchronize()
        _check_time(rep, engine, t, F.clamped_time(time))
        xs_h = xs.cpu().numpy()
        for b, mi in enumerate(meshes):
            r0, n = mb.row_begin[b], rows[b]
            ks = slice(b * K, (b + 1) * K)
            gold = F.diffusion_fwd(*mi[:4], time, engine, x_spec_out=xs_h[ks], sm=sm, split=split, tree=8)
            rep("{} x_spec mesh {}".format(engine, b), xs[ks], gold["x_spec"])
            rep("{} x_diffuse mesh {}".format(engine, b), xd[r0:r0 + n], gold["x_diffuse"])
            for what, buf in (("x_diffuse", xd), ("from_basis_batched", fbo)):
                if not bool((buf[r0 + n:mb.row_begin[b + 1]] == 0).all()):
                    rep.misses.append("{} mesh {}: padding rows of {} are not exactly 0".format(engine, b, what))
            rep("{} to_basis_batched mesh {}".format(engine, b), tbo[ks],
                F.to_basis_batched(mi[0], mi[1], mi[3], engine, split, sm=sm))
            rep("{} from_basis_batched mesh {}".format(engine, b), fbo[r0:r0 + n],
                F.from_basis_batched(G[ks], mi[3], mi[1], engine))
    rep.done()


# ---- gradient features ----------------------------------------------------------------------------------------------
def feat_inputs(rows, cols, V, C, rot, seed=SEED):
    """(gX, gY) as scipy CSR on one pattern (one entry per (row, col)) and the exact fp32 inputs of
    dn_gradient_features_fwd.  A row's values are scaled by 1 / sqrt(its entries), so that the features' arguments
    are O(1) on every row, long ones included, and the tanh does not saturate."""
    import scipy.sparse as sp
    rs = np.random.RandomState(seed)
    key = np.unique(np.asarray(rows, np.int64) * V + cols)
    rows, cols = key // V, key % V
    f32 = lambda a: np.asarray(a, np.float32)
    scale = 1 / np.sqrt(np.bincount(rows, minlength=V)[rows])
    gx, gy = f32(rs.randn(len(rows)) * scale), f32(rs.randn(len(rows)) * scale)
    gX = sp.csr_matrix((gx.astype(np.float64), (rows, cols)), shape=(V, V))
    gY = sp.csr_matrix((gy.astype(np.float64), (rows, cols)), shape=(V, V))
    a = dict(rows=rows, cols=cols, gx=gx, gy=gy, x_diffuse=f32(rs.randn(V, C)),
             A_re=f32(rs.randn(C, C) / np.sqrt(C)), A_im=f32(rs.randn(C, C) / np.sqrt(C)) if rot else None)
    return gX, gY, a


def torus_feat_inputs(n, m, C, rot, long_rows=0, long_width=300, seed=SEED):
    """An n x m torus pattern; ``long_rows`` rows (the first of a 64-row block) get ``long_width`` more entries, so
    that block holds more than the block gather's 1024 staged entries."""
    from diffusion_net_b200 import synthetic
    V = n * m
    rows, cols = synthetic.torus_pattern(n, m)
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    if long_rows:
        rs = np.random.RandomState(seed + 1)
        r0 = 64 * (V // 128)
        extra_r = np.repeat(np.arange(r0, r0 + long_rows), long_width)
        extra_c = rs.randint(0, V, len(extra_r))
        rows, cols = np.concatenate([rows, extra_r]), np.concatenate([cols, extra_c])
    return feat_inputs(rows, cols, V, C, rot, seed)


# name: (n, m, C, rotations, patched, long rows).  The gather launch_spmm_features picks: the patched kernel (C = 128,
# patches built as ops builds them), the block kernel (C = 128, 256; long rows past its 1024 staged entries), float4
# lanes (C % 4 == 0 otherwise), float lanes (C % 4 != 0).  The [P|Q] layer: TF32 under bf16 at C = 40, SIMT at C = 256
# with rotations (npq = 512), SIMT for K = C not on the 8 grid
FWD_FEAT_CASES = dict({k: v + (False, 0) for k, v in FEAT_CASES.items()}, **{
    "c128_rot_patched": (84, 84, 128, True, True, 0), "c128_norot_patched": (84, 84, 128, False, True, 0),
    "c128_rot_long": (40, 41, 128, True, False, 6), "c128_norot_long": (40, 41, 128, False, False, 6),
    "c256_rot_long": (20, 33, 256, True, False, 5), "c256_norot": (20, 33, 256, False, False, 0),
    "c1_rot": (17, 19, 1, True, False, 0), "c1_norot": (17, 19, 1, False, False, 0),
    "c3_rot": (17, 19, 3, True, False, 0), "c6_norot": (17, 19, 6, False, False, 0),
    "c30_rot": (23, 31, 30, True, False, 0), "c30_norot": (23, 31, 30, False, False, 0),
    "c40_norot": (30, 41, 40, False, False, 0), "c48_rot_long": (23, 31, 48, True, False, 4),
})


def run_features_fwd(lib, engine, a, V, C, patched=False):
    import diffusion_net_b200 as d
    rot = a["A_im"] is not None
    idx = torch.from_numpy(np.stack([a["rows"], a["cols"]]))
    coo = lambda v: torch.sparse_coo_tensor(idx, torch.from_numpy(v), (V, V)).coalesce().cuda()
    gops = d.ops.GradOperators(coo(a["gx"]), coo(a["gy"]))
    if patched:
        gops.build_patches()
        assert gops._patches, "no patches were built"
    npq = 2 * C if rot else C
    xd, are = _dev(a["x_diffuse"]), _dev(a["A_re"])
    aim = _dev(a["A_im"]) if rot else None
    feat, pq = _nan_buf(V, C), _nan_buf(V, npq)
    ws = _ws(V, 4 * C)
    rc = lib.dn_gradient_features_fwd(ctypes.byref(gops.csr[0]), xd.data_ptr(), are.data_ptr(),
                                      aim.data_ptr() if rot else None, 1 if rot else 0, V, C, feat.data_ptr(),
                                      pq.data_ptr(), ws.data_ptr(), ws.numel(), ENGINE_ID[engine], _stream())
    torch.cuda.synchronize()
    return rc, feat, pq


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(FWD_FEAT_CASES))
def test_gradient_features_fwd(lib, case):
    """pq_out = xd [A_re; A_im]^T as one run_chain layer; the features = dn_feat_tanh(gX Bre + gY Bim) on the call's
    own pq_out, with the gather's fmaf chains and the tanh's derived error in the bound."""
    n, m, C, rot, patched, long_rows = FWD_FEAT_CASES[case]
    V = n * m
    gX, gY, a = torus_feat_inputs(n, m, C, rot, long_rows)
    if long_rows:
        assert np.diff(gX.indptr)[64 * (V // 128):64 * (V // 128) + 64].sum() > 1024
    rep = Report("features_fwd/{}".format(case))
    for engine in ENGINES:
        rc, feat, pq = run_features_fwd(lib, engine, a, V, C, patched)
        assert rc == 0, (engine, rc)
        gold = F.features_fwd(gX, gY, a["x_diffuse"], a["A_re"], a["A_im"], engine, pq_out=pq[:V].cpu().numpy())
        rep(engine + " pq", pq[:V], gold["pq"])
        rep(engine + " features", feat[:V], gold["features"])
        rep.nan_rows(engine + " pq", pq, V)
        rep.nan_rows(engine + " features", feat, V)
    rep.done()


TANH_STATED = 6.9e-7      # dn_simt.cu's stated absolute error of dn_feat_tanh: 11.5 * 2^-24, the sup of tanh_error
SWEEP_LOG2 = 27
SWEEP_CHUNK = 1 << 24


def _sweep_args(seed):
    """SWEEP_CHUNK fp32 arguments: random mantissas over the binades [2^e, 2^(e+1)), e = -40 .. 3, both signs."""
    rs = np.random.RandomState(seed)
    e = rs.randint(-40, 4, SWEEP_CHUNK)
    mant = rs.randint(0, 1 << 23, SWEEP_CHUNK)
    bits = ((e + 127).astype(np.uint32) << 23) | mant.astype(np.uint32)
    bits |= (rs.rand(SWEEP_CHUNK) < 0.5).astype(np.uint32) << 31
    return bits.view(np.float32)


def run_feat_tanh(lib, s, x0=None):
    """dn_gradient_features_fwd without rotations on C = 2, one CSR entry per row (its diagonal, gx = 1, gy = 0),
    x_diffuse row v = (x0_v, s_v) and A_re = [[0, 1], [1, 0]]: P[v, 0] = s_v exactly (a SIMT layer: x0 * 0 + s * 1), so
    channel 0's argument gX Bre + gY Bim = x0_v s_v + 0 is s_v for x0 = 1 and the feature is dn_feat_tanh(s_v)."""
    import diffusion_net_b200 as d
    V = len(s)
    rowptr = torch.arange(V + 1, dtype=torch.int32, device="cuda")
    colidx = torch.arange(V, dtype=torch.int32, device="cuda")
    vals = torch.zeros(V, 2, device="cuda")
    vals[:, 0] = 1
    gops = d.ops.GradOperators.from_csr(V, rowptr, colidx, vals)
    xd = torch.ones(V, 2, device="cuda")
    xd[:, 1] = torch.from_numpy(s).cuda()
    if x0 is not None:
        xd[:, 0] = torch.from_numpy(x0).cuda()
    are = torch.tensor([[0.0, 1.0], [1.0, 0.0]], device="cuda")
    feat, pq = torch.empty(V, 2, device="cuda"), torch.empty(V, 2, device="cuda")
    ws = _ws(V, 8)
    rc = lib.dn_gradient_features_fwd(ctypes.byref(gops.csr[0]), xd.data_ptr(), are.data_ptr(), None, 0, V, 2,
                                      feat.data_ptr(), pq.data_ptr(), ws.data_ptr(), ws.numel(), ENGINE_ID["simt"],
                                      _stream())
    torch.cuda.synchronize()
    assert rc == 0, rc
    p0 = pq[:, 0].cpu().numpy()
    assert np.array_equal(p0.view(np.int32), s.view(np.int32)) or np.isnan(s).any(), "P[:, 0] is not the argument"
    return feat[:, 0].cpu().numpy()


@pytest.mark.gpu
def test_feat_tanh_sweep(lib):
    """dn_feat_tanh over 2^27 arguments within its derived error T(x) (oracle tanh_error), and within the error its
    comment states."""
    worst, worst_x, worst_ratio, n = 0.0, 0.0, 0.0, 0
    for chunk in range(1 << (SWEEP_LOG2 - 24)):
        s = _sweep_args(chunk)
        f = run_feat_tanh(lib, s).astype(np.float64)
        x = s.astype(np.float64)
        err = np.abs(f - np.tanh(x))
        T = F.tanh_error(x, x)
        r = err / T
        i = int(np.argmax(err))
        if err[i] > worst:
            worst, worst_x = float(err[i]), float(x[i])
        worst_ratio = max(worst_ratio, float(r.max()))
        n += len(s)
        assert (err <= T).all(), ("dn_feat_tanh exceeds its derived error", x[np.argmax(r)], float(r.max()))
    # +-0; +-inf as the argument 2^64 * (+-2^64), which overflows in the final fmaf; NaN
    big = np.float32(2.0 ** 64)
    specials = np.array([0.0, -0.0, big, -big, np.nan], np.float32)
    x0 = np.array([1, 1, big, big, 1], np.float32)
    f = run_feat_tanh(lib, np.resize(specials, 64), np.resize(x0, 64))[:5]
    assert abs(f[0]) <= F.tanh_error(0.0, 0.0) and abs(f[1]) <= F.tanh_error(0.0, 0.0)
    assert f[2] == 1.0 and f[3] == -1.0 and np.isnan(f[4]), f
    print("[measured] dn_feat_tanh over {} arguments: worst |err| = {:.3g} at x = {!r}, worst err/T = {:.3g}".format(
        n, worst, worst_x, worst_ratio))
    assert worst <= TANH_STATED, "dn_feat_tanh's measured error {:.3g} exceeds the stated {:.3g}".format(
        worst, TANH_STATED)


# ---- MiniMLP --------------------------------------------------------------------------------------------------------
# the backward's cases, plus (V, C, hidden, p, biased layers, residual): a residual, a first layer on the TF32 fallback
# under bf16 (K = 120), and the three-warpgroup chain (C =
# 128, a hidden layer of 128, V past one wave of 128-row tiles) at the last-192-row-tile edges and at V = 200037.
# "wg3_last<n>" is resolved at run time to the size whose last 192-row tile holds n rows.
FWD_MLP_CASES = dict({k: v + (False,) for k, v in MLP_CASES.items()}, **{
    "residual_v7000": (7000, 64, [64], 0.1, None, True), "c40_hidden48": (1230, 40, [48], 0.1, None, False), "residual_depth3_v129": (129, 48, [48, 48], 0.5, None, True),
    "wg3_v20000": (20000, 128, [128], 0.1, None, True), "wg3_v200037": (200037, 128, [128], 0.0, None, True),
    "wg3_last1": (1, 128, [128], 0.0, None, True), "wg3_last64": (64, 128, [128], 0.5, None, True),
    "wg3_last65": (65, 128, [128], 0.0, None, True), "wg3_last129": (129, 128, [128], 0.1, None, True),
    "wg3_last191": (191, 128, [128], 0.0, None, True),
})
WG3_ENGINES = ("tc3x", "tc1x")


def _mlp_case(case, sm):
    V, C, hidden, p, hb, res = FWD_MLP_CASES[case]
    if case.startswith("wg3_last"):
        V = 192 * ((128 * sm) // 192 + 1) + V
    return V, C, hidden, p, hb, res


def mlp_fwd_inputs(V, C, hidden, p, has_bias, residual, seed=SEED):
    _, srcs, weights, _, drops, dims = mlp_inputs(V, C, hidden, p, seed)
    rs = np.random.RandomState(seed + 5)
    biases = [np.asarray(rs.randn(w.shape[0]) * 0.1, np.float32) if (has_bias is None or has_bias[i]) else None
              for i, w in enumerate(weights)]
    res = np.asarray(rs.randn(V, C), np.float32) if residual else None
    return srcs, weights, biases, drops, res


def run_mini_mlp_fwd(lib, engine, srcs, weights, biases, drops, residual, with_hidden=True):
    from diffusion_net_b200 import _lib as L
    V = srcs[0].shape[0]
    n = len(weights)
    dims = [sum(s.shape[1] for s in srcs)] + [w.shape[0] for w in weights]
    d_s, d_w = [_dev(s) for s in srcs], [_dev(w) for w in weights]
    d_b = [_dev(b) if b is not None else None for b in biases]
    d_m = [_dev(m) for m in drops] if drops else None
    d_r = _dev(residual) if residual is not None else None
    hid = [_nan_buf(V, dims[l + 1]) for l in range(n - 1)] if with_hidden else []
    out = _nan_buf(V, dims[-1])
    ws = _ws(V, max(dims))
    rc = lib.dn_mini_mlp_fwd(
        L.ptr_array([s.data_ptr() for s in d_s]), L.int_array([s.shape[1] for s in srcs]), len(srcs),
        L.ptr_array([w.data_ptr() for w in d_w]), L.ptr_array([b.data_ptr() if b is not None else None for b in d_b]),
        L.int_array(dims), n, L.ptr_array([m.data_ptr() for m in d_m]) if d_m else None,
        d_r.data_ptr() if d_r is not None else None, V,
        L.ptr_array([h.data_ptr() for h in hid]) if hid else None, out.data_ptr(), ws.data_ptr(), ws.numel(),
        ENGINE_ID[engine], _stream())
    torch.cuda.synchronize()
    return rc, hid, out


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(FWD_MLP_CASES))
def test_mini_mlp_fwd(lib, case):
    """Each layer on the call's own previous activation (the sources for layer 0): bias, relu, the dropout multiplier,
    the residual on the last layer.  ``out`` with hidden_out = NULL is bitwise ``out`` with it."""
    sm = _sm(lib)
    V, C, hidden, p, hb, res = _mlp_case(case, sm)
    srcs, weights, biases, drops, r = mlp_fwd_inputs(V, C, hidden, p, hb, res)
    rep = Report("mini_mlp_fwd/{}".format(case))
    for engine in (WG3_ENGINES if case.startswith("wg3") else ENGINES):
        rc, hid, out = run_mini_mlp_fwd(lib, engine, srcs, weights, biases, drops, r)
        assert rc == 0, (engine, rc)
        hid_h = [h[:V].cpu().numpy() for h in hid]
        gold = F.mini_mlp_fwd(srcs, weights, biases, drops, r, engine, hidden=hid_h)
        for l, h in enumerate(hid):
            rep("{} hidden{}".format(engine, l), hid_h[l], gold["hidden"][l])
            rep.nan_rows("{} hidden{}".format(engine, l), h, V)
        rep(engine + " out", out[:V], gold["out"])
        rep.nan_rows(engine + " out", out, V)
        if hidden:
            rc, _, out0 = run_mini_mlp_fwd(lib, engine, srcs, weights, biases, drops, r, with_hidden=False)
            assert rc == 0, (engine, rc)
            if not torch.equal(out0[:V].view(torch.int32), out[:V].view(torch.int32)):
                rep.misses.append("{}: out without hidden_out differs from out with it".format(engine))
    rep.done()


# ---- heat kernel signature ------------------------------------------------------------------------------------------
# name: (V, K, S).  hks_warp_kernel for K in {32, 64, 96, 128, 256} and S <= 16 (V = 200k: past its grid cap, the
# grid-stride loop), hks_generic_kernel otherwise (K = 16, 160; S = 17)
HKS_CASES = {"k16_s16": (3000, 16, 16), "k160_s17": (3001, 160, 17), "k32_s1": (200000, 32, 1),
             "k96_s3": (777, 96, 3), "k128_s16": (200000, 128, 16), "k256_s16": (5000, 256, 16),
             "k256_s17": (5000, 256, 17), "k128_s17": (1000, 128, 17)}


def hks_inputs(V, K, S, seed=SEED):
    rs = np.random.RandomState(seed)
    f32 = lambda a: np.asarray(a, np.float32)
    evals = f32(np.sort(rs.rand(K)) * 500.0)
    evals[0] = 0.0
    evecs = f32(rs.randn(V, K) / np.sqrt(V) * np.exp(rs.uniform(-3, 3, (V, 1))))
    scales = f32(np.logspace(-4, 2, S))
    return evals, evecs, scales


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(HKS_CASES))
def test_compute_hks(lib, case):
    """dn_compute_hks within a bound relative to each element (every term is >= 0)."""
    V, K, S = HKS_CASES[case]
    evals, evecs, scales = hks_inputs(V, K, S)
    out = _nan_buf(V, S)
    ins = [_dev(a) for a in (evals, evecs, scales)]
    rc = lib.dn_compute_hks(*[t.data_ptr() for t in ins], V, K, S, out.data_ptr(), _stream())
    torch.cuda.synchronize()
    assert rc == 0, rc
    rep = Report("compute_hks/{}".format(case))
    rep("out", out[:V], F.compute_hks(evals, evecs, scales))
    rep.nan_rows("out", out, V)
    rep.done()


@pytest.mark.gpu
def test_flip_allowance_fraction():
    """Of S's elements, the share whose band holds a rounding boundary of the engine's format: the elements where the
    x_diffuse bound pays for a possible flip."""
    if not FLIPS:
        pytest.skip("runs after the diffusion cases")
    for engine, (n, k) in sorted(FLIPS.items()):
        if n:
            print("[measured] S flip allowance {}: {} of {} elements ({:.3%})".format(engine, k, n, k / n))


# ---- routes ---------------------------------------------------------------------------------------------------------
def route_table():
    """{case/engine: True if every layer of the case stays on tensor cores} from the oracle's route table."""
    want = {}
    for engine in TC_ENGINES:
        for name, (V, K, C) in DIFF_CASES.items():
            r = F.routes(engine, K, C, [3 * C, C])
            want["diff/{}/{}".format(name, engine)] = "simt" not in (r["diffusion/to_basis"],
                                                                     r["diffusion/from_basis"])
        for name, (n, m, C, rot, patched, lr) in FWD_FEAT_CASES.items():
            r = F.routes(engine, 40, C, [3 * C, C])
            want["feat/{}/{}".format(name, engine)] = r["features/pq" if rot else "features/pq_norot"] != "simt"
        for name, (V, C, hidden, p, hb, res) in FWD_MLP_CASES.items():
            if name.startswith("wg3_last"):
                continue
            want["mlp/{}/{}".format(name, engine)] = F.mlp_on_tc(engine, C, [3 * C] + hidden + [C])
    return want


def _route_report():
    """Run in a DN_STRICT_TC=1 subprocess: each case on each tensor-core engine; prints one JSON line."""
    import diffusion_net_b200 as d
    lib = d._lib.load()
    got = {}
    for key in route_table():
        kind, name, engine = key.split("/")
        if kind == "diff":
            V, K, C = DIFF_CASES[name]
            rc = run_diffusion_fwd(lib, engine, *diffusion_fwd_inputs(min(V, 1000), K, C))[0]
        elif kind == "feat":
            n, m, C, rot, patched, lr = FWD_FEAT_CASES[name]
            rc = run_features_fwd(lib, engine, torus_feat_inputs(n, m, C, rot, lr)[2], n * m, C, patched)[0]
        else:
            V, C, hidden, p, hb, res = FWD_MLP_CASES[name]
            rc = run_mini_mlp_fwd(lib, engine, *mlp_fwd_inputs(min(V, 1000), C, hidden, p, hb, res))[0]
        got[key] = rc == 0
    print(json.dumps(got))


@pytest.mark.gpu
def test_routes_under_strict_tc(lib):
    tests_dir = os.path.join(ROOT, "tests")
    env = dict(os.environ, DN_STRICT_TC="1")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", "import sys; sys.path[:0] = [{!r}, {!r}]; import test_gpu_forward_engines as t; t._route_report()".format(
            tests_dir, ROOT)]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    want = route_table()
    assert got == want, {k: (got.get(k), want[k]) for k in want if got.get(k) != want[k]}
