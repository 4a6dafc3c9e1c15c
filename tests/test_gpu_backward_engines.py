"""The backward entry points dn_learned_time_diffusion_bwd, dn_from_basis (row_scale) and dn_mini_mlp_bwd, called
through the C-ABI on every engine with exact fp32 inputs the test chooses, against the engine-emulating fp64 gold of
oracle/dn_oracle_engines_bwd.py under its componentwise bound: |ours - gold| <= bound element by element.

Inputs reach the edges: hidden activations with exact zeros (the relu mask m > 0 decides), dropout masks of 0 and
1 / (1 - p) for p = 0.1 and 0.5, a mass spanning e^-6 .. e^3, times of -0.1, 0, 1e-9 (clamped to 1e-8) and one where
every exp(-lambda t) but the first underflows.  Output buffers have NAN_ROWS extra rows prefilled with NaN that must
stay NaN; weight-gradient and grad_time buffers are prefilled with a nonzero value (accumulate = 1).

``test_routes_under_strict_tc`` runs every case in a DN_STRICT_TC=1 subprocess: a call succeeds there iff the oracle's
route table keeps each of its contractions on tensor cores."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle_engines_bwd as B  # noqa: E402  (checker only)

ENGINE_ID = {"simt": 0, "tc3x": 1, "tc1x": 2, "bf16": 3}
NAN_ROWS = 5
GRAD_W_INIT = 0.25
GRAD_T_INIT = 0.5
GRAD_B_INIT = -0.75
T_UNDERFLOW = 100.0
SEED = 31

# (V, K, C): test_gpu_backward's CASES (tiny, k12, k160, c40, c256, full), the 128-row tile edges, K from 8 (bf16 falls
# back to TF32) past 128 (to_basis on SIMT) to 256, and C off and on the 16 grid up to the two-slice to_basis
DIFF_CASES = {
    "tiny": (50, 40, 16), "k12": (713, 12, 48), "k160": (2000, 160, 96), "c40": (1230, 64, 40),
    "c256": (4980, 128, 256), "full": (200000, 128, 128),
    "v1": (1, 40, 16), "v127": (127, 128, 128), "v128": (128, 64, 64), "v129": (129, 128, 128),
    "v7000": (7000, 128, 128), "v200037": (200037, 128, 128),
    "k8": (700, 8, 48), "k256": (700, 256, 48), "c20": (700, 40, 20), "c128_k40": (700, 40, 128),
}

# name: (V, C, hidden widths, dropout p, biased layers (None: all)) -- three sources of width C as in the block
MLP_CASES = {
    "depth1_v129": (129, 48, [], 0.0, None),
    "depth2_v1": (1, 16, [16], 0.5, None),
    "depth2_v128": (128, 64, [64], 0.0, None),
    "depth2_v7000_p01": (7000, 128, [128], 0.1, None),
    "depth3_v127_p05": (127, 16, [16, 16], 0.5, None),
    "depth8": (1000, 64, [64] * 7, 0.0, None),
    "depth9_layer_by_layer": (1000, 64, [64] * 8, 0.5, None),
    "hidden256": (2000, 128, [256], 0.0, None),
    "c20_hidden40": (713, 20, [40], 0.0, None),
    "c40": (1230, 40, [40, 40], 0.1, None),
    "bias_none": (2000, 48, [48, 48], 0.0, [True, False, True]),
    "full_v200037": (200037, 64, [64], 0.5, None),
}


# gradient features: name: (n, m, C, rotations) on an n x m torus pattern (V = n m).  c40: the grad_x layer and the
# weight gradients on SIMT (simt_layer's two-pass split); c256: grad_x on tensor cores, weight gradients on SIMT
FEAT_CASES = {
    "c48_rot": (23, 31, 48, True), "c48_norot": (23, 31, 48, False), "c40_rot": (30, 41, 40, True),
    "c256_rot": (60, 83, 256, True), "c128_rot_v7056": (84, 84, 128, True), "c128_norot_v7056": (84, 84, 128, False),
}


def features_inputs(n, m, C, rot, seed=SEED):
    """(gX, gY) as scipy CSR on one torus pattern, and the exact fp32 arrays of dn_gradient_features_bwd."""
    import scipy.sparse as sp
    from diffusion_net_b200 import synthetic
    rs = np.random.RandomState(seed)
    V = n * m
    rows, cols = synthetic.torus_pattern(n, m)
    keep = np.ones(len(rows), bool)
    keep[np.unique(rows * V + cols, return_index=True)[1]] = False
    rows, cols = rows[~keep], cols[~keep]          # one entry per (row, col)
    f32 = lambda a: np.asarray(a, np.float32)
    gx, gy = f32(rs.randn(len(rows)) * 3), f32(rs.randn(len(rows)) * 3)
    gX = sp.csr_matrix((gx.astype(np.float64), (rows, cols)), shape=(V, V))
    gY = sp.csr_matrix((gy.astype(np.float64), (rows, cols)), shape=(V, V))
    npq = 2 * C if rot else C
    a = dict(rows=rows, cols=cols, gx=gx, gy=gy, grad_features=f32(rs.randn(V, C)), x_diffuse=f32(rs.randn(V, C)),
             pq=f32(rs.randn(V, npq)), features=f32(rs.uniform(-0.999, 0.999, (V, C))),
             A_re=f32(rs.randn(C, C) / np.sqrt(C)), A_im=f32(rs.randn(C, C) / np.sqrt(C)) if rot else None)
    return gX, gY, a


def diffusion_inputs(V, K, C, seed=SEED):
    rs = np.random.RandomState(seed)
    f32 = lambda a: np.asarray(a, np.float32)
    evecs = f32(rs.randn(V, K) / np.sqrt(V))
    evals = f32(np.sort(rs.rand(K)) * 200.0)
    evals[0] = 0.0
    mass = f32(np.exp(rs.uniform(-6, 3, V)))
    time = f32(rs.rand(C) * 0.3)
    time[:4] = [-0.1, 0.0, 1e-9, T_UNDERFLOW][:C]
    x_spec = f32(rs.randn(K, C))
    grad_out = f32(rs.randn(V, C))
    return grad_out, mass, evals, evecs, time, x_spec


def mlp_inputs(V, C, hidden, p, seed=SEED):
    rs = np.random.RandomState(seed)
    f32 = lambda a: np.asarray(a, np.float32)
    dims = [3 * C] + list(hidden) + [C]
    srcs = [f32(rs.randn(V, C)) for _ in range(3)]
    weights = [f32(rs.uniform(-1, 1, (dims[i + 1], dims[i])) / np.sqrt(dims[i])) for i in range(len(dims) - 1)]
    drops = None
    if p > 0:
        drops = [f32(np.where(rs.rand(V, w) < p, 0.0, np.float32(1.0) / np.float32(1.0 - p))) for w in hidden]
    # saved activations relu(z) (* mask): about half exact zeros, so the relu mask decides
    hid = [f32(np.maximum(rs.randn(V, w), 0) * (drops[i] if drops else 1.0)) for i, w in enumerate(hidden)]
    grad_out = f32(rs.randn(V, C))
    return grad_out, srcs, weights, hid, drops, dims


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import diffusion_net_b200 as d
    return d._lib.load()


def _sm(lib):
    sm, cc, smem = ctypes.c_int(), ctypes.c_int(), ctypes.c_int64()
    assert lib.dn_device_query(0, ctypes.byref(sm), ctypes.byref(cc), ctypes.byref(smem)) == 0
    return sm.value


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _nan_buf(V, N):
    return torch.full((V + NAN_ROWS, N), float("nan"), device="cuda")


def _ws(V, N):
    return torch.empty(4 * (2 * V * N) + (320 << 20), dtype=torch.uint8, device="cuda")


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class Report:
    """Collects every comparison of a test against its componentwise bound and fails with all misses listed."""

    def __init__(self, label):
        self.label, self.misses = label, []

    def __call__(self, what, ours, gold_bound):
        gold, bound = gold_bound
        ours = ours.detach().cpu().double().numpy() if torch.is_tensor(ours) else ours
        err = np.abs(ours - gold)
        ok = err <= bound
        ratio = float(np.max(np.where(bound > 0, err / np.where(bound > 0, bound, 1), np.where(err > 0, np.inf, 0))))
        print("[measured] {} {} worst err/bound={:.3g}".format(self.label, what, ratio))
        if not ok.all():
            i = np.unravel_index(np.argmax(~ok), ok.shape)
            self.misses.append("{}: {} of {} elements out, first at {} ours={!r} gold={!r} bound={:.3g}".format(
                what, int((~ok).sum()), ok.size, i, ours[i], gold[i], bound[i]))

    def nan_rows(self, what, buf, V):
        if not bool(torch.isnan(buf[V:]).all()):
            self.misses.append("{}: rows past V were written".format(what))

    def done(self):
        assert not self.misses, "{}: {}".format(self.label, "; ".join(self.misses))


def run_diffusion_bwd(lib, engine, grad_out, mass, evals, evecs, time, x_spec):
    V, C = grad_out.shape
    K = evecs.shape[1]
    gx = _nan_buf(V, C)
    gt = torch.full((C,), GRAD_T_INIT, device="cuda")
    ins = [_dev(a) for a in (grad_out, mass, evals, evecs, time, x_spec)]
    ws = _ws(V, C)
    rc = lib.dn_learned_time_diffusion_bwd(*[t.data_ptr() for t in ins], V, K, C, gx.data_ptr(), gt.data_ptr(),
                                           ws.data_ptr(), ws.numel(), ENGINE_ID[engine], _stream())
    torch.cuda.synchronize()
    return rc, gx, gt


def run_from_basis(lib, engine, values, basis, row_scale):
    K, C = values.shape
    V = basis.shape[0]
    out = _nan_buf(V, C)
    ins = [_dev(a) for a in (values, basis, row_scale)]
    ws = _ws(V, C)
    rc = lib.dn_from_basis(*[t.data_ptr() for t in ins], V, K, C, out.data_ptr(), ws.data_ptr(), ws.numel(),
                           ENGINE_ID[engine], _stream())
    torch.cuda.synchronize()
    return rc, out


def run_mini_mlp_bwd(lib, engine, grad_out, srcs, weights, hid, drops, has_bias):
    from diffusion_net_b200 import _lib as L
    V = grad_out.shape[0]
    n = len(weights)
    dims = [sum(s.shape[1] for s in srcs)] + [w.shape[0] for w in weights]
    d_srcs, d_w, d_h = [_dev(s) for s in srcs], [_dev(w) for w in weights], [_dev(h) for h in hid]
    d_m = [_dev(m) for m in drops] if drops else None
    g_src = [_nan_buf(V, s.shape[1]) for s in srcs]
    g_w = [torch.full(tuple(w.shape), GRAD_W_INIT, device="cuda") for w in weights]
    g_b = [torch.full((w.shape[0],), GRAD_B_INIT, device="cuda") if (has_bias is None or has_bias[i]) else None
           for i, w in enumerate(weights)]
    g = _dev(grad_out)
    ws = _ws(V, max(dims))
    rc = lib.dn_mini_mlp_bwd(
        g.data_ptr(), L.ptr_array([s.data_ptr() for s in d_srcs]), L.int_array([s.shape[1] for s in srcs]), len(srcs),
        L.ptr_array([w.data_ptr() for w in d_w]), L.int_array(dims), n,
        L.ptr_array([h.data_ptr() for h in d_h]) if d_h else None,
        L.ptr_array([m.data_ptr() for m in d_m]) if d_m else None, V,
        L.ptr_array([x.data_ptr() for x in g_src]), L.ptr_array([x.data_ptr() for x in g_w]),
        L.ptr_array([x.data_ptr() if x is not None else None for x in g_b]), ws.data_ptr(), ws.numel(),
        ENGINE_ID[engine], _stream())
    torch.cuda.synchronize()
    return rc, g_src, g_w, g_b


FLIPS = {}   # engine -> [elements of rounded intermediates, elements with a rounding boundary in their band]


def _flip(engine, st):
    f = FLIPS.setdefault(engine, [0, 0])
    f[0] += st.n
    f[1] += st.flip


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(DIFF_CASES))
def test_diffusion_bwd_and_from_basis(lib, case):
    V, K, C = DIFF_CASES[case]
    sm = _sm(lib)
    a = diffusion_inputs(V, K, C)
    grad_out, mass, evals, evecs, time, x_spec = a
    rep = Report("diffusion_bwd/{}".format(case))
    cache = {}
    for engine in B.ENGINES:
        rc, gx, gt = run_diffusion_bwd(lib, engine, *a)
        assert rc == 0, (engine, rc)
        st = B.Stats()
        (gxb, gtb) = B.diffusion_bwd(*a, engine, sm=sm, grad_time_init=np.full(C, GRAD_T_INIT), stats=st, cache=cache)
        _flip(engine, st)
        rep(engine + " grad_x", gx[:V], gxb)
        rep(engine + " grad_time", gt, gtb)
        rep.nan_rows(engine + " grad_x", gx, V)
        # dn_from_basis with row_scale on exact inputs (the primitive the diffusion backward ends in)
        rc, out = run_from_basis(lib, engine, x_spec, evecs, mass)
        assert rc == 0, (engine, rc)
        rep(engine + " from_basis", out[:V], B.from_basis(x_spec, evecs, mass, engine))
        rep.nan_rows(engine + " from_basis", out, V)
    rep.done()


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(MLP_CASES))
def test_mini_mlp_bwd(lib, case):
    V, C, hidden, p, has_bias = MLP_CASES[case]
    sm = _sm(lib)
    grad_out, srcs, weights, hid, drops, dims = mlp_inputs(V, C, hidden, p)
    rep = Report("mini_mlp_bwd/{}".format(case))
    init = [np.full(w.shape, GRAD_W_INIT) for w in weights]
    for engine in B.ENGINES:
        rc, g_src, g_w, g_b = run_mini_mlp_bwd(lib, engine, grad_out, srcs, weights, hid, drops, has_bias)
        assert rc == 0, (engine, rc)
        st = B.Stats()
        gold = B.mini_mlp_bwd(grad_out, srcs, weights, hid, drops, engine, sm=sm, grad_w_init=init,
                              has_bias=has_bias, stats=st, grad_b_init=GRAD_B_INIT)
        _flip(engine, st)
        for q in range(3):
            rep("{} grad_src{}".format(engine, q), g_src[q][:V], gold["src"][q])
            rep.nan_rows("{} grad_src{}".format(engine, q), g_src[q], V)
        for l in range(len(weights)):
            rep("{} grad_W{}".format(engine, l), g_w[l], gold["w"][l])
            if gold["b"][l] is not None:
                rep("{} grad_b{}".format(engine, l), g_b[l], gold["b"][l])
            else:
                assert g_b[l] is None
    rep.done()


def run_features_bwd(lib, engine, a, V, C):
    import diffusion_net_b200 as d
    rot = a["A_im"] is not None
    idx = torch.from_numpy(np.stack([a["rows"], a["cols"]]))
    coo = lambda v: torch.sparse_coo_tensor(idx, torch.from_numpy(v), (V, V)).coalesce().cuda()
    gops = d.ops.GradOperators(coo(a["gx"]), coo(a["gy"]))
    csr_t = gops.csr_t
    ins = [_dev(a[k]) for k in ("grad_features", "x_diffuse", "pq", "features", "A_re")]
    a_im = _dev(a["A_im"]) if rot else None
    gx = _nan_buf(V, C)
    g_re = torch.full((C, C), GRAD_W_INIT, device="cuda")
    g_im = torch.full((C, C), GRAD_W_INIT, device="cuda") if rot else None
    ws = _ws(V, 8 * C)
    rc = lib.dn_gradient_features_bwd(ctypes.byref(gops.csr[0]), ctypes.byref(csr_t[0]),
                                      *[t.data_ptr() for t in ins], a_im.data_ptr() if rot else None, 1 if rot else 0,
                                      V, C, gx.data_ptr(), g_re.data_ptr(), g_im.data_ptr() if rot else None,
                                      ws.data_ptr(), ws.numel(), ENGINE_ID[engine], _stream())
    torch.cuda.synchronize()
    return rc, gx, g_re, g_im


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(FEAT_CASES))
def test_gradient_features_bwd(lib, case):
    """grad_x = dxd + dP A_re + dQ A_im (two weight blocks over two sources, dxd the residual), grad_A_re / grad_A_im
    accumulated into a prefilled buffer; dxd, dP and dQ are the gather's fp32 intermediates, carried with their band."""
    n, m, C, rot = FEAT_CASES[case]
    V = n * m
    sm = _sm(lib)
    gX, gY, a = features_inputs(n, m, C, rot)
    rep = Report("features_bwd/{}".format(case))
    init = [np.full((C, C), GRAD_W_INIT)] * 2
    for engine in B.ENGINES:
        rc, gx, g_re, g_im = run_features_bwd(lib, engine, a, V, C)
        assert rc == 0, (engine, rc)
        st = B.Stats()
        gold = B.gradient_features_bwd(gX, gY, a["grad_features"], a["x_diffuse"], a["pq"], a["features"], a["A_re"],
                                       a["A_im"], engine, sm=sm, grad_A_init=init, stats=st)
        _flip(engine, st)
        rep(engine + " grad_x", gx[:V], gold[0])
        rep.nan_rows(engine + " grad_x", gx, V)
        rep(engine + " grad_A_re", g_re, gold[1])
        if rot:
            rep(engine + " grad_A_im", g_im, gold[2])
    rep.done()


# ragged mesh batches: (rows of each mesh, K, C)
BATCH_CASES = {"ragged3_k64_c64": ([700, 129, 2000], 64, 64), "ragged4_k128_c128": ([1, 4000, 383, 1280], 128, 128)}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(BATCH_CASES))
def test_diffusion_bwd_batched(lib, case):
    """dn_learned_time_diffusion_bwd_batched on a ragged MeshBatch against each mesh's emulated gold; the time gradient
    is the sum over the meshes; padding rows of grad_x are exactly 0."""
    import diffusion_net_b200 as d
    rows, K, C = BATCH_CASES[case]
    sm = _sm(lib)
    meshes = [diffusion_inputs(v, K, C, seed=SEED + i) for i, v in enumerate(rows)]
    time = meshes[0][4]
    eye = lambda v: torch.sparse_coo_tensor(torch.arange(v).repeat(2, 1), torch.ones(v), (v, v)).cuda()
    items = [dict(mass=_dev(mi[1]), evals=_dev(mi[2]), evecs=_dev(mi[3]), gradX=eye(v), gradY=eye(v))
             for mi, v in zip(meshes, rows)]
    mb = d.MeshBatch(items)
    tb = mb._tb_rows.cpu().numpy().reshape(-1, 2)
    split = (len(tb), int((tb[:, 1] - tb[:, 0]).max()))    # every CTA of the plan, its longest row range
    # spectral_time_grad_batched sums n_meshes K terms as (n_meshes K / 16 + 16) sequential adds: within the per-mesh
    # bound's (K + 4) u sum |terms|, summed over the meshes
    assert len(rows) * K / 16 + 17 <= K + 4
    V = mb.V
    g = mb.pack([torch.from_numpy(mi[0]).cuda() for mi in meshes])
    xs = torch.from_numpy(np.concatenate([mi[5] for mi in meshes])).cuda()
    t = _dev(time)
    rep = Report("diffusion_bwd_batched/{}".format(case))
    for engine in ("tc3x", "tc1x", "bf16"):
        gx = torch.full((V, C), float("nan"), device="cuda")
        gt = torch.full((C,), GRAD_T_INIT, device="cuda")
        ws = _ws(V, 2 * C)
        rc = lib.dn_learned_time_diffusion_bwd_batched(
            g.data_ptr(), mb.mass.data_ptr(), mb.evals.data_ptr(), mb.evecs.data_ptr(), t.data_ptr(), xs.data_ptr(),
            ctypes.byref(mb.desc), V, K, C, gx.data_ptr(), gt.data_ptr(), ws.data_ptr(), ws.numel(),
            ENGINE_ID[engine], _stream())
        torch.cuda.synchronize()
        assert rc == 0, (engine, rc)
        gt_gold, U0 = np.full(C, GRAD_T_INIT), np.zeros(C)
        for b, mi in enumerate(meshes):
            (gxb, (gtv, gte)) = B.diffusion_bwd(*mi[:4], time, mi[5], engine, sm=sm, split=split)   # one time vector
            r0, nb = mb.row_begin[b], rows[b]
            rep("{} grad_x mesh {}".format(engine, b), gx[r0:r0 + nb], gxb)
            pad = gx[r0 + nb:mb.row_begin[b + 1]]
            if not bool((pad == 0).all()):
                rep.misses.append("{} mesh {}: padding rows of grad_x are not exactly 0".format(engine, b))
            gt_gold = gt_gold + gtv
            U0 = U0 + gte
        rep(engine + " grad_time", gt, (gt_gold, U0 + B.U * np.abs(gt_gold)))
    rep.done()


@pytest.mark.gpu
def test_flip_allowance_fraction():
    """Of the rounded intermediates' elements (dS, the deeper layers' dz), the share whose band holds a rounding
    boundary of the engine's format -- the elements where the bound pays for a possible flip."""
    if not FLIPS:
        pytest.skip("runs after the cases above")
    for engine, (n, k) in sorted(FLIPS.items()):
        if n:
            print("[measured] flip allowance {}: {} of {} elements ({:.3%})".format(engine, k, n, k / n))


@pytest.mark.gpu
@pytest.mark.parametrize("V,K,C", [(7000, 128, 128), (713, 12, 48), (200037, 64, 32)])
def test_bf16_engine_to_basis_is_tc1x(lib, V, K, C):
    """to_basis runs single-pass TF32 under the bf16 engine: bitwise tc1x's result."""
    _, mass, _, evecs, _, _ = diffusion_inputs(V, K, C)
    x = _dev(np.random.RandomState(3).randn(V, C).astype(np.float32))
    m, e = _dev(mass), _dev(evecs)
    outs = []
    for engine in ("tc1x", "bf16"):
        out = torch.empty(K, C, device="cuda")
        ws = _ws(V, C)
        assert lib.dn_to_basis(x.data_ptr(), e.data_ptr(), m.data_ptr(), V, K, C, out.data_ptr(), ws.data_ptr(),
                               ws.numel(), ENGINE_ID[engine], _stream()) == 0
        outs.append(out.cpu())
    assert torch.equal(outs[0], outs[1])


def route_table():
    """{case/engine: True if every contraction of the case stays on tensor cores} from the oracle's route table."""
    want = {}
    for engine in ("tc3x", "tc1x", "bf16"):
        for name, (V, K, C) in DIFF_CASES.items():
            r = B.routes(engine, V, K, C, [3 * C, C])
            want["diff/{}/{}".format(name, engine)] = "simt" not in (r["diffusion/to_basis"], r["diffusion/from_basis"])
        for name, (V, C, hidden, p, hb) in MLP_CASES.items():
            r = B.routes(engine, V, 40, C, [3 * C] + hidden + [C])
            want["mlp/{}/{}".format(name, engine)] = "simt" not in [v for k, v in r.items() if k.startswith("mlp/")]
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
            rc = run_diffusion_bwd(lib, engine, *diffusion_inputs(V, K, C))[0]
        else:
            V, C, hidden, p, hb = MLP_CASES[name]
            V = min(V, 1000)
            g, s, w, h, dr, _ = mlp_inputs(V, C, hidden, p)
            rc = run_mini_mlp_bwd(lib, engine, g, s, w, h, dr, hb)[0]
        got[key] = rc == 0
    print(json.dumps(got))


@pytest.mark.gpu
def test_routes_under_strict_tc(lib):
    tests_dir = os.path.join(ROOT, "tests")
    env = dict(os.environ, DN_STRICT_TC="1")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", "import sys; sys.path[:0] = [{!r}, {!r}]; import test_gpu_backward_engines as t; t._route_report()".format(
            tests_dir, ROOT)]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    want = route_table()
    assert got == want, {k: (got.get(k), want[k]) for k in want if got.get(k) != want[k]}
