"""The forward restatement of oracle/dn_oracle_engines_fwd.py on the CPU: unrounded, it is dn_oracle / plain fp64 of
the same operations; its route table is dn_oracle_engines.dispatch and agrees with the backward's; and each structural
error a forward kernel could make exceeds the componentwise bound of tests/test_gpu_forward_engines.py by >= 100x on at
least one case on every engine where it applies (exceptions named below with their measured factor)."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle as O  # noqa: E402  (checker only)
import dn_oracle_engines as E  # noqa: E402
import dn_oracle_engines_bwd as B  # noqa: E402
import dn_oracle_engines_fwd as F  # noqa: E402
from test_gpu_backward_engines import DIFF_CASES  # noqa: E402
from test_gpu_forward_engines import (FWD_FEAT_CASES, FWD_MLP_CASES, HKS_CASES, diffusion_fwd_inputs,  # noqa: E402
                                      hks_inputs, mlp_fwd_inputs, torus_feat_inputs)

SM = 132      # H100 SXM


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(float(np.abs(b).max()), 1e-300))


@pytest.mark.parametrize("case", ["tiny", "k12", "c40", "v129", "k160"])
def test_unrounded_diffusion_fwd_is_the_fp64_diffusion(case):
    V, K, C = DIFF_CASES[case]
    x, mass, evals, evecs, time = diffusion_fwd_inputs(V, K, C)
    g = F.diffusion_fwd(x, mass, evals, evecs, time, "simt", sm=SM)
    f = lambda a: np.asarray(a, np.float64)
    # the one rounding the restatement keeps unrounded: the fp32 product m * x every to_basis kernel forms first
    mx = f(np.float32(x) * np.float32(mass)[:, None])
    spec = O.to_basis(mx, f(evecs), np.ones(V))
    assert _rel(spec, O.to_basis(f(x), f(evecs), f(mass))) <= 1e-6
    assert _rel(g["x_spec"][0], spec) <= 1e-12
    t = np.maximum(f(time), 1e-8)
    assert _rel(g["x_diffuse"][0], O.from_basis(np.exp(-f(evals)[:, None] * t[None, :]) * spec, f(evecs))) <= 1e-12
    _, tc = O.learned_time_diffusion(f(x), f(mass), f(evals), f(evecs), f(time))
    assert _rel(g["time"], tc) <= 1e-12
    assert np.array_equal(g["time"], np.maximum(np.float32(time), np.float32(1e-8)))


@pytest.mark.parametrize("case", ["c48_rot", "c48_norot", "c3_rot", "c128_rot_long"])
def test_unrounded_features_fwd_is_the_fp64_features(case):
    n, m, C, rot, patched, lr = FWD_FEAT_CASES[case]
    gX, gY, a = torus_feat_inputs(n, m, C, rot, lr)
    g = F.features_fwd(gX, gY, a["x_diffuse"], a["A_re"], a["A_im"], "simt")
    xd = a["x_diffuse"].astype(np.float64)
    A_re = a["A_re"].astype(np.float64)
    A_im = a["A_im"].astype(np.float64) if rot else None
    P = xd @ A_re.T
    Q = xd @ A_im.T if rot else None
    assert _rel(g["pq"][0], np.hstack([P, Q]) if rot else P) <= 1e-12
    vec = O.grad_spmm(gX, gY, xd)
    want = O.spatial_gradient_features(vec, A_re, A_im) if rot else O.spatial_gradient_features(vec, A=A_re)
    assert _rel(g["features"][0], want) <= 1e-12


@pytest.mark.parametrize("case", ["depth1_v129", "depth3_v127_p05", "depth9_layer_by_layer", "bias_none",
                                  "residual_v7000"])
def test_unrounded_mini_mlp_fwd_is_the_fp64_mlp(case):
    V, C, hidden, p, hb, res = FWD_MLP_CASES[case]
    srcs, weights, biases, drops, r = mlp_fwd_inputs(V, C, hidden, p, hb, res)
    g = F.mini_mlp_fwd(srcs, weights, biases, drops, r, "simt")
    f = lambda a: np.asarray(a, np.float64)
    h = np.hstack([f(s) for s in srcs])
    if not drops and r is None:
        want = O.mini_mlp(h, [f(w) for w in weights], [f(b) if b is not None else 0.0 for b in biases])
        assert _rel(g["out"][0], want) <= 1e-12
    for l, w in enumerate(weights):
        z = h @ f(w).T + (f(biases[l]) if biases[l] is not None else 0)
        if l + 1 < len(weights):
            h = np.maximum(z, 0) * (f(drops[l]) if drops else 1.0)
            assert _rel(g["hidden"][l][0], h) <= 1e-12
        else:
            assert _rel(g["out"][0], z + (f(r) if r is not None else 0)) <= 1e-12


@pytest.mark.parametrize("case", ["k16_s16", "k96_s3", "k256_s17"])
def test_unrounded_hks_is_the_fp64_hks(case):
    V, K, S = HKS_CASES[case]
    V = min(V, 2000)
    evals, evecs, scales = hks_inputs(V, K, S)
    want = O.compute_hks(*[np.asarray(a, np.float64) for a in (evals, evecs, scales)])
    assert _rel(F.compute_hks(evals, evecs, scales)[0], want) <= 1e-12


def test_tanh_error_is_the_derivation():
    """Near 0 the documented errors add up to 7 * 2^-24 (expf 2 ulp through (1 - t^2) / 2, the add's half ulp and
    fdividef's 2 ulp through 1 - t); far out on the negative side the division's 2 (1 - t) doubles the latter."""
    T0 = F.tanh_error(0.0, 0.0)
    assert abs(T0 / (7 * 2.0 ** -24) - 1) < 1e-5
    assert F.tanh_error(-16.0, -16.0) > F.tanh_error(16.0, 16.0)
    assert F.tanh_error(-1.0, 1.0) >= max(F.tanh_error(-1.0, -1.0), F.tanh_error(1.0, 1.0), T0)
    # the sup over the whole range, which dn_simt.cu states for dn_feat_tanh
    x = np.linspace(-20, 20, 400001)
    assert 11.4 * 2.0 ** -24 < F.tanh_error(x, x).max() < 11.5 * 2.0 ** -24 < 6.9e-7


# dn_oracle_engines.dispatch / tc_chain_plan read off their conditions; the backward's route table where they overlap
@pytest.mark.parametrize("engine", B.ENGINES)
@pytest.mark.parametrize("K,C,dims", [(128, 128, [384, 128, 128]), (12, 48, [144, 40, 48]), (40, 40, [120, 40, 40]),
                                      (160, 96, [288, 96]), (8, 48, [144, 48]), (128, 256, [768, 256, 256]),
                                      (64, 64, [192] + [64] * 8 + [64])])
def test_route_table_is_the_dispatch(engine, K, C, dims):
    r = F.routes(engine, K, C, dims, sm=SM)
    d = E.dispatch(engine, K, C, dims)
    assert r["diffusion/to_basis"] == d["to_basis"]
    assert r["mlp/fused"] == d["mlp_fused"]
    assert [r["mlp/l%d" % l] for l in range(len(dims) - 1)] == d["mlp"]
    bw = B.routes(engine, 1000, K, C, dims, sm=SM)
    assert r["diffusion/to_basis"] == bw["diffusion/to_basis"]
    assert r["diffusion/from_basis"] == bw["diffusion/from_basis"]


EXPECTED_ROUTES = [   # the pq layer: tc_chain_plan on K = C, N = npq <= 256; bf16 where C % 16 == 0
    ("bf16", 40, {"features/pq": "1x", "features/pq_norot": "simt"}),
    ("bf16", 48, {"features/pq": "bf16", "features/pq_norot": "bf16"}),
    ("tc3x", 256, {"features/pq": "simt", "features/pq_norot": "3x"}),
    ("tc1x", 30, {"features/pq": "simt", "features/pq_norot": "simt"}),
    ("tc3x", 128, {"features/pq": "3x", "features/pq_norot": "3x"}),
    ("simt", 128, {"features/pq": "simt", "features/pq_norot": "simt"}),
]


@pytest.mark.parametrize("engine,C,want", EXPECTED_ROUTES)
def test_pq_route_is_the_chain_plan(engine, C, want):
    r = F.routes(engine, 64, C, [3 * C, C], sm=SM)
    assert {k: r[k] for k in want} == want


# ---- sensitivity ----------------------------------------------------------------------------------------------------
SENS_DIFF = ["tiny", "k12", "c40", "v129", "v7000", "k8", "c128_k40", "c20"]
SENS_FEAT = ["c48_rot", "c48_norot", "c40_rot", "c3_rot", "c6_norot", "c128_rot_long"]
SENS_MLP = ["depth1_v129", "depth2_v1", "depth2_v128", "depth3_v127_p05", "depth9_layer_by_layer", "c20_hidden40",
            "c40", "bias_none", "residual_v7000", "residual_depth3_v129", "c40_hidden48"]
SENS_HKS = ["k16_s16", "k96_s3", "k256_s17"]
# (engine, perturbation) -> the best factor over the cases, measured, where it is below 100 (asserted as stated)
BELOW_100 = {}


def _factor(gold_bound, pert):
    (g, b), (p, _) = gold_bound, pert
    d = np.abs(np.asarray(p, np.float64) - g)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(b > 0, d / b, np.where(d > 0, np.inf, 0.0))
    return float(r.max()) if r.size else 0.0


def _diff_outputs(a, engine, pert=()):
    g = F.diffusion_fwd(*a, engine, sm=SM, pert=pert)
    # "time" is checked bitwise: any difference counts as an infinite factor
    t = (g["time"].astype(np.float64), np.zeros(len(g["time"])))
    return {"x_spec": g["x_spec"], "x_diffuse": g["x_diffuse"], "time": t}


def test_structural_errors_exceed_the_forward_bound():
    best = {}

    def note(engine, p, f):
        best[(engine, p)] = max(best.get((engine, p), 0.0), f)

    for name in SENS_DIFF:
        V, K, C = DIFF_CASES[name]
        a = diffusion_fwd_inputs(V, K, C)
        for engine in B.ENGINES:
            gold = _diff_outputs(a, engine)
            r = F.routes(engine, K, C, [3 * C, C], sm=SM)
            tb = r["diffusion/to_basis"]
            P = B.atb_split(tb, V, K, C, SM, B.PARTIAL_FLOATS)[0]
            perts = ["drop_eig", "time_scaled", "no_clamp", "x_spec_scaled"] + (["drop_last_partial"] if P > 1 else [])
            perts += {"bf16": ["1x_for_bf16"] if r["diffusion/from_basis"] == "bf16" else [],
                      "tc3x": ["1x_for_3x"]}.get(engine, [])
            for p in perts:
                y = _diff_outputs(a, engine, pert={p})
                f = max(_factor(gold[k], y[k]) for k in gold)
                note(engine, p, f)
                print("[measured] diffusion/{}/{}/{} factor={:.3g}".format(name, engine, p, f))
    for name in SENS_FEAT:
        n, m, C, rot, patched, lr = FWD_FEAT_CASES[name]
        gX, gY, a = torus_feat_inputs(n, m, C, rot, lr)
        for engine in B.ENGINES:
            outs = lambda pert=(): F.features_fwd(gX, gY, a["x_diffuse"], a["A_re"], a["A_im"], engine, pert=pert)
            gold = outs()
            perts = ["drop_last_entry", "drop_gy_bim", "zero_channel", "tanh_2e-16"]
            perts += ["swap_re_im", "q_from_re"] if rot else []
            r = F.routes(engine, 40, C, [3 * C, C], sm=SM)
            pm = r["features/pq" if rot else "features/pq_norot"]
            perts += {"bf16": ["1x_for_bf16"] if pm == "bf16" else [], "tc3x": ["1x_for_3x"] if pm == "3x" else []
                      }.get(engine, [])
            for p in perts:
                y = outs({p})
                f = max(_factor(gold[k], y[k]) for k in ("pq", "features"))
                note(engine, p, f)
                print("[measured] features/{}/{}/{} factor={:.3g}".format(name, engine, p, f))
    for name in SENS_MLP:
        V, C, hidden, pdrop, hb, res = FWD_MLP_CASES[name]
        srcs, weights, biases, drops, r = mlp_fwd_inputs(V, C, hidden, pdrop, hb, res)
        dims = [3 * C] + hidden + [C]
        for engine in B.ENGINES:
            def outs(pert=()):
                g = F.mini_mlp_fwd(srcs, weights, biases, drops, r, engine, pert=pert)
                return g["hidden"] + [g["out"]]
            gold = outs()
            modes = set(E._mlp_modes([C] * 3, dims, B.PASSES[engine])[0])
            perts = ["relu_last", "wrong_w0_block"]
            perts += ["drop_hidden_bias"] if hidden and (hb is None or hb[0]) else []
            perts += ["hidden_before_emul", "dropout_col"] if pdrop > 0 and hidden else []
            perts += ["residual_last_tile"] if r is not None and V % 128 else []
            perts += {"bf16": (["1x_for_bf16"] if "bf16" in modes else []) + (["bf16_for_1x"] if "1x" in modes else []),
                      "tc3x": ["1x_for_3x"] if "3x" in modes else []}.get(engine, [])
            for p in perts:
                y = outs({p})
                f = max(_factor(gb, yb) for gb, yb in zip(gold, y))
                note(engine, p, f)
                print("[measured] mlp/{}/{}/{} factor={:.3g}".format(name, engine, p, f))
    for name in SENS_HKS:
        V, K, S = HKS_CASES[name]
        evals, evecs, scales = hks_inputs(min(V, 2000), K, S)
        gold = F.compute_hks(evals, evecs, scales)
        for p in F.PERTURBATIONS["hks"]:
            f = _factor(gold, F.compute_hks(evals, evecs, scales, pert={p}))
            note("simt", "hks/" + p, f)
            print("[measured] hks/{}/{} factor={:.3g}".format(name, p, f))
    misses = []
    print("[measured] best factor per engine and structural error:")
    for (engine, p), f in sorted(best.items()):
        need = min(100.0, BELOW_100.get((engine, p), 100.0))
        print("[measured]   {:5s} {:22s} {:.3g}".format(engine, p, f))
        if not f >= need:
            misses.append("{}/{}: {:.3g} < {}".format(engine, p, f, need))
    named = {p for ps in F.PERTURBATIONS.values() for p in ps}
    seen = {p.split("/")[-1] for _, p in best}
    assert named <= seen, named - seen
    assert not misses, misses
