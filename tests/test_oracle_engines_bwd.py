"""The backward restatement of oracle/dn_oracle_engines_bwd.py on the CPU: unrounded, it is fp64 autograd of the same
operations; its route table is dn_capi.cu's dispatch; and each structural error a backward kernel could make exceeds
the componentwise bound of tests/test_gpu_backward_engines.py by >= 100x on at least one case per engine where it
applies (exceptions named below with their measured factor)."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle_engines_bwd as B  # noqa: E402  (checker only)
from test_gpu_backward_engines import (DIFF_CASES, FEAT_CASES, GRAD_B_INIT, GRAD_T_INIT, GRAD_W_INIT, MLP_CASES,  # noqa: E402
                                      diffusion_inputs, features_inputs, mlp_inputs)

D = torch.float64
SM = 132      # H100 SXM


def _rel(a, b):
    return float(np.abs(np.asarray(a) - b.detach().numpy()).max() / max(float(b.abs().max()), 1e-300))


@pytest.mark.parametrize("case", ["k12", "c40", "v129", "k160"])
def test_unrounded_diffusion_bwd_is_fp64_autograd(case):
    V, K, C = DIFF_CASES[case]
    g, mass, evals, evecs, time, x_spec = diffusion_inputs(V, K, C)
    (gx, _), (gt, _) = B.diffusion_bwd(g, mass, evals, evecs, time, x_spec, "simt", sm=SM)
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    x = t(np.random.RandomState(0).randn(V, C)).requires_grad_(True)
    tt = t(time).clamp(min=1e-8).requires_grad_(True)
    E, lam, m = t(evecs), t(evals), t(mass)
    spec = E.t() @ (x * m[:, None])
    out = E @ (torch.exp(-lam[:, None] * tt[None, :]) * spec)
    out.backward(t(g))
    # the kernel's time gradient reads the saved x_spec: autograd's is at spec, so feed it the same spectrum
    tt2 = t(time).clamp(min=1e-8).requires_grad_(True)
    (E @ (torch.exp(-lam[:, None] * tt2[None, :]) * t(x_spec))).backward(t(g))
    assert _rel(gx, x.grad) <= 1e-12
    assert _rel(gt, tt2.grad) <= 1e-12


@pytest.mark.parametrize("case", ["depth1_v129", "depth3_v127_p05", "depth9_layer_by_layer", "bias_none"])
def test_unrounded_mini_mlp_bwd_is_fp64_autograd(case):
    V, C, hidden, p, hb = MLP_CASES[case]
    g, srcs, weights, hid, drops, dims = mlp_inputs(V, C, hidden, p)
    res = B.mini_mlp_bwd(g, srcs, weights, hid, drops, "simt", sm=SM, has_bias=hb)
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    s6 = [t(s).requires_grad_(True) for s in srcs]
    w6 = [t(w).requires_grad_(True) for w in weights]
    b6 = [torch.zeros(w.shape[0], dtype=D, requires_grad=True) for w in weights]
    h = torch.cat(s6, 1)
    for i in range(len(w6)):
        h = h @ w6[i].t() + b6[i]
        if i + 1 < len(w6):
            # the next layer reads the saved activation; the gradient passes its relu mask and the dropout mask
            h = t(hid[i]) + (h - h.detach()) * (t(hid[i]) > 0).to(D) * (t(drops[i]) if drops else 1.0)
    h.backward(t(g))
    for q in range(3):
        assert _rel(res["src"][q][0], s6[q].grad) <= 1e-12
    for i in range(len(w6)):
        assert _rel(res["w"][i][0], w6[i].grad) <= 1e-12
        if hb is None or hb[i]:
            assert _rel(res["b"][i][0], b6[i].grad) <= 1e-12


# dn_capi.cu's dispatch, read off its conditions: to_basis_partials (tensor cores iff K % 4 == 0, 4 <= K <= 128 and C
# in 16..128 on the 16 grid, or C a multiple of 128 in 128-column slices), run_chain on one layer (tc_chain_plan: bf16
# where K % 16 == 0, TF32 where K % 8 == 0, N % 16 == 0, 16 <= N <= 256), atb (to_basis's shape rule without slices)
EXPECTED_ROUTES = [
    ("tc3x", 2000, 160, 96, None, {"diffusion/to_basis": "simt", "diffusion/from_basis": "3x"}),
    ("tc3x", 1230, 64, 40, [120, 40, 40], {"diffusion/to_basis": "simt", "diffusion/from_basis": "simt",
                                           "mlp/atb0": "simt", "mlp/dx0": "simt", "mlp/dx1": "simt"}),
    ("tc1x", 4980, 128, 256, [768, 256, 256], {"diffusion/to_basis": "1x", "diffusion/from_basis": "1x",
                                                "mlp/atb1": "simt", "mlp/dx1": "1x"}),
    ("bf16", 700, 8, 48, None, {"diffusion/to_basis": "1x", "diffusion/from_basis": "1x"}),
    ("bf16", 700, 40, 128, None, {"diffusion/to_basis": "1x", "diffusion/from_basis": "1x"}),
    ("bf16", 7000, 128, 128, [384, 128, 128], {"diffusion/to_basis": "1x", "diffusion/from_basis": "bf16",
                                                "mlp/atb0": "1x", "mlp/dx0": "bf16", "mlp/dx1": "bf16"}),
    ("bf16", 713, 12, 48, [144, 40, 48], {"diffusion/to_basis": "1x", "diffusion/from_basis": "simt",
                                           "mlp/atb1": "simt", "mlp/dx1": "simt", "mlp/dx0": "1x"}),
    ("tc1x", 700, 256, 48, None, {"diffusion/to_basis": "simt", "diffusion/from_basis": "1x"}),
    ("simt", 7000, 128, 128, [384, 128, 128], {"diffusion/to_basis": "simt", "mlp/atb0": "simt", "mlp/dx1": "simt"}),
]


@pytest.mark.parametrize("engine,V,K,C,dims,want", EXPECTED_ROUTES)
def test_route_table_is_the_capi_dispatch(engine, V, K, C, dims, want):
    r = B.routes(engine, V, K, C, dims or [3 * C, C], sm=SM)
    assert {k: r[k] for k in want} == want


# ---- sensitivity ----------------------------------------------------------------------------------------------------
SENS_DIFF = ["tiny", "k12", "c40", "v129", "v7000", "k8", "c128_k40"]
SENS_MLP = [n for n, c in MLP_CASES.items() if c[0] <= 7000]
# dn_gradient_features_bwd: every FEAT_CASES entry (V <= 7056)
# (engine, perturbation) -> the best factor over the cases, measured, where it is below 100 (asserted as stated):
#   no_clamp@1e-9: exp(-lambda 1e-9) and exp(-lambda 1e-8) differ by lambda * 9e-9 <= 1.8e-6 relative, below every
#   engine's accumulation bound (K u ~ 1.5e-5 on grad_time; the TF32 / bf16 rounding of dS on grad_x)
BELOW_100 = {("simt", "no_clamp@1e-9"): 0.01, ("tc3x", "no_clamp@1e-9"): 0.01, ("tc1x", "no_clamp@1e-9"): 0.003,
             ("bf16", "no_clamp@1e-9"): 0.003}


def _factor(gold_bound, pert):
    (g, b), (p, _) = gold_bound, pert
    d = np.abs(p - g)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(b > 0, d / b, np.where(d > 0, np.inf, 0.0))
    return float(r.max()) if r.size else 0.0


def _diffusion_outputs(a, engine, pert=()):
    (gx, gt) = B.diffusion_bwd(*a, engine, sm=SM, grad_time_init=np.full(a[0].shape[1], GRAD_T_INIT), pert=pert)
    fb = B.from_basis(a[5], a[3], a[1], engine, pert=pert)
    return {"grad_x": gx, "grad_time": gt, "from_basis": fb}


def _mlp_outputs(a, hb, engine, pert=()):
    g, srcs, weights, hid, drops, dims = a
    init = [np.full(w.shape, GRAD_W_INIT) for w in weights]
    r = B.mini_mlp_bwd(g, srcs, weights, hid, drops, engine, sm=SM, grad_w_init=init, has_bias=hb, pert=pert,
                       grad_b_init=GRAD_B_INIT)
    out = {"src%d" % q: r["src"][q] for q in range(3)}
    out.update({"W%d" % l: r["w"][l] for l in range(len(weights))})
    out.update({"b%d" % l: r["b"][l] for l in range(len(weights)) if r["b"][l] is not None})
    return out


def test_structural_errors_exceed_the_backward_bound():
    best = {}

    def note(engine, p, f):
        best[(engine, p)] = max(best.get((engine, p), 0.0), f)

    for name in SENS_DIFF:
        V, K, C = DIFF_CASES[name]
        a = diffusion_inputs(V, K, C)
        for engine in B.ENGINES:
            gold = _diffusion_outputs(a, engine)
            r = B.routes(engine, V, K, C, [3 * C, C], sm=SM)
            modes = {r["diffusion/to_basis"], r["diffusion/from_basis"]}
            perts = ["drop_eig", "no_clamp"] + (["row_scale_last_tile"] if V % 128 else [])
            perts += {"bf16": ["1x_for_bf16"] if "bf16" in modes else [], "tc3x": ["1x_for_3x"]}.get(engine, [])
            perts += ["bf16_for_1x"] if engine == "bf16" else []
            for p in perts:
                y = _diffusion_outputs(a, engine, pert={p})
                if p == "no_clamp":
                    for col, label in ((0, "no_clamp@-0.1"), (2, "no_clamp@1e-9")):
                        f = max(_factor((gold[k][0][..., col], gold[k][1][..., col]), (y[k][0][..., col], None))
                                for k in gold)
                        note(engine, label, f)
                        print("[measured] diffusion/{}/{}/{} factor={:.3g}".format(name, engine, label, f))
                    continue
                f = max(_factor(gold[k], y[k]) for k in gold)
                note(engine, p, f)
                print("[measured] diffusion/{}/{}/{} factor={:.3g}".format(name, engine, p, f))
    for name in SENS_MLP:
        V, C, hidden, pdrop, hb = MLP_CASES[name]
        a = mlp_inputs(V, C, hidden, pdrop)
        for engine in B.ENGINES:
            gold = _mlp_outputs(a, hb, engine)
            dims = a[5]
            r = B.routes(engine, V, 40, C, dims, sm=SM)
            modes = set(r.values())
            P = max(B.atb_split(r["mlp/atb%d" % l], V, dims[l + 1], dims[l] if l else C, SM, B.PARTIAL_FLOATS // 2)[0]
                    for l in range(len(dims) - 1))
            perts = ["wrong_w0_block", "accumulate0"] + (["drop_last_partial"] if P > 1 else [])
            perts += ["relu_mask_last_tile"] if V % 128 and hidden else []
            perts += ["dropout_col"] if pdrop > 0 else []
            perts += {"bf16": (["1x_for_bf16"] if "bf16" in modes else []) + (["bf16_for_1x"] if "1x" in modes else []),
                      "tc3x": ["1x_for_3x"] if "3x" in modes else []}.get(engine, [])
            for p in perts:
                y = _mlp_outputs(a, hb, engine, pert={p})
                f = max(_factor(gold[k], y[k]) for k in gold)
                note(engine, p, f)
                print("[measured] mlp/{}/{}/{} factor={:.3g}".format(name, engine, p, f))
    for name, (n, m, C, rot) in FEAT_CASES.items():
        gX, gY, a = features_inputs(n, m, C, rot)
        args = (gX, gY, a["grad_features"], a["x_diffuse"], a["pq"], a["features"], a["A_re"], a["A_im"])
        init = [np.full((C, C), GRAD_W_INIT)] * 2
        V = n * m
        for engine in B.ENGINES:
            outs = lambda pert=(): [o for o in B.gradient_features_bwd(*args, engine, sm=SM, grad_A_init=init,
                                                                        pert=pert) if o is not None]
            gold = outs()
            r = B.routes(engine, V, 40, C, [3 * C, C], sm=SM)
            modes = {r["features/dx" if rot else "features/dx_norot"], r["features/atb"]}
            P = B.atb_split(r["features/atb"], V, C, C, SM, B.PARTIAL_FLOATS // 4)[0]
            perts = ["drop_dxd", "accumulate0"] + (["drop_dq_a_im"] if rot else []) + (
                ["drop_last_partial"] if P > 1 else [])
            perts += {"bf16": (["1x_for_bf16"] if "bf16" in modes else []) + (["bf16_for_1x"] if "1x" in modes else []),
                      "tc3x": ["1x_for_3x"] if "3x" in modes else []}.get(engine, [])
            for p in perts:
                y = outs({p})
                f = max(_factor(gb, yb) for gb, yb in zip(gold, y))
                note(engine, p, f)
                print("[measured] features/{}/{}/{} factor={:.3g}".format(name, engine, p, f))
    misses = []
    print("[measured] best factor per engine and structural error:")
    for (engine, p), f in sorted(best.items()):
        need = min(100.0, BELOW_100.get((engine, p), 100.0))
        print("[measured]   {:5s} {:22s} {:.3g}".format(engine, p, f))
        if not f >= need:
            misses.append("{}/{}: {:.3g} < {}".format(engine, p, f, need))
    assert not misses, misses
