"""The per-stage check of the fused block (tests/test_gpu_block_stages.py) on the CPU: its restatement of block_fwd_impl's
workspace carve fits the workspace the modules allocate (dn_workspace_bytes), ``tree_sum`` is the fp32 tree it says it
is, and each structural error the end-to-end metric of tests/test_gpu_forward.py misses on tc1x and bf16 (DESIGN.md
section 2) exceeds the per-stage bound >= 100x on some fused case, on every engine, as do three errors of the head in
the MiniMLP epilogue (exceptions named below with their measured factor)."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT
from test_gpu_backward_engines import BATCH_CASES
from test_gpu_block_stages import BIG, regions
from test_gpu_forward import CASES
from test_gpu_forward_engines import diffusion_fwd_inputs, mlp_fwd_inputs, torus_feat_inputs
from test_oracle_engines_fwd import SM, _factor

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle_engines as E  # noqa: E402  (checker only)
import dn_oracle_engines_bwd as B  # noqa: E402
import dn_oracle_engines_fwd as F  # noqa: E402


def _shapes():
    """(V, K, C, width, with_features, rot, n_meshes) of every block the GPU file calls."""
    for n, m, K, C, kw, hid, _ in [s for s in CASES.values()] + [s for s, _ in BIG.values()]:
        dims = [C] + list(hid if hid is not None else [C, C]) + [C]
        yield (n * m, K, C, max(dims[1:]), kw.get("with_gradient_features", True),
               kw.get("with_gradient_rotations", True), 0)
    for rows, K, C in BATCH_CASES.values():
        V = sum(-(-v // 128) * 128 for v in rows)
        yield V, K, C, C, True, True, len(rows)


def test_regions_fit_the_workspace():
    """The restated carve ends inside the workspace ops.workspace sizes for the block (the packed weights follow it)."""
    import diffusion_net_b200 as d
    lib = d._lib.load()
    for V, K, C, width, wgf, rot, nb in _shapes():
        end = regions(V, K, C, wgf, rot)["end"][0] * 4
        have = lib.dn_workspace_bytes(V, K, width) + nb * K * C * 8 + 4096
        assert end < have, (V, K, C, end, have)
        r = regions(V, K, C, wgf, rot)
        offs = [r[k][0] for k in ("S", "xd", "pq", "feat", "partial") if k in r]
        assert all(o % 64 == 0 for o in offs) and offs == sorted(offs)


@pytest.mark.parametrize("tree", [4, 8])
def test_tree_sum_is_the_fp32_tree(tree):
    rs = np.random.RandomState(tree)
    for P in (1, 3, tree, tree + 1, 132, 133):
        p = np.asarray(rs.randn(P, 5, 7) * np.exp(rs.uniform(-8, 8, (P, 1, 1))), np.float32)
        slices = [np.float32(0) * p[0] for _ in range(tree)]
        for q in range(P):
            slices[q % tree] = np.float32(slices[q % tree] + p[q])
        want = slices
        while len(want) > 1:
            want = [np.float32(want[i] + want[i + 1]) for i in range(0, len(want), 2)]
        got = F.tree_sum(p, tree)
        assert got.dtype == np.float32 and np.array_equal(got.view(np.int32), want[0].view(np.int32))
        exact = p.astype(np.float64).sum(0)
        L = -(-P // tree) + int(np.log2(tree))
        assert (np.abs(got - exact) <= L * B.U * np.abs(p.astype(np.float64)).sum(0)).all()


# ---- sensitivity ----------------------------------------------------------------------------------------------------
# the fused front cases of test_gpu_forward.CASES (the first: from_basis -> P -> Q with Q the sibling at C = 128;
# the second: one [P|Q] layer with W2; the third: P and Q as separate layers at C = 256), default MiniMLP [C, C]
SENS_CASES = ["c128_front_from_basis_p_q_fused", "c64_pq_one_layer_w2_split", "c256_p_q_split_two_slice_to_basis"]
BLOCK_PERTS = ("drop_eig", "drop_hidden_bias", "zero_channel", "swap_re_im")
# (engine, perturbation) -> the best factor over the cases, measured, where it is below 100 (asserted as stated)
BELOW_100 = {}


def _stage_outputs(name, engine, pert=()):
    """Every per-stage gold (gold, bound) of the GPU file at the case's shapes on the oracle's own inputs."""
    n, m, K, C, kw, hid, _ = CASES[name]
    V = n * m
    dims = [3 * C] + list(hid if hid is not None else [C, C]) + [C]
    d = E.dispatch(engine, K, C, dims)
    a = diffusion_fwd_inputs(V, K, C)
    g = F.diffusion_fwd(*a, engine, sm=SM, pert=pert, tree=8 if d["front_fused"] else 4, fb_mode=d["from_basis"])
    gX, gY, fa = torus_feat_inputs(n, m, C, True)
    f = F.features_fwd(gX, gY, fa["x_diffuse"], fa["A_re"], fa["A_im"], engine, pert=pert, mode=d["pq"][0])
    srcs, weights, biases, drops, r = mlp_fwd_inputs(V, C, dims[1:-1], 0.0, None, True)
    mo = F.mini_mlp_fwd(srcs, weights, biases, drops, r, engine, pert=pert)
    return [g["x_spec"], g["x_diffuse"], f["pq"], f["features"]] + mo["hidden"] + [mo["out"]], (mo["out"][0], r)


def test_structural_errors_exceed_the_stage_bound():
    best = {}
    for name in SENS_CASES:
        for engine in B.ENGINES:
            gold, (out, x_in) = _stage_outputs(name, engine)
            for p in BLOCK_PERTS:
                y, _ = _stage_outputs(name, engine, pert={p})
                fct = max(_factor(gb, yb) for gb, yb in zip(gold, y))
                best[(engine, p)] = max(best.get((engine, p), 0.0), fct)
                print("[measured] block/{}/{}/{} factor={:.3g}".format(name, engine, p, fct))
            for n_out in (1, 5, 8):
                rs = np.random.RandomState(100 + n_out)
                W = np.asarray(rs.randn(n_out, out.shape[1]) / np.sqrt(out.shape[1]), np.float32)
                b = np.asarray(rs.randn(n_out), np.float32)
                hg = F.head_fwd(out, W, b)
                for p in F.HEAD_PERTURBATIONS:
                    fct = _factor(hg, F.head_fwd(out, W, b, x_in=x_in, pert={p}))
                    best[(engine, p)] = max(best.get((engine, p), 0.0), fct)
                    print("[measured] head{}/{}/{}/{} factor={:.3g}".format(n_out, name, engine, p, fct))
    misses = []
    print("[measured] best factor per engine and structural error:")
    for (engine, p), fct in sorted(best.items()):
        need = min(100.0, BELOW_100.get((engine, p), 100.0))
        print("[measured]   {:5s} {:22s} {:.3g}".format(engine, p, fct))
        if not fct >= need:
            misses.append("{}/{}: {:.3g} < {}".format(engine, p, fct, need))
    assert not misses, misses
