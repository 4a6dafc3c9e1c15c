#!/usr/bin/env python
"""Benchmark of the functional-map correspondence model (diffusion_net_b200/fmaps.py) on one GPU.  Prints one JSON line
per measurement, the first one naming the card and its power limit.

  * pair training step (forward + backward of mean((C_pred - C_gt)^2) over two 4 x 128 nets, n_fmap = 30, K = 128
    eigenpairs, dropout off) at V = 5k (FAUST-sized), 20k and 200k per shape, three routes:
      - ``reference_head``: our DiffusionNet features, then the reference's head as it is written (fmaps_model.py:79's
        dense ``evecs.t()[:30] @ torch.diag(mass)`` and ``compute_correspondence``), from the staged unmodified
        ``oracle/_ref/fmaps_model.py``; "oom" where the V x V matrix cannot be allocated;
      - ``eager``: FunctionalMapCorrespondenceWithDiffusionNetFeatures;
      - ``graphed``: the same under graphs.GraphedTrainStep;
  * the solve alone (n = 30, d = 128), forward + backward: dn_fmap_solve_* against the reference's torch loop;
  * pointwise_map at V_x = V_y = 5k, 20k, 200k (n = 30), with the search's work model: V_x V_y n difference-and-FMA
    steps, each two fp32 instructions (FADD + FFMA), against the H100 SXM data-sheet fp32 rate (67 TFLOP/s = 33.5 T
    FFMA/s per the 700 W card); at 5k also sklearn's KD-tree on the host, as the reference's evaluation runs it.

    python bench_fmaps.py [--steps 20] [--warmup 5] [--sizes 5000,20000,200000]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.dont_write_bytecode = True      # the tree may be read-only; nothing is cached in it
ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import diffusion_net_b200 as dn  # noqa: E402

GRIDS = {5000: (50, 100), 20000: (100, 200), 200000: (400, 500)}
N_FMAP = 30
FP32_INST_PER_S = 33.5e12


def emit(**kw):
    print(json.dumps(kw), flush=True)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:  # the number is reported beside what is known
        pl = "unknown ({})".format(e)
    return name, pl


def time_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def reference_head():
    """The staged, unmodified fmaps_model.py (its DiffusionNet import resolves to the staged reference package)."""
    import importlib.util
    from ref_import import import_reference
    import_reference()
    path = os.path.join(ROOT, "oracle", "_ref", "fmaps_model.py")
    if not os.path.isfile(path):
        return None
    spec = importlib.util.spec_from_file_location("fmaps_model", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def make_pair(V):
    n, m = GRIDS[V]
    shapes = []
    for seed in (0, 1):
        mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, 128, seed=seed, device="cuda")
        x = torch.randn(n * m, 3, generator=torch.Generator().manual_seed(seed)).cuda()
        shapes.append([x, None, None, mass, None, evals, evecs, gX, gY, None, None])
    return shapes


def bench_train(V, args, fm):
    torch.manual_seed(0)
    model = dn.FunctionalMapCorrespondenceWithDiffusionNetFeatures(n_feat=128, input_features="xyz").cuda().eval()
    s1, s2 = make_pair(V)
    C_gt = torch.randn(N_FMAP, N_FMAP, generator=torch.Generator().manual_seed(3)).cuda() * 0.2

    def loss_ours(net, a, b, c):
        C_pred, _, _ = net(a, b)
        return torch.mean(torch.square(C_pred.squeeze(0) - c))

    def loss_ref(net, a, b, c):
        fe = net.feature_extractor
        f1 = fe(a[0], a[3], evals=a[5], evecs=a[6], gradX=a[7], gradY=a[8])
        f2 = fe(b[0], b[3], evals=b[5], evecs=b[6], gradX=b[7], gradY=b[8])
        et1 = a[6].t()[:N_FMAP] @ torch.diag(a[3])                       # fmaps_model.py:79
        et2 = b[6].t()[:N_FMAP] @ torch.diag(b[3])
        C_pred = fm.compute_correspondence(f1, f2, a[5][:N_FMAP], b[5][:N_FMAP], et1, et2, lambda_param=1e-3)
        return torch.mean(torch.square(C_pred.squeeze(0) - c))

    res = {"V": V}
    if fm is None:
        res["reference_head_ms"] = "not measured (fmaps_model.py not staged)"
    else:
        try:
            res["reference_head_ms"] = time_ms(lambda: loss_ref(model, s1, s2, C_gt).backward(), args.steps, args.warmup)
        except torch.cuda.OutOfMemoryError:
            res["reference_head_ms"] = "oom"
        torch.cuda.empty_cache()
    res["eager_ms"] = time_ms(lambda: loss_ours(model, s1, s2, C_gt).backward(), args.steps, args.warmup)
    step = dn.graphs.GraphedTrainStep(model, loss_ours, (s1, s2, C_gt))
    res["graphed_ms"] = time_ms(step.replay, args.steps, args.warmup)
    res["peak_mem_gb"] = torch.cuda.max_memory_allocated() / 1e9
    emit(what="pair_train_step", **res)
    del step
    torch.cuda.empty_cache()


def bench_solve(args, fm):
    g = torch.Generator().manual_seed(0)
    n, d = N_FMAP, 128
    A = torch.randn(n, d, generator=g).cuda().requires_grad_(True)
    B = torch.randn(n, d, generator=g).cuda().requires_grad_(True)
    ex, ey = (torch.sort(torch.rand(n, generator=g) * 40)[0].cuda() for _ in range(2))
    G = torch.randn(n, n, generator=g).cuda()
    ours = time_ms(lambda: dn.fmaps.fmap_solve(A, B, ex, ey, 1e-3).backward(G), args.steps * 10, args.warmup)
    res = {"n": n, "d": d, "ours_ms": ours}
    if fm is not None:
        eye = torch.eye(n, device="cuda")
        ref = time_ms(lambda: fm.compute_correspondence(A, B, ex, ey, eye, eye)[0].backward(G),
                      args.steps * 10, args.warmup)
        res["reference_ms"] = ref
        res["speedup"] = ref / ours
    emit(what="fmap_solve_fwd_bwd", **res)


def bench_pointwise(V, args):
    s1, s2 = make_pair(V)
    C = torch.randn(N_FMAP, N_FMAP, generator=torch.Generator().manual_seed(4)).cuda()
    ex, ey = s1[6], s2[6]
    ms = time_ms(lambda: dn.pointwise_map(C, ex, ey, n_fmap=N_FMAP), max(3, args.steps // 4), 1)
    steps = float(V) * V * N_FMAP
    res = {"V": V, "n": N_FMAP, "ms": ms, "diff_fma_steps": steps, "steps_per_s": steps / (ms * 1e-3),
           "fp32_issue_bound_ms": 2 * steps / FP32_INST_PER_S * 1e3,
           "hbm_bytes_min": (2 * V * N_FMAP) * 4 + V * 8}
    res["share_of_fp32_issue_bound"] = res["fp32_issue_bound_ms"] / ms
    if V <= 5000:
        import sklearn.neighbors
        tgt = dn.fmaps._apply_basis_exact(C.t().contiguous(), ex[:, :N_FMAP].contiguous()).cpu().numpy()
        src = ey[:, :N_FMAP].cpu().numpy()
        t0 = time.perf_counter()
        tree = sklearn.neighbors.KDTree(tgt)
        _, kd = tree.query(src, k=1)
        res["sklearn_kdtree_host_ms"] = (time.perf_counter() - t0) * 1e3
        mine = dn.pointwise_map(C, ex, ey, n_fmap=N_FMAP).cpu().numpy()
        res["agree_with_kdtree"] = float((kd[:, 0] == mine).mean())
    emit(what="pointwise_map", **res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--sizes", default="5000,20000,200000")
    ap.add_argument("--skip-train", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_fmaps.py needs a GPU"
    name, pl = card()
    emit(what="device", name=name, power_limit=pl, engine=dn.get_engine())
    fm = reference_head()
    sizes = [int(s) for s in args.sizes.split(",")]
    bench_solve(args, fm)
    for V in sizes:
        bench_pointwise(V, args)
    if not args.skip_train:
        for V in sizes:
            bench_train(V, args, fm)


if __name__ == "__main__":
    main()
