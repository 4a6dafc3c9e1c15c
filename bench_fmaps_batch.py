#!/usr/bin/env python
"""Benchmark of the functional-map model over pair batches (fmaps.PairBatch, forward_pairs, pointwise_map_batch) on one
GPU.  Prints one JSON line per measurement, the first one naming the card and its power limit.

Shapes: S = 20 synthetic shapes of 5000 .. 5400 vertices (synthetic.structural_operators, K = 128 eigenpairs), a 4 x 128
feature net (FunctionalMapCorrespondenceWithDiffusionNetFeatures, n_fmap = 30), tc3x, dropout off (eval mode).

  * training: forward + backward of sum_p mean((C_pred[p] - C_gt)^2) for P in {1, 8, 32, 128} pairs drawn from the 20
    shapes, in ms per pair (the batch holds all 20 shapes, features included, except at P = 1, where it holds the
    pair's two shapes):
      - ``pair_graphed``: one graphs.GraphedTrainStep per pair, replayed in a loop (the fastest per-pair route).  Its
        per-pair cost does not depend on P, so it is measured once over 16 pairs (a graph per pair holds its own
        activations) and reported beside every P;
      - ``batch_eager``: one eager step over forward_pairs;
      - ``batch_graphed``: the same step under graphs.GraphedTrainStep;
  * evaluation: all 190 pairs of the 20 shapes (itertools.combinations), C and the pointwise map of every pair:
      - ``pair_loop``: forward + pointwise_map per pair;
      - ``batch``: forward_pairs + pointwise_map_batch.
Peak memory (torch.cuda.max_memory_allocated over the timed route) is reported beside each row.

    python bench_fmaps_batch.py [--steps 10] [--warmup 3] [--pairs 1,8,32,128]
"""
from __future__ import annotations

import argparse
import itertools
import json
import os
import random
import subprocess
import sys

import torch

sys.dont_write_bytecode = True      # the tree may be read-only; nothing is cached in it
ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import diffusion_net_b200 as dn  # noqa: E402

N_SHAPES = 20
K_EIG = 128
N_FMAP = 30


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
    torch.cuda.reset_peak_memory_stats()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps, torch.cuda.max_memory_allocated() / 2 ** 20


def shapes():
    items, xs, tuples = [], [], []
    for s in range(N_SHAPES):
        n, m = 50 + s % 5, 100 + 2 * (s % 3)
        mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K_EIG, seed=s, device="cuda")
        x = torch.randn(n * m, 3, generator=torch.Generator().manual_seed(100 + s)).cuda()
        items.append({"mass": mass, "evals": evals, "evecs": evecs, "gradX": gX, "gradY": gY})
        xs.append(x)
        tuples.append([x, None, None, mass, None, evals, evecs, gX, gY, None, None])
    return items, xs, tuples


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pairs", default="1,8,32,128")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fmaps_batch.py needs a GPU")
    name, pl = card()
    emit(card=name, power_limit=pl, engine="tc3x", shapes=N_SHAPES, k_eig=K_EIG, n_fmap=N_FMAP)
    dn.set_engine("tc3x")
    torch.manual_seed(0)
    model = dn.FunctionalMapCorrespondenceWithDiffusionNetFeatures(n_feat=128, input_features="xyz").cuda().eval()
    items, xs, tuples = shapes()
    C_gt = (torch.randn(N_FMAP, N_FMAP, generator=torch.Generator().manual_seed(1)) * 0.1).cuda()
    rng = random.Random(0)
    all_pairs = list(itertools.permutations(range(N_SHAPES), 2))

    # ---- training ----
    def pair_loss(net, s1, s2, c):
        C_pred, _, _ = net(s1, s2)
        return torch.mean(torch.square(C_pred.squeeze(0) - c))

    def batch_loss(net, pb, inputs, c):
        C_pred, _ = net.forward_pairs(pb, inputs)
        return torch.square(C_pred - c).mean(dim=(1, 2)).sum()

    loop_pairs = rng.sample(all_pairs, 16)
    steps_pp = [dn.graphs.GraphedTrainStep(model, pair_loss, (tuples[a], tuples[b], C_gt)) for a, b in loop_pairs]

    def pair_graphed():
        for st in steps_pp:
            st.replay()
    ms, mem = time_ms(pair_graphed, args.steps, args.warmup)
    pair_ms = ms / len(steps_pp)
    emit(bench="train", route="pair_graphed", pairs=len(steps_pp), ms_per_pair=round(pair_ms, 4),
         peak_mib=round(mem, 1))
    del steps_pp
    torch.cuda.empty_cache()

    for P in [int(p) for p in args.pairs.split(",")]:
        pairs = rng.sample(all_pairs, P)
        its, ins = items, xs
        if P == 1:
            (a, b), = pairs
            its, ins, pairs = [items[a], items[b]], [xs[a], xs[b]], [(0, 1)]
        pb = dn.PairBatch(its, pairs)

        def eager():
            batch_loss(model, pb, ins, C_gt).backward()
        ms_e, mem_e = time_ms(eager, args.steps, args.warmup)
        emit(bench="train", route="batch_eager", pairs=P, ms_per_step=round(ms_e, 3), ms_per_pair=round(ms_e / P, 4),
             speedup_vs_pair_graphed=round(pair_ms * P / ms_e, 3), peak_mib=round(mem_e, 1))
        step = dn.graphs.GraphedTrainStep(model, batch_loss, (pb, ins, C_gt))
        ms_g, mem_g = time_ms(step.replay, args.steps, args.warmup)
        emit(bench="train", route="batch_graphed", pairs=P, ms_per_step=round(ms_g, 3), ms_per_pair=round(ms_g / P, 4),
             speedup_vs_pair_graphed=round(pair_ms * P / ms_g, 3), peak_mib=round(mem_g, 1))
        del step, pb
        torch.cuda.empty_cache()

    # ---- evaluation ----
    ev_pairs = list(itertools.combinations(range(N_SHAPES), 2))
    pb = dn.PairBatch(items, ev_pairs)

    def eval_loop():
        with torch.no_grad():
            for a, b in ev_pairs:
                C_pred, _, _ = model(tuples[a], tuples[b])
                dn.pointwise_map(C_pred, items[a]["evecs"], items[b]["evecs"], n_fmap=N_FMAP)

    def eval_batch():
        with torch.no_grad():
            C_pred, _ = model.forward_pairs(pb, xs)
            dn.pointwise_map_batch(C_pred, pb, n_fmap=N_FMAP)
    ev_steps = max(1, args.steps // 5)
    ms_l, mem_l = time_ms(eval_loop, ev_steps, 1)
    emit(bench="eval", route="pair_loop", pairs=len(ev_pairs), ms=round(ms_l, 2), peak_mib=round(mem_l, 1))
    ms_b, mem_b = time_ms(eval_batch, ev_steps, 1)
    emit(bench="eval", route="batch", pairs=len(ev_pairs), ms=round(ms_b, 2), speedup=round(ms_l / ms_b, 3),
         peak_mib=round(mem_b, 1))


if __name__ == "__main__":
    main()
