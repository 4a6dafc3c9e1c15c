#!/usr/bin/env python
"""Benchmark of the functional-map model's shuffled training step (fmaps.PairDataset, PairSlot) on one GPU.  Prints
one JSON line per measurement, the first one naming the card, its power limit and its maximum SM clock.

Workload, FAUST-sized and synthetic: 80 shapes of 5000 .. 5406 vertices (synthetic.structural_operators, K = 128
eigenpairs), 6890 template correspondences per shape (random vertices, with repeats), every ordered pair of distinct
shapes allowed (6320 pairs, the reference's ``permutations(range(80), 2)``), the 4 x 128 feature net of
FunctionalMapCorrespondenceWithDiffusionNetFeatures (xyz input, n_fmap = 30) in training mode (dropout on), tc3x.
Every step draws fresh random pairs and a fresh random rotation per shape, computes the ground-truth maps and runs
forward + backward of mean((C_pred - C_gt)^2) (no optimizer step), at P = 1 pair per step (the reference's loop) and
P = 8:
  * ``pair_eager``: the reference's loop, per pair: torch rotations ``verts @ R``, ``model.forward(shape1, shape2)``,
    ``pds.ground_truth([pair])`` and a backward;
  * ``slot_eager``: ``slot.fill(ids)``, ``slot.pack(verts, rotations=random_rotations(2P))``, ``forward_pairs``,
    ``slot.ground_truth()``, the loss and its backward, eagerly;
  * ``slot_graphed``: the same step captured once in ``graphs.GraphedTrainStep`` and replayed with new ids.
Reported: ms per step and pairs/s; ``dn_fmap_ground_truth``'s own time per call (CUDA events around a graph of 20
calls, replayed 10 times); and, as
a check that the routes compute the same thing, their losses on one step with the same pairs and rotations and dropout
off (max relative difference to the slot's).

    python bench_fmaps_shuffled.py [--steps 20] [--warmup 3] [--pairs 1,8]
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

N_SHAPES = 80
K_EIG = 128
N_CORR = 6890


def emit(**kw):
    print(json.dumps(kw), flush=True)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=60).stdout.strip().split(", ")
        pl, clk = q[0], q[1] if len(q) > 1 else "unknown"
    except Exception as e:  # the numbers are reported beside what is known
        pl = clk = "unknown ({})".format(e)
    return name, pl, clk


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


def dataset():
    items, tuples = [], []
    g = torch.Generator().manual_seed(7)
    for s in range(N_SHAPES):
        n, m = 50 + s % 7, 100 + s % 3
        mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K_EIG, seed=s, device="cuda")
        items.append({"mass": mass, "evals": evals, "evecs": evecs, "gradX": gX, "gradY": gY})
        tuples.append([None, None, None, mass, None, evals, evecs, gX, gY, None, None])
    ds = dn.MeshDataset(items)
    verts = torch.randn(ds.V, 3, generator=g).cuda()
    vts = [torch.randint(0, ds.n_rows[s], (N_CORR,), generator=g) for s in range(N_SHAPES)]
    pds = dn.PairDataset(ds, vts, itertools.permutations(range(N_SHAPES), 2))
    return ds, pds, verts, tuples


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pairs", default="1,8")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fmaps_shuffled.py needs a GPU")
    name, pl, clk = card()
    emit(card=name, power_limit=pl, max_sm_clock=clk, engine="tc3x", shapes=N_SHAPES, k_eig=K_EIG, n_fmap=30, correspondences=N_CORR)
    dn.set_engine("tc3x")
    torch.manual_seed(0)
    model = dn.FunctionalMapCorrespondenceWithDiffusionNetFeatures(n_feat=128, input_features="xyz").cuda().train()
    ds, pds, verts, tuples = dataset()
    rng = random.Random(0)

    def shape(s, R):
        t = list(tuples[s])
        t[0] = verts[ds.row_begin[s]:ds.row_begin[s + 1]] @ R
        return t

    def pair_loss(i, R1, R2):
        C_pred, _, _ = model(shape(pds.pair_x_host[i], R1), shape(pds.pair_y_host[i], R2))
        return (C_pred - pds.ground_truth([i]).unsqueeze(0)).square().mean()

    for P in [int(p) for p in args.pairs.split(",")]:
        slot = pds.slot(P)
        ids = torch.zeros(P, dtype=torch.int64, device="cuda")

        def slot_loss(net, ids_, R=None):
            slot.fill(ids_)
            x = slot.pack(verts, rotations=dn.batch.random_rotations(2 * P, device="cuda") if R is None else R)
            C_pred, _ = net.forward_pairs(slot, x)
            return (C_pred - slot.ground_truth()).square().mean()

        # the routes' losses on one step: same pairs, same rotations, dropout off
        draw = [rng.randrange(len(pds)) for _ in range(P)]
        R = dn.batch.random_rotations(2 * P, device="cuda")
        model.eval()
        with torch.no_grad():
            l_slot = slot_loss(model, torch.tensor(draw, device="cuda"), R)
            l_pair = sum(pair_loss(i, R[p], R[P + p]) for p, i in enumerate(draw)) / P
        model.train()
        agree = abs(l_pair.item() - l_slot.item()) / abs(l_slot.item())

        def pair_step():
            for _ in range(P):
                i = rng.randrange(len(pds))
                Rr = dn.batch.random_rotations(2, device="cuda")
                pair_loss(i, Rr[0], Rr[1]).backward()

        def slot_step():
            ids.copy_(torch.randint(len(pds), (P,), device="cuda"))
            slot_loss(model, ids).backward()

        t_pair = time_ms(pair_step, args.steps, args.warmup)
        t_slot = time_ms(slot_step, args.steps, args.warmup)
        gs = dn.graphs.GraphedTrainStep(model, slot_loss, (ids,))

        def graph_step():
            ids.copy_(torch.randint(len(pds), (P,), device="cuda"))
            gs.replay()

        t_graph = time_ms(graph_step, args.steps, args.warmup)
        # the ground truth's two kernels alone: 20 calls captured in one graph, so the host does not set the pace
        gt_graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gt_graph):
            for _ in range(20):
                slot.ground_truth()
        t_gt = time_ms(gt_graph.replay, 10, 2) / 20
        model.zero_grad(set_to_none=True)
        pds.check()
        slot.check()
        for route, t in (("pair_eager", t_pair), ("slot_eager", t_slot), ("slot_graphed", t_graph)):
            emit(pairs=P, route=route, ms_per_step=round(t, 3), pairs_per_s=round(1e3 * P / t, 1))
        emit(pairs=P, ground_truth_ms=round(t_gt, 4), first_step_loss_rel_diff_pair_vs_slot=agree,
             loss_slot=l_slot.item(), loss_pair=l_pair.item())


if __name__ == "__main__":
    main()
