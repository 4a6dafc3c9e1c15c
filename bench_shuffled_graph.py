"""Shuffled training steps replayed as one CUDA graph (batch.BatchSlot): what a fixed-capacity slot costs and saves.

Workloads (K = 128, synthetic tori with the operator statistics of get_operators, bench_dataset_batch.py's datasets):
  shrec11  whole-shape classification (outputs_at='global_mean', C_width 64, 4 blocks, 30 classes, label smoothing
           0.2, bench_classify.py's step): 32 meshes of 250-750 vertices per step, drawn from 600
  seg1     per-vertex segmentation (C_width 128, 4 blocks, 8 classes, forward_batch_nll with labels in the batch
           layout): 1 mesh of 5k-10k vertices per step (the reference's batch_size=None loop), drawn from 64
  seg8     the same with 8 meshes per step
  faces1   seg1 with outputs_at='faces' (per-face labels, the human segmentation experiment's head): the slot routes
           take the labels in the slot's element layout (slot.pack_elements), eager_ds_batch as per-mesh lists
  faces8   the same with 8 meshes per step
Routes, alternated, each a full step (zero grads, forward, backward) on a fresh random draw of ids every step:
  eager_ds_batch  ds.batch(ids) + ds.pack + the step, issued eagerly
  eager_slot      slot.fill(device ids) + slot.pack + the step, issued eagerly
  graph_slot      the eager_slot step captured once with graphs.GraphedTrainStep, replayed after ids.copy_()
  graph_fixed     the reference point: GraphedTrainStep over one fixed ds.batch (the same meshes every step)
Printed per workload: V_cap / V (the padding a fixed shape costs, averaged over the draws), library launches per step
of each eager route, and the kernel time of one fill (plan_kernel + batch_gather_kernel, torch.profiler, in a pass of
its own).  Each time is the median and [min, max] over the repetitions; the card's name, power limit and max SM clock
are printed first.

  python bench_shuffled_graph.py [--reps 5] [--iters 20] [--workloads shrec11,seg1,seg8,faces1,faces8]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import diffusion_net_b200 as dn  # noqa: E402
from bench_classify import card, spread, timed  # noqa: E402
from bench_dataset_batch import WORKLOADS as DATASETS, dataset_items  # noqa: E402

WORKLOADS = {"shrec11": dict(data="shrec11", batch=32, C_width=64, classes=30, head="global"),
             "seg1": dict(data="large", batch=1, C_width=128, classes=8, head="vertices"),
             "seg8": dict(data="large", batch=8, C_width=128, classes=8, head="vertices"),
             "faces1": dict(data="large_faces", batch=1, C_width=128, classes=8, head="faces"),
             "faces8": dict(data="large_faces", batch=8, C_width=128, classes=8, head="faces")}
SMOOTHING = 0.2


def _launches():
    return dn._lib.load().dn_kernel_launch_count()


def fill_kernel_us(fn, n):
    """Mean device time per fill of the planner and the gather kernel, from torch.profiler."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for name in ("plan_kernel", "batch_gather_kernel"):
            if name in e.key:
                tot = getattr(e, "device_time_total", None) or e.cuda_time_total
                out[name] = out.get(name, 0.0) + tot / n
    assert set(out) == {"plan_kernel", "batch_gather_kernel"}, out
    return out


def bench(a, name, w, ds):
    torch.manual_seed(0)
    nb, global_head, faces = w["batch"], w["head"] == "global", w["head"] == "faces"
    net = dn.DiffusionNet(C_in=16, C_out=w["classes"], C_width=w["C_width"], N_block=4, dropout=False,
                          outputs_at="global_mean" if global_head else w["head"],
                          last_activation=lambda t: F.log_softmax(t, dim=-1)).cuda().train()
    X = torch.randn(ds.V, 16, device="cuda")
    Yv = torch.randint(0, w["classes"], (ds.V,), device="cuda")
    Yg = torch.randint(0, w["classes"], (ds.n_meshes,), device="cuda")
    if faces:
        n_faces = ds._elems["faces"][1]
        Yf = torch.randint(0, w["classes"], (sum(n_faces),), device="cuda")
        f0 = [0]
        for c in n_faces:
            f0.append(f0[-1] + c)
        Yf_mesh = [Yf[f0[i]:f0[i + 1]] for i in range(ds.n_meshes)]
    g = torch.Generator().manual_seed(1)
    draws = [torch.randperm(ds.n_meshes, generator=g)[:nb] for _ in range(max(a.iters, 8))]
    draws_host = [d.tolist() for d in draws]
    draws_dev = [d.cuda() for d in draws]
    state = {"k": 0}

    def next_k():
        state["k"] = (state["k"] + 1) % len(draws)
        return state["k"]

    def loss(net_, b, x, k_ids=None, lab_v=None):
        if global_head:
            lab = Yg[draws_dev[k_ids]] if k_ids is not None else slot.take(Yg)
            return net_.forward_batch_global_nll(b, x, lab, label_smoothing=SMOOTHING)[0].sum()
        return net_.forward_batch_nll(b, x, lab_v)[0].sum()

    def batch_labels(b, k):
        if global_head:
            return None
        return [Yf_mesh[i] for i in draws_host[k]] if faces else ds.pack(Yv, b)

    def eager_ds_batch():
        k = next_k()
        b = ds.batch(draws_host[k])
        net.zero_grad(set_to_none=False)
        loss(net, b, ds.pack(X, b), k, batch_labels(b, k)).backward()

    slot = ds.slot(nb, elements="faces") if faces else ds.slot(nb)
    ids = torch.zeros(nb, dtype=torch.int64, device="cuda")

    def slot_loss(net_, ids_):
        slot.fill(ids_)
        lab = None if global_head else slot.pack_elements(Yf, "faces") if faces else slot.pack(Yv)
        return loss(net_, slot, slot.pack(X), None, lab)

    def eager_slot():
        ids.copy_(draws_dev[next_k()])
        net.zero_grad(set_to_none=False)
        slot_loss(net, ids).backward()

    graph = dn.graphs.GraphedTrainStep(net, slot_loss, (ids,))

    def graph_slot():
        ids.copy_(draws_dev[next_k()])
        graph.zero_grads(net)
        graph.replay()

    fb = ds.batch(draws_host[0])
    fx, fy = ds.pack(X, fb), batch_labels(fb, 0)
    fixed = dn.graphs.GraphedTrainStep(net, lambda n_: loss(n_, fb, fx, 0, fy), ())

    def graph_fixed():
        fixed.zero_grads(net)
        fixed.replay()

    routes = {"eager_ds_batch": eager_ds_batch, "eager_slot": eager_slot, "graph_slot": graph_slot,
              "graph_fixed": graph_fixed}
    for fn in routes.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    launches = {}
    for k in ("eager_ds_batch", "eager_slot"):
        l0 = _launches()
        routes[k]()
        launches[k] = _launches() - l0
    times = {k: [] for k in routes}
    for _ in range(a.reps):
        for k, fn in routes.items():
            times[k].append(timed(fn, a.iters))
    V_actual = [ds.batch(d).V for d in draws_host]
    fill_us = fill_kernel_us(lambda: slot.fill(draws_dev[next_k()]), 4 * a.iters)
    slot.check()
    base = {"workload": name, "dataset_meshes": ds.n_meshes, "batch_meshes": nb, "C_width": w["C_width"], "K": 128,
            "classes": w["classes"]}
    shape = dict(base, bench="slot_shape", V_cap=slot.V, V_mean=sum(V_actual) / len(V_actual),
                 V_cap_over_V=slot.V * len(V_actual) / sum(V_actual), library_launches_per_step=launches,
                 fill_kernel_us=fill_us)
    if faces:
        F_actual = [sum((n_faces[i] + 127) // 128 * 128 for i in d) for d in draws_host]
        shape.update(F_cap=slot.element_capacity["faces"],
                     F_cap_over_F=slot.element_capacity["faces"] * len(F_actual) / sum(F_actual))
    print(json.dumps(shape))
    for k in routes:
        print(json.dumps(dict(base, bench="shuffled_train_step", route=k, ms=spread(times[k]))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_shuffled_graph.py needs a GPU"
    dn.set_engine("tc3x")
    print("card:", card())
    datasets = {}
    for name in a.workloads.split(","):
        w = WORKLOADS[name]
        if w["data"] not in datasets:
            data = w["data"].replace("_faces", "")
            datasets[w["data"]] = dn.MeshDataset(dataset_items(DATASETS[data], faces=data != w["data"]))
        bench(a, name, w, datasets[w["data"]])


if __name__ == "__main__":
    main()
