"""Shuffled mesh batches from a device-resident dataset (batch.MeshDataset): what assembling a batch costs, per call
and inside a training step.

Workloads (K = 128, synthetic tori with the operator statistics of get_operators):
  shrec11  32 meshes of 250-750 vertices drawn from a 600-mesh dataset (the SHREC11 classification experiment's size)
  large    8 meshes of 5k-10k vertices drawn from a 64-mesh dataset
Measurements:
  1. ds.batch(ids) for random ids: host wall time of the call followed by a synchronise, and the gather kernel's own
     time (torch.profiler, in a pass of its own) with the achieved rate over the bytes it must move.
  2. MeshBatch(subset) of the same random subsets: this tree's (the dataset gathered in order) and, with
     --parent-batch PATH (the previous host-concatenation batch.py, run against this package), the host pipeline it
     replaced, alternated in the same process.  Without it the parent is reported as not measured.
  3. bench_classify.py's batch_fused step (C_width 64, 4 blocks, 30 classes, label smoothing 0.2) on shrec11: a fresh
     shuffled batch every step (ds.batch + ds.pack inside the step) against the same step reused on one fixed batch.

Every shape is warmed up, the variants alternate, and each number is the median and [min, max] of the repetitions.
Prints the card's name, power limit and max SM clock, and one JSON line per result.

  python bench_dataset_batch.py [--reps 5] [--iters 20] [--parent-batch PATH]
"""
import argparse
import importlib.util
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import diffusion_net_b200 as dn  # noqa: E402
from bench_classify import card, spread, timed  # noqa: E402

K, C_WIDTH, N_CLASS, SMOOTHING = 128, 64, 30, 0.2
WORKLOADS = {"shrec11": dict(n_data=600, batch=32, v_lo=250, v_hi=750, nm=(12, 40)),
             "large": dict(n_data=64, batch=8, v_lo=5000, v_hi=10000, nm=(60, 130))}


def dataset_items(w, seed=0, faces=False):
    """The workload's synthetic tori; ``faces``: each item also carries its grid's faces (synthetic.torus_mesh)."""
    g = torch.Generator().manual_seed(seed)
    out = []
    while len(out) < w["n_data"]:
        n, m = (int(v) for v in torch.randint(w["nm"][0], w["nm"][1], (2,), generator=g))
        if w["v_lo"] <= n * m <= w["v_hi"]:
            mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=len(out), device="cuda")
            for _ in range(2):         # resident operators: the CSR and the locality decision are made before timing
                dn.prepare_operators(gX, gY)
            out.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY))
            if faces:
                out[-1]["faces"] = dn.synthetic.torus_mesh(n, m)[1].cuda()
    return out


def gather_bytes(b, ds, ids):
    """Bytes dn_batch_gather must move for batch b: every dataset row, eigenvalue and CSR entry of its meshes read
    once, every batch array (padding included) written once."""
    nnz = b.gops.nnz
    rows = sum(ds.n_rows[i] for i in ids)
    read = 4 * rows * (1 + b.K) + 4 * len(ids) * b.K + 4 * (rows + len(ids)) + 12 * nnz
    write = 4 * b.V * (1 + b.K) + 4 * len(ids) * b.K + 4 * (b.V + 1) + 12 * nnz
    return read + write


def kernel_us(fn, n):
    """Mean device time of the batch_gather kernel over n calls of fn, from torch.profiler."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if "batch_gather_kernel" in e.key]
    assert ev, "no batch_gather_kernel in the trace"
    tot = getattr(ev[0], "device_time_total", None) or ev[0].cuda_time_total
    return tot / ev[0].count


def host_ms(fn, iters):
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
        torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / iters


def bench_batch(a, name, w, items, ds, parent):
    g = torch.Generator().manual_seed(1)
    draws = [torch.randperm(w["n_data"], generator=g)[:w["batch"]].tolist() for _ in range(a.iters)]
    state = {"k": 0}

    def next_ids():
        state["k"] = (state["k"] + 1) % len(draws)
        return draws[state["k"]]

    routes = {"ds.batch": lambda: ds.batch(next_ids()),
              "MeshBatch": lambda: dn.MeshBatch([items[i] for i in next_ids()])}
    if parent is not None:
        routes["MeshBatch_parent"] = lambda: parent.MeshBatch([items[i] for i in next_ids()])
    for fn in routes.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in routes}
    for _ in range(a.reps):
        for k, fn in routes.items():
            times[k].append(host_ms(fn, a.iters))
    # the kernel on every draw in turn (a dataset larger than L2 is read from HBM), bytes averaged over the draws
    nbytes = sum(gather_bytes(ds.batch(d), ds, d) for d in draws) / len(draws)
    us = kernel_us(lambda: ds.batch(next_ids()), 4 * a.iters)
    ids = draws[0]
    b = ds.batch(ids)
    V = [ds.n_rows[i] for i in ids]
    base = {"workload": name, "dataset_meshes": w["n_data"], "batch_meshes": w["batch"], "V_batch": sum(V),
            "V_layout": b.V, "K": K}
    print(json.dumps(dict(base, bench="dataset_batch_gather_kernel", us=us, MB=nbytes / 1e6,
                          GBps=nbytes / (1e-6 * us) / 1e9)))
    for k in routes:
        print(json.dumps(dict(base, bench="batch_build_host_wall", route=k, ms=spread(times[k]))))
    if parent is None:
        print(json.dumps(dict(base, bench="batch_build_host_wall", route="MeshBatch_parent", ms="not measured")))


def bench_step(a, items, ds):
    torch.manual_seed(0)
    net = dn.DiffusionNet(C_in=16, C_out=N_CLASS, C_width=C_WIDTH, N_block=4, dropout=False, outputs_at="global_mean",
                          last_activation=lambda t: F.log_softmax(t, dim=-1)).cuda().train()
    X = torch.randn(ds.V, 16, device="cuda")
    labels = torch.randint(0, N_CLASS, (ds.n_meshes,))
    bs = WORKLOADS["shrec11"]["batch"]
    g = torch.Generator().manual_seed(2)
    perm = {"ids": [], "k": 0}

    def next_ids():
        if perm["k"] + bs > len(perm["ids"]):
            perm["ids"], perm["k"] = torch.randperm(ds.n_meshes, generator=g).tolist(), 0
        perm["k"] += bs
        return perm["ids"][perm["k"] - bs:perm["k"]]

    def step(b, x, lab):
        net.zero_grad(set_to_none=False)
        net.forward_batch_global_nll(b, x, lab, label_smoothing=SMOOTHING)[0].sum().backward()

    fixed_ids = next_ids()
    fb = ds.batch(fixed_ids)
    fx = ds.pack(X, fb)
    flab = labels[fixed_ids].cuda()

    def fresh():
        ids = next_ids()
        b = ds.batch(ids)
        step(b, ds.pack(X, b), labels[ids].pin_memory().to("cuda", non_blocking=True))

    routes = {"batch_fused_fixed_batch": lambda: step(fb, fx, flab), "batch_fused_shuffled_batch": fresh}
    for fn in routes.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in routes}
    for _ in range(a.reps):
        for k, fn in routes.items():
            times[k].append(timed(fn, a.iters))
    for k in routes:
        print(json.dumps({"bench": "shrec11_train_step", "route": k, "dataset_meshes": ds.n_meshes, "batch_meshes": bs,
                          "C_width": C_WIDTH, "K": K, "classes": N_CLASS, "ms": spread(times[k])}))


def load_parent(path):
    """The previous batch.py as a module of this package (its ops / _lib), so both builders run side by side."""
    spec = importlib.util.spec_from_file_location("diffusion_net_b200._parent_batch", path)
    mod = importlib.util.module_from_spec(spec)
    mod.__package__ = "diffusion_net_b200"
    spec.loader.exec_module(mod)
    return mod


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--parent-batch", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dataset_batch.py needs a GPU"
    dn.set_engine("tc3x")
    print("card:", card())
    parent = load_parent(a.parent_batch) if a.parent_batch else None
    for name, w in WORKLOADS.items():
        items = dataset_items(w)
        ds = dn.MeshDataset(items)
        bench_batch(a, name, w, items, ds, parent)
        if name == "shrec11":
            bench_step(a, items, ds)


if __name__ == "__main__":
    main()
