"""Training step of the SHREC11 whole-shape classifier (outputs_at='global_mean', label smoothing 0.2) over a batch of
32 meshes, on five routes, and the mass-weighted mean pool alone at dataset scale.

Net: C_in 16, C_width 64, 4 blocks, K 128, 30 classes, no dropout.  Data: 32 synthetic tori of 250-750 vertices.
Routes, each one forward + backward of the summed per-mesh losses:
  loop_composed     per-mesh loop of net(...) and the reference's label_smoothing_log_loss (written below)
  loop_fused        per-mesh loop of DiffusionNet.forward_global_nll
  batch_composed    DiffusionNet.forward_batch and the same composed loss
  batch_fused       DiffusionNet.forward_batch_global_nll
  batch_fused_graph batch_fused captured once in graphs.GraphedTrainStep and replayed
Pool: dn_global_mean_fwd / _bwd at V = 200k, C = 128, with the achieved rate over the bytes the algorithm must move.

CUDA events, every route and shape warmed up, the routes alternated and repeated for the spread (median and
[min, max] of the repetitions).  Prints the card's name, power limit and max SM clock beside the numbers, and one JSON
line per result.

  python bench_classify.py [--reps 5] [--iters 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import diffusion_net_b200 as dn  # noqa: E402

N_MESH, K, C_WIDTH, N_CLASS, SMOOTHING = 32, 128, 64, 30, 0.2


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "unknown ({})".format(e)


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def spread(v):
    v = sorted(v)
    return {"median": v[len(v) // 2], "min": v[0], "max": v[-1]}


def label_smoothing_log_loss(pred, labels, smoothing=0.0):
    """The reference's loss of the classification experiment (utils.py), on one mesh's 1-D log-probabilities."""
    n_class = pred.shape[-1]
    one_hot = torch.zeros_like(pred)
    one_hot[labels] = 1.
    one_hot = one_hot * (1 - smoothing) + (1 - one_hot) * smoothing / (n_class - 1)
    return -(one_hot * pred).sum(dim=-1).mean()


def meshes(seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    while len(out) < N_MESH:
        n, m = (int(v) for v in torch.randint(12, 40, (2,), generator=g))
        if 250 <= n * m <= 750:
            mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=len(out), device="cuda")
            out.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY))
    return out


def bench_step(a):
    items = meshes()
    mb = dn.MeshBatch(items)
    torch.manual_seed(0)
    net = dn.DiffusionNet(C_in=16, C_out=N_CLASS, C_width=C_WIDTH, N_block=4, dropout=False, outputs_at="global_mean",
                          last_activation=lambda t: F.log_softmax(t, dim=-1)).cuda().train()
    xs = [torch.randn(it["mass"].shape[0], 16, device="cuda") for it in items]
    labs = torch.randint(0, N_CLASS, (N_MESH,), device="cuda")
    lab1 = [labs[i:i + 1] for i in range(N_MESH)]
    kw = [dict(evals=it["evals"], evecs=it["evecs"], gradX=it["gradX"], gradY=it["gradY"]) for it in items]

    def loop_composed():
        net.zero_grad(set_to_none=False)
        sum(label_smoothing_log_loss(net(xs[i], items[i]["mass"], **kw[i]), lab1[i], SMOOTHING)
            for i in range(N_MESH)).backward()

    def loop_fused():
        net.zero_grad(set_to_none=False)
        sum(net.forward_global_nll(xs[i], items[i]["mass"], labels=lab1[i], label_smoothing=SMOOTHING, **kw[i])[0]
            for i in range(N_MESH)).backward()

    def batch_composed():
        net.zero_grad(set_to_none=False)
        outs = net.forward_batch(mb, xs)
        sum(label_smoothing_log_loss(o, lab1[i], SMOOTHING) for i, o in enumerate(outs)).backward()

    def batch_loss(net_, xs_, labs_):
        return net_.forward_batch_global_nll(mb, xs_, labs_, label_smoothing=SMOOTHING)[0].sum()

    def batch_fused():
        net.zero_grad(set_to_none=False)
        batch_loss(net, xs, labs).backward()

    graphed = dn.graphs.GraphedTrainStep(net, batch_loss, (xs, labs))

    def batch_fused_graph():
        dn.graphs.GraphedTrainStep.zero_grads(net)
        graphed.replay()

    routes = {"loop_composed": loop_composed, "loop_fused": loop_fused, "batch_composed": batch_composed,
              "batch_fused": batch_fused, "batch_fused_graph": batch_fused_graph}
    lib = dn._lib.load()
    launches = {}
    for k, fn in routes.items():             # warm-up of every route
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        l0 = lib.dn_kernel_launch_count()
        fn()
        launches[k] = int(lib.dn_kernel_launch_count() - l0)   # a graph replay launches nothing through the library
    torch.cuda.synchronize()
    times = {k: [] for k in routes}
    for _ in range(a.reps):
        for k, fn in routes.items():         # alternated
            times[k].append(timed(fn, a.iters))
    V = [int(it["mass"].shape[0]) for it in items]
    for k in routes:
        print(json.dumps({"bench": "shrec11_train_step", "route": k, "meshes": N_MESH, "V_min": min(V),
                          "V_max": max(V), "V_total": sum(V), "C_width": C_WIDTH, "K": K, "classes": N_CLASS,
                          "label_smoothing": SMOOTHING, "ms": spread(times[k]), "dn_launches": launches[k]}))


def bench_pool(a, V=200000, C=128):
    lib = dn._lib.load()
    x = torch.randn(V, C, device="cuda")
    mass = torch.rand(V, device="cuda") + 0.25
    seg = dn.ops.single_segment(V, x.device)
    pooled = torch.empty(1, C, device="cuda")
    msum = torch.empty(1, device="cuda")
    g = torch.randn(1, C, device="cuda")
    gx = torch.empty(V, C, device="cuda")
    need = lib.dn_global_mean_workspace_bytes(V, C)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    tabs = (seg.begin.data_ptr(), seg.rows.data_ptr(), seg.tile_seg.data_ptr(), seg.n_seg)

    def fwd():
        dn._lib.check(lib.dn_global_mean_fwd(x.data_ptr(), mass.data_ptr(), V, C, *tabs, pooled.data_ptr(),
                                             msum.data_ptr(), ws.data_ptr(), need, st), "dn_global_mean_fwd")

    def bwd():
        dn._lib.check(lib.dn_global_mean_bwd(g.data_ptr(), mass.data_ptr(), msum.data_ptr(), V, C, *tabs,
                                             gx.data_ptr(), st), "dn_global_mean_bwd")

    # algorithmic bytes: forward reads x and mass; backward reads mass and writes grad_x (the (1, C) rows are noise)
    nbytes = {"fwd": 4 * V * C + 4 * V, "bwd": 4 * V + 4 * V * C}
    routes = {"fwd": fwd, "bwd": bwd}
    for fn in routes.values():
        for _ in range(5):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in routes}
    for _ in range(a.reps):
        for k, fn in routes.items():
            times[k].append(timed(fn, 20 * a.iters))
    for k in routes:
        t = spread(times[k])
        print(json.dumps({"bench": "global_mean_pool", "pass": k, "V": V, "C": C, "MB": nbytes[k] / 1e6,
                          "us": {q: 1e3 * v for q, v in t.items()},
                          "GBps": {q: nbytes[k] / (1e-3 * t[w]) / 1e9 for q, w in
                                   (("median", "median"), ("min", "max"), ("max", "min"))}}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_classify.py needs a GPU"
    dn.set_engine("tc3x")
    print("card:", card())
    bench_step(a)
    bench_pool(a)


if __name__ == "__main__":
    main()
