"""Training step of an implicit-diffusion whole-shape classifier (diffusion_method='implicit_dense', the SHREC11 net
shape) over a batch of 32 meshes, on four routes.

Net: C_in 16, C_width 64, 4 blocks, 30 classes, outputs_at 'global_mean', label smoothing 0.2, no dropout, with the
diffusion times of the reference's shipped human-segmentation checkpoint (tests/golden/human_seg_xyz_4x128_f16.npz,
block i's first 64 channels in block i), as a trained net has them.  Data: 32 jittered synthetic tori of 250-750
vertices, normalised to unit max radius, with their cotan Laplacian, mass and gradient operators from
geometry.compute_operators (the batch items carry L and no eigenbasis).  Routes, each one forward + backward of the
summed per-mesh losses:
  loop_fused        per-mesh loop of DiffusionNet.forward_global_nll
  loop_composed     per-mesh loop of net(...) and the reference's label_smoothing_log_loss (written below)
  batch_composed    DiffusionNet.forward_batch and the same composed loss
  batch_fused       DiffusionNet.forward_batch_global_nll
Every implicit solve reads its convergence status on the host once; the step's count of those reads is printed beside
its library launch count, and the iteration counts of the step's solves (the largest per-pair count of each) beside
the times.

CUDA events, every route warmed up, the routes alternated and repeated for the spread (median and [min, max] of the
repetitions).  Prints the card's name, power limit and max SM clock beside the numbers, and one JSON line per route.

  python bench_implicit_batch.py [--reps 5] [--iters 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import diffusion_net_b200 as dn  # noqa: E402

N_MESH, C_WIDTH, N_CLASS, SMOOTHING = 32, 64, 30, 0.2
ROOT = os.path.dirname(os.path.abspath(__file__))


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


def checkpoint_times():
    """Block i's learned diffusion times of the shipped checkpoint, its first C_WIDTH channels."""
    with np.load(os.path.join(ROOT, "tests", "golden", "human_seg_xyz_4x128_f16.npz")) as z:
        return [torch.from_numpy(z["block_{}.diffusion.diffusion_time".format(i)].astype(np.float32)[:C_WIDTH])
                for i in range(4)]


def meshes(seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    while len(out) < N_MESH:
        n, m = (int(v) for v in torch.randint(12, 40, (2,), generator=g))
        if 250 <= n * m <= 750:
            verts, faces = dn.synthetic.torus_mesh(n, m, seed=len(out))
            verts = verts - verts.mean(0)
            verts = verts / verts.norm(dim=1).max()
            _, mass, L, _, _, gX, gY = dn.geometry.compute_operators(verts.cuda(), faces.cuda(), 4)
            out.append(dict(mass=mass, L=L, gradX=gX, gradY=gY))
    return out


class StatusReads:
    """Counts the implicit solves' host reads of their status (one per ops._implicit_call) and keeps each solve's
    largest per-pair iteration count."""

    def __init__(self):
        self.n = 0
        self.iters = []
        self._orig = dn.ops._implicit_call

    def __enter__(self):
        def counting(*a, **k):
            self.n += 1
            st = self._orig(*a, **k)
            self.iters.append(int(st[1]))
            return st
        dn.ops._implicit_call = counting
        return self

    def __exit__(self, *exc):
        dn.ops._implicit_call = self._orig


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_implicit_batch.py needs a GPU"
    dn.set_engine("tc3x")
    print("card:", card())
    items = meshes()
    mb = dn.MeshBatch(items)
    torch.manual_seed(0)
    net = dn.DiffusionNet(C_in=16, C_out=N_CLASS, C_width=C_WIDTH, N_block=4, dropout=False, outputs_at="global_mean",
                          last_activation=lambda t: F.log_softmax(t, dim=-1),
                          diffusion_method="implicit_dense").cuda().train()
    dtimes = checkpoint_times()
    with torch.no_grad():
        for blk, t in zip(net.blocks, dtimes):
            blk.diffusion.diffusion_time.copy_(t)
    print("diffusion times per block [min, max]:", [[float(t.min()), float(t.max())] for t in dtimes])
    xs = [torch.randn(it["mass"].shape[0], 16, device="cuda") for it in items]
    labs = torch.randint(0, N_CLASS, (N_MESH,), device="cuda")
    lab1 = [labs[i:i + 1] for i in range(N_MESH)]
    kw = [dict(L=it["L"], gradX=it["gradX"], gradY=it["gradY"]) for it in items]

    def loop_fused():
        net.zero_grad(set_to_none=False)
        sum(net.forward_global_nll(xs[i], items[i]["mass"], labels=lab1[i], label_smoothing=SMOOTHING, **kw[i])[0]
            for i in range(N_MESH)).backward()

    def loop_composed():
        net.zero_grad(set_to_none=False)
        sum(label_smoothing_log_loss(net(xs[i], items[i]["mass"], **kw[i]), lab1[i], SMOOTHING)
            for i in range(N_MESH)).backward()

    def batch_composed():
        net.zero_grad(set_to_none=False)
        outs = net.forward_batch(mb, xs)
        sum(label_smoothing_log_loss(o, lab1[i], SMOOTHING) for i, o in enumerate(outs)).backward()

    def batch_fused():
        net.zero_grad(set_to_none=False)
        net.forward_batch_global_nll(mb, xs, labs, label_smoothing=SMOOTHING)[0].sum().backward()

    routes = {"loop_fused": loop_fused, "loop_composed": loop_composed, "batch_composed": batch_composed,
              "batch_fused": batch_fused}
    lib = dn._lib.load()
    launches, reads, iters = {}, {}, {}
    for k, fn in routes.items():             # warm-up of every route
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        l0 = lib.dn_kernel_launch_count()
        with StatusReads() as sr:
            fn()
        launches[k] = int(lib.dn_kernel_launch_count() - l0)
        reads[k] = sr.n
        iters[k] = sr.iters
    torch.cuda.synchronize()
    times = {k: [] for k in routes}
    for _ in range(a.reps):
        for k, fn in routes.items():         # alternated
            times[k].append(timed(fn, a.iters))
    V = [int(it["mass"].shape[0]) for it in items]
    for k in routes:
        print(json.dumps({"bench": "implicit_shrec11_train_step", "route": k, "meshes": N_MESH, "V_min": min(V),
                          "V_max": max(V), "V_total": sum(V), "C_width": C_WIDTH, "classes": N_CLASS,
                          "label_smoothing": SMOOTHING, "ms": spread(times[k]), "dn_launches": launches[k],
                          "status_reads": reads[k], "solve_iterations": spread(iters[k]),
                          "solve_iterations_total": sum(iters[k])}))
        if k.startswith("batch"):
            print("  {}: largest per-pair iteration count of each solve, forward then backward:".format(k), iters[k])


if __name__ == "__main__":
    main()
