"""Training-step time over a batch of meshes: the per-mesh routes against the batched one (DiffusionNet.forward_batch,
one launch sequence for all meshes).

Workloads (4-block net, C_width = K = 128, C_in = 16, C_out = 8, dropout off, NLL loss summed over the meshes):
  small  32 meshes of 36..44 x 50 torus vertices (the launch-bound case: SHREC11 / human-seg / RNA sized meshes)
  large   8 meshes of 100 x 200 torus vertices
Routes, one optimiser-free step each (zero the gradients, forward, backward):
  a  per-mesh graphs.GraphedTrainStep loop     b  per-mesh eager autograd
  c  batched eager autograd                    d  batched graphs.GraphedTrainStep
Prints one JSON line per workload: median ms per step (CUDA events) and Mverts/s for each route, library kernel
launches per step, the max relative gradient difference of c and d against b, and the GPU name and power limit.
Inputs are seeded synthetic operators (synthetic.structural_operators); nothing is written."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import diffusion_net_b200 as dn  # noqa: E402

WORKLOADS = {"small": [(36 + i % 9, 50) for i in range(32)], "large": [(100, 200)] * 8}
C_IN, C_OUT, WIDTH, K, N_BLOCK = 16, 8, 128, 128, 4


def gpu_info():
    """Name, power limit and max SM clock of the card, read (never set) with nvidia-smi."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        idx = torch.cuda.current_device()
        name, power, clock = (s.strip() for s in r.stdout.strip().splitlines()[idx].split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the timing is still valid; say what could not be read
        return {"gpu": torch.cuda.get_device_name(), "power_limit": "unknown ({})".format(type(e).__name__)}


def nll(out, y):
    return torch.nn.functional.nll_loss(torch.log_softmax(out, dim=-1), y)


def median_ms(step, warmup, steps):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def grads(net):
    return [p.grad.detach().clone() for p in net.parameters()]


def max_rel_diff(net, gs, ref):
    """max over parameters of max|g - r| / max|r|, and the parameter it is reached on"""
    diffs = [(float((g - r).abs().max() / r.abs().max().clamp_min(1e-30)), n_)
             for (n_, _), g, r in zip(net.named_parameters(), gs, ref)]
    d, n_ = max(diffs)
    return {"value": d, "parameter": n_}


def run(name, shapes, warmup, steps):
    lib = dn._lib.load()
    torch.manual_seed(0)
    net = dn.DiffusionNet(C_in=C_IN, C_out=C_OUT, C_width=WIDTH, N_block=N_BLOCK, dropout=False).cuda().train()
    with torch.no_grad():
        for n_, p_ in net.named_parameters():
            if n_.endswith("diffusion_time"):
                p_.uniform_(1e-3, 0.3)
    meshes = []
    for i, (n, m) in enumerate(shapes):
        mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=i, device="cuda")
        g = torch.Generator().manual_seed(1000 + i)
        x = torch.randn(n * m, C_IN, generator=g).cuda()
        y = torch.randint(0, C_OUT, (n * m,), generator=g).cuda()
        meshes.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY, x=x, y=y))
    n_verts = sum(n * m for n, m in shapes)
    mb = dn.MeshBatch(meshes)
    xs, ys = [it["x"] for it in meshes], [it["y"] for it in meshes]

    def mesh_loss(net_, x, y, it):
        return nll(net_(x, it["mass"], evals=it["evals"], evecs=it["evecs"], gradX=it["gradX"], gradY=it["gradY"]), y)

    def batch_loss(net_, xs_, ys_):
        return sum(nll(o, y) for o, y in zip(net_.forward_batch(mb, xs_), ys_))

    def step_b():
        dn.graphs.GraphedTrainStep.zero_grads(net)
        for it in meshes:
            mesh_loss(net, it["x"], it["y"], it).backward()

    def step_c():
        dn.graphs.GraphedTrainStep.zero_grads(net)
        batch_loss(net, xs, ys).backward()

    def launches(step):
        step()
        torch.cuda.synchronize()
        l0 = lib.dn_kernel_launch_count()
        step()
        torch.cuda.synchronize()
        return lib.dn_kernel_launch_count() - l0

    res = {}
    step_b()
    torch.cuda.synchronize()
    ref = grads(net)
    launches_b, launches_c = launches(step_b), launches(step_c)
    res["b"] = median_ms(step_b, warmup, steps)
    step_c()
    torch.cuda.synchronize()
    diff_c = max_rel_diff(net, grads(net), ref)
    res["c"] = median_ms(step_c, warmup, steps)

    per_mesh = [dn.graphs.GraphedTrainStep(net, lambda n_, x, y, it=it: mesh_loss(n_, x, y, it), (it["x"], it["y"]))
                for it in meshes]

    def step_a():
        dn.graphs.GraphedTrainStep.zero_grads(net)
        for gts in per_mesh:
            gts.replay()

    res["a"] = median_ms(step_a, warmup, steps)
    batched = dn.graphs.GraphedTrainStep(net, batch_loss, (xs, ys))

    def step_d():
        dn.graphs.GraphedTrainStep.zero_grads(net)
        batched.replay()

    step_d()
    torch.cuda.synchronize()
    diff_d = max_rel_diff(net, grads(net), ref)
    res["d"] = median_ms(step_d, warmup, steps)

    labels = {"a": "per_mesh_graphs", "b": "per_mesh_eager", "c": "batched_eager", "d": "batched_graph"}
    out = {"workload": name, "n_meshes": len(shapes), "n_verts": n_verts, "padded_rows": mb.V,
           "net": "4 blocks C_width={} K={} C_in={} C_out={}".format(WIDTH, K, C_IN, C_OUT), "engine": dn.get_engine(),
           "ms_per_step": {labels[k]: round(v, 4) for k, v in sorted(res.items())},
           "mverts_per_s": {labels[k]: round(n_verts / (v * 1e-3) / 1e6, 3) for k, v in sorted(res.items())},
           "speedup_batched_graph_vs_per_mesh_graphs": round(res["a"] / res["d"], 3),
           "library_launches_per_step": {"per_mesh": launches_b, "batched": launches_c},
           "graph_launches_per_step": {labels["a"]: len(shapes), labels["d"]: 1},
           "max_rel_grad_diff_vs_per_mesh_eager": {labels["c"]: diff_c, labels["d"]: diff_d},
           "steps": steps, "warmup": warmup}
    out.update(gpu_info())
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--workloads", default="small,large")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--engine", default=os.environ.get("DN_B200_ENGINE", "tc3x"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_batch_train.py needs a CUDA GPU")
    if args.steps < 20 or args.warmup < 3:
        sys.exit("use --steps >= 20 and --warmup >= 3")
    dn.set_engine(args.engine)
    for name in args.workloads.split(","):
        print(json.dumps(run(name, WORKLOADS[name], args.warmup, args.steps)), flush=True)


if __name__ == "__main__":
    main()
