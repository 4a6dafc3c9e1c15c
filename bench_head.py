"""Training step of the classification head: DiffusionNet.forward_nll (fused last_lin + log_softmax + nll_loss) against
nll_loss(net(...)) on the same net, at the shapes of the three segmentation / correspondence experiments.

Per shape: the head alone (forward + backward of the op on the last block's output) and the whole step (forward +
backward of the net), CUDA events, every shape warmed up, the two routes alternated in one process and repeated for the
spread, peak memory of each route.  Prints the card's name, power limit and max SM clock beside the numbers, and one
JSON line per shape.

  python bench_head.py [--reps 5] [--iters 10]
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

# (name, grid n x m -> V vertices, K, C_width, classes, outputs_at)
SHAPES = [
    ("human_seg_faces", (70, 86), 128, 128, 8, "faces"),          # ~6k vertices, ~12k faces
    ("rna_vertices", (150, 160), 128, 128, 260, "vertices"),      # 24k vertices
    ("faust_correspondence", (65, 106), 128, 256, 6890, "vertices"),  # 6890 vertices
]


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


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_head.py needs a GPU"
    dn.set_engine("tc3x")
    print("card:", card())
    for name, (n, m), K, C, n_class, outputs_at in SHAPES:
        mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=0, device="cuda")
        _, faces = dn.synthetic.torus_mesh(n, m, seed=0)
        faces = faces.cuda()
        V = mass.shape[0]
        torch.manual_seed(0)
        net = dn.DiffusionNet(C_in=16, C_out=n_class, C_width=C, N_block=4, dropout=False, outputs_at=outputs_at,
                              last_activation=lambda t: F.log_softmax(t, dim=-1)).cuda().train()
        x = torch.randn(V, 16, device="cuda")
        rows = faces.shape[0] if outputs_at == "faces" else V
        lab = torch.randint(0, n_class, (rows,), device="cuda")
        kw = dict(evals=evals, evecs=evecs, gradX=gX, gradY=gY, faces=faces)
        feats = torch.randn(rows, C, device="cuda", requires_grad=True)
        W, b = net.last_lin.weight, net.last_lin.bias

        def step_fused():
            net.zero_grad(set_to_none=False)
            net.forward_nll(x, mass, labels=lab, **kw)[0].backward()

        def step_composed():
            net.zero_grad(set_to_none=False)
            F.nll_loss(net(x, mass, **kw), lab).backward()

        def head_fused():
            nll, _ = dn.ops.linear_nll(feats, W, b, lab)
            (nll.sum() / rows).backward()

        def head_composed():
            z = dn.ops.mlp_apply([feats], [W], [b])
            F.nll_loss(F.log_softmax(z, dim=-1), lab).backward()

        routes = {"step_fused": step_fused, "step_composed": step_composed, "head_fused": head_fused,
                  "head_composed": head_composed}
        for fn in routes.values():            # warm-up of every route at this shape
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in routes}
        for _ in range(a.reps):
            for k, fn in routes.items():      # alternated
                times[k].append(timed(fn, a.iters))
        mem = {k: peak(fn) for k, fn in routes.items()}
        res = {"shape": name, "V": V, "rows": rows, "C": C, "classes": n_class,
               "ms_median": {k: sorted(v)[len(v) // 2] for k, v in times.items()},
               "ms_min": {k: min(v) for k, v in times.items()}, "ms_max": {k: max(v) for k, v in times.items()},
               "peak_MiB": mem}
        print(json.dumps(res))
        del net, routes
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
