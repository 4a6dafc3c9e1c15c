"""Time ``geometry.compute_operators`` (frames, Laplacian, mass, k lowest eigenpairs, build_grad on the GPU) on the
jittered torus at V = 20k and V = 200k, k = 128, and the reference's ``compute_operators`` (CPU: potpourri3d
restatement + ARPACK ``eigsh`` + Python build_grad) beside it.  One JSON line per size.

    python bench_operators.py [--sizes 100x200,400x500] [--k 128] [--reference-200k] [--no-reference]

The reference is timed through ``oracle/ref_import`` (the mounted reference, else the copy ``build()`` staged under
oracle/_ref) -- by default only up to V = 20k, where its eigsh takes seconds; ``--reference-200k`` includes 200k (about a
minute and a half of eigsh alone).  Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import diffusion_net_b200 as dn  # noqa: E402


def filter_bytes(V, nnz, stats):
    """Byte model of the filter kernel: every step reads its V x n input block and the previous one and writes one
    (fp64; the first step of each filter reads no previous block, ignored here), plus the operator once (int32
    column + fp64 value per entry, int32 row pointer + fp64 diagonal per row)."""
    return 3 * 8 * V * stats["filter_col_steps"] + stats["filter_steps"] * (12 * nnz + 12 * V)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = float(r.stdout.strip().splitlines()[0])
    except Exception:
        power = None
    return name, power


def time_reference(verts, faces, k):
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    from ref_import import import_reference, reference_available
    if not reference_available():
        return None
    ref = import_reference()
    t = time.perf_counter()
    ref.geometry.compute_operators(verts, faces, k)
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100x200,400x500")
    ap.add_argument("--k", type=int, default=128)
    ap.add_argument("--reference-200k", action="store_true")
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    name, power = card()
    dev = torch.device("cuda", 0)
    for size in a.sizes.split(","):
        n, m = (int(x) for x in size.split("x"))
        verts, faces = dn.synthetic.torus_mesh(n, m, seed=0)
        V = n * m
        dn.geometry.compute_operators(verts, faces, a.k, device=dev)           # warm-up
        torch.cuda.synchronize()
        st = {}
        t = time.perf_counter()
        out = dn.geometry.compute_operators(verts, faces, a.k, device=dev, stats=st)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t
        fb = filter_bytes(V, st["nnz"], st)
        res = dict(mesh="torus({},{})".format(n, m), V=V, k=a.k, gpu=name, power_limit_w=power,
                   wall_s=round(wall, 4), frames_ms=round(st["frames_ms"], 3), laplacian_ms=round(st["laplacian_ms"], 3),
                   eig_filter_ms=round(st["filter_ms"], 2), eig_rayleigh_ritz_ms=round(st["rr_ms"], 2),
                   eig_ms=round(st["eig_ms"], 2), build_grad_ms=round(st["build_grad_ms"], 3),
                   filter_steps=st["filter_steps"], outer_iterations=st["iterations"], block=st["block"],
                   spectral_bound=st["bound"], filter_gb=round(fb / 1e9, 2),
                   filter_gb_per_s=round(fb / (st["filter_ms"] * 1e-3) / 1e9, 1) if st["filter_ms"] > 0 else None,
                   lambda_k=float(out[3][-1]))
        if not a.no_reference and (V <= 20000 or a.reference_200k):
            ref_s = time_reference(verts, faces, a.k)
            res["reference_s"] = None if ref_s is None else round(ref_s, 2)
            if ref_s is not None:
                res["speedup"] = round(ref_s / wall, 1)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
