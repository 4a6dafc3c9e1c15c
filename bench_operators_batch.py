"""Time ``geometry.compute_operators_batch`` against ``geometry.compute_operators`` in a loop on datasets of small
meshes, k = 128: 64 x torus(36 + i % 9, 50) (V ~ 2k, the meshes of BASELINE config 4), 64 x V ~ 500 (SHREC11-like) and
16 x torus(70, 100) (V = 7k).  One JSON line per dataset.

    python bench_operators_batch.py [--datasets torus2k,v500,torus7k] [--k 128] [--rounds 3] [--no-reference]

Both routes run in the same process, alternated, after one warm-up call each; a time is a host clock around a call
that ends in a device synchronise, reported as the median over the rounds with the min and max beside it.  Stage times
come from CUDA events in one further call per route (``stats=``; the per-mesh route synchronises once per mesh for
it, so that call is not the one timed).  The card, its power limit and its clocks are reported as found.  The
reference's CPU ``compute_operators`` is timed on the first mesh of each dataset, only through ``oracle/ref_import``
and only when it is there.  Writes nothing to the tree."""
import argparse
import json
import statistics
import subprocess
import time

import torch

from bench_operators import card, time_reference

import diffusion_net_b200 as dn

T = dn.synthetic.torus_mesh
DATASETS = {
    "torus2k": lambda: [T(36 + i % 9, 50, seed=i) for i in range(64)],
    "v500": lambda: [T(18 + i % 7, 26, seed=i) for i in range(64)],
    "torus7k": lambda: [T(70, 100, seed=i) for i in range(16)],
}


def clocks():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return [float(x) for x in r.stdout.strip().splitlines()[0].split(",")]
    except Exception:
        return [None, None]


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def spread(ts):
    return dict(median=round(statistics.median(ts), 4), min=round(min(ts), 4), max=round(max(ts), 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--datasets", default="torus2k,v500,torus7k")
    ap.add_argument("--k", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_operators_batch.py needs a GPU")
    name, power = card()
    sm_mhz, sm_max_mhz = clocks()
    dev = torch.device("cuda", 0)
    geo = dn.geometry
    for ds in a.datasets.split(","):
        meshes = DATASETS[ds]()
        vl, fl = [v for v, _ in meshes], [f for _, f in meshes]
        loop = lambda st=None: [geo.compute_operators(v, f, a.k, device=dev, stats=None if st is None else st.setdefault(i, {}))
                                for i, (v, f) in enumerate(meshes)]
        batch = lambda st=None: geo.compute_operators_batch(vl, fl, a.k, device=dev, stats=st)
        loop(), batch()                                                 # warm-up
        t_loop, t_batch = [], []
        for _ in range(a.rounds):
            t_loop.append(timed(loop))
            t_batch.append(timed(batch))
        ls, bs = {}, {}
        loop(ls)
        batch(bs)
        tot = lambda key: round(sum(s[key] for s in ls.values()), 2)
        eig = bs["eig"]
        esum = lambda key: round(sum(e.get(key, 0.0) for e in eig), 2)
        Vs = [int(v.shape[0]) for v in vl]
        res = dict(dataset=ds, n_meshes=len(meshes), V_min=min(Vs), V_max=max(Vs), V_total=sum(Vs), k=a.k, gpu=name,
                   power_limit_w=power, sm_mhz=sm_mhz, sm_max_mhz=sm_max_mhz, rounds=a.rounds,
                   loop_s=spread(t_loop), batch_s=spread(t_batch),
                   loop_ms_per_mesh=round(1e3 * statistics.median(t_loop) / len(meshes), 2),
                   batch_ms_per_mesh=round(1e3 * statistics.median(t_batch) / len(meshes), 2),
                   speedup=round(statistics.median(t_loop) / statistics.median(t_batch), 2),
                   loop=dict(frames_ms=tot("frames_ms"), laplacian_ms=tot("laplacian_ms"), eig_ms=tot("eig_ms"),
                             eig_filter_ms=tot("filter_ms"), eig_rayleigh_ritz_ms=tot("rr_ms"),
                             build_grad_ms=tot("build_grad_ms"),
                             outer_iterations=sum(s["iterations"] for s in ls.values()),
                             filter_steps=sum(s["filter_steps"] for s in ls.values())),
                   batch=dict(groups=bs["groups"], frames_ms=round(bs["frames_ms"], 2),
                              laplacian_ms=round(bs["laplacian_ms"], 2), eig_ms=round(bs["eig_ms"], 2),
                              eig_filter_ms=esum("filter_ms"), eig_rayleigh_ritz_ms=esum("rr_ms"),
                              eig_gram_rotate_ms=round(esum("rr_ms") - esum("dense_ms"), 2), eig_dense_linalg_ms=esum("dense_ms"),
                              build_grad_ms=round(bs["build_grad_ms"], 2), split_ms=round(bs["split_ms"], 2),
                              outer_iterations=sum(e["iterations"] for e in eig),
                              filter_steps=sum(e["filter_steps"] for e in eig)))
        res["batch"]["dense_linalg_share_of_eig"] = round(res["batch"]["eig_dense_linalg_ms"] / max(bs["eig_ms"], 1e-9), 3)
        if not a.no_reference:
            ref_s = time_reference(vl[0], fl[0], a.k)
            res["reference_s_first_mesh"] = None if ref_s is None else round(ref_s, 2)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
