"""Time the implicit heat diffusion (diffusion_method='implicit_dense': fp64 block Jacobi-PCG on L's CSR, one cooperative
launch per solve) on the jittered torus at V = 20k and V = 200k, C = 128, with the diffusion times of the reference's
shipped human-segmentation checkpoint (tests/golden/human_seg_xyz_4x128_f16.npz), beside the spectral path at the same
size (k = 128) and the reference's own dense ``implicit_dense`` at the largest size where its (B, C, V, V) matrix fits
(V = 2k).  One JSON line per case:

    python bench_implicit.py [--sizes 100x200,400x500] [--reps 3] [--no-reference]

Cases: ``solve_fwd`` / ``solve_bwd`` (one LearnedTimeDiffusion solve; the backward is one adjoint solve plus the time
gradient), ``net_fwd`` / ``net_fwd_bwd`` (a 4-block C = 128 DiffusionNet, 3 inputs, 8 outputs), the same two for the
spectral net, and ``reference_dense_fwd`` (the reference's LearnedTimeDiffusion on the same GPU through oracle/ref_import:
the mounted reference, else the copy ``build()`` staged under oracle/_ref).

Byte model of one CG iteration (fp64 state, V x C): the SpMM reads p once and writes q (16 V C) and reads L once
(int32 column + fp32 value pair, 12 B per entry); the x / r update reads x, r, p, q and writes x, r (48 V C); the p update
reads r, p and writes p (24 V C).  GB/s = iterations x (88 V C + 12 nnz) / time.  Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import diffusion_net_b200 as dn  # noqa: E402

C = 128


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = float(r.stdout.strip().splitlines()[0])
    except Exception:
        power = None
    return name, power


def checkpoint_times():
    with np.load(os.path.join(ROOT, "tests", "golden", "human_seg_xyz_4x128_f16.npz")) as z:
        return {k: torch.from_numpy(z[k].astype(np.float32)) for k in z.files if k.endswith("diffusion_time")}


def mesh(n, m, k, dev):
    verts, faces = dn.synthetic.torus_mesh(n, m, seed=0)
    verts = verts - verts.mean(0)
    verts = verts / verts.norm(dim=1).max()                          # unit max radius, as normalize_positions
    return dn.geometry.compute_operators(verts, faces, k, device=dev), faces


def timed(fn, reps):
    """Median ms of ``fn`` over ``reps`` calls after one warm-up call (events around a synchronised call)."""
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def iteration_bytes(V, nnz):
    return 88 * V * C + 12 * nnz


def emit(rec, gpu, power):
    rec.update(gpu=gpu, power_limit_w=power)
    print(json.dumps(rec), flush=True)


def bench_size(n, m, reps, times, gpu, power, dev):
    ops_k, _ = mesh(n, m, 128, dev)
    frames, mass, L, evals, evecs, gx, gy = ops_k
    V, nnz = int(mass.shape[0]), int(L.coalesce().indices().shape[1])
    size = dict(V=V, C=C, nnz_L=nnz)
    # one solve, block 0's learned times
    ltd = dn.LearnedTimeDiffusion(C, method="implicit_dense").to(dev)
    x = torch.randn(V, C, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    g = torch.randn(V, C, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    with torch.no_grad():
        ltd.diffusion_time.copy_(times["block_0.diffusion.diffusion_time"])
    with torch.no_grad():
        ms_f = timed(lambda: ltd(x, L, mass, None, None), reps)
    it_f = int(dn.ops.implicit_last_status[1])
    xg = x.clone().requires_grad_(True)

    def fwd_bwd():
        y = ltd(xg, L, mass, None, None)
        y.backward(g)
    ms_fb = timed(fwd_bwd, reps)
    it_b = int(dn.ops.implicit_last_status[1])
    ms_b = ms_fb - ms_f
    ib = iteration_bytes(V, nnz)
    emit(dict(case="solve_fwd", ms=ms_f, iterations=it_f, gb_s=it_f * ib / ms_f / 1e6, **size), gpu, power)
    emit(dict(case="solve_bwd", ms=ms_b, iterations=it_b, gb_s=it_b * ib / ms_b / 1e6, **size), gpu, power)
    # 4-block nets, implicit and spectral, with the checkpoint's times in every block
    xin = torch.randn(V, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(2))
    for method in ("implicit_dense", "spectral"):
        torch.manual_seed(0)
        net = dn.DiffusionNet(C_in=3, C_out=8, C_width=C, N_block=4, dropout=False, diffusion_method=method).to(dev)
        with torch.no_grad():
            for i, b in enumerate(net.blocks):
                b.diffusion.diffusion_time.copy_(times["block_{}.diffusion.diffusion_time".format(i)])
        kw = dict(L=L, gradX=gx, gradY=gy) if method == "implicit_dense" else dict(evals=evals, evecs=evecs, gradX=gx,
                                                                                   gradY=gy)
        with torch.no_grad():
            ms_nf = timed(lambda: net(xin, mass, **kw), reps)

        def net_step():
            net.zero_grad(set_to_none=True)
            net(xin, mass, **kw).square().mean().backward()
        ms_nfb = timed(net_step, reps)
        tag = "net" if method == "implicit_dense" else "spectral_net"
        emit(dict(case=tag + "_fwd", ms=ms_nf, N_block=4, **size), gpu, power)
        emit(dict(case=tag + "_fwd_bwd", ms=ms_nfb, N_block=4, **size), gpu, power)


def bench_reference(reps, times, gpu, power, dev):
    """The reference's dense implicit_dense (cholesky of a (1, C, V, V) fp32 matrix) beside ours, V = 2k."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import ref_import
    if not ref_import.reference_available():
        print(json.dumps(dict(case="reference_dense_fwd", skipped="reference not present or staged")), flush=True)
        return
    ref = ref_import.import_reference()
    ops_k, _ = mesh(40, 50, 0, dev)
    mass, L = ops_k[1], ops_k[2]
    V = int(mass.shape[0])
    t = times["block_0.diffusion.diffusion_time"]
    x = torch.randn(1, V, C, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    rl = ref.layers.LearnedTimeDiffusion(C, method="implicit_dense").to(dev)
    ours = dn.LearnedTimeDiffusion(C, method="implicit_dense").to(dev)
    with torch.no_grad():
        rl.diffusion_time.copy_(t)
        ours.diffusion_time.copy_(t)
        Lb, mb = torch.stack([L]), mass.unsqueeze(0)
        ms_ref = timed(lambda: rl(x, Lb, mb, None, None), reps)
        y_ref = rl(x, Lb, mb, None, None)
        ms_ours = timed(lambda: ours(x, Lb, mb, None, None), reps)
        y = ours(x, Lb, mb, None, None)
    err = float((y - y_ref).abs().max() / y_ref.abs().max())
    emit(dict(case="reference_dense_fwd", V=V, C=C, ms=ms_ref, ours_ms=ms_ours, speedup=ms_ref / ms_ours,
              max_rel_diff=err), gpu, power)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100x200,400x500")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_implicit.py needs a GPU")
    dev = torch.device("cuda")
    gpu, power = card()
    times = checkpoint_times()
    for s in a.sizes.split(","):
        n, m = (int(v) for v in s.split("x"))
        bench_size(n, m, a.reps, times, gpu, power, dev)
    if not a.no_reference:
        bench_reference(a.reps, times, gpu, power, dev)


if __name__ == "__main__":
    main()
