"""Per-chain timing of the fused row-chain kernel (rows_chain_kernel), and of to_basis, at the headline block's shapes.

Each chain is called alone through its C-ABI entry point, tc3x, K = C = 128:

  from_basis   dn_from_basis,   evecs (V, 128) -> (V, 128)
  pq           dn_mini_mlp_fwd, one 128 -> 256 layer (the [P|Q] shape of the gradient features)
  front        from_basis, P and Q as the one chain the block forward runs (dn_block_fwd_profile, its from_basis_pq
               stage): evecs (V, 128) -> x_diffuse (V, 128), then P, Q (V, 128) each into one (V, 256) buffer
  mlp          dn_mini_mlp_fwd, cat(3 x (V, 128)) -> 128 -> 128 with ReLU, biases and the residual (the MiniMLP)
  to_basis     dn_to_basis,     evecs^T (mass * x): the split-V to_basis kernel and its partial reduction

A call is the weight-pack launch (a few microseconds) plus the chain launch; it is timed with CUDA events over
--iters calls after --warmup calls.  The front chain is timed inside a whole block forward (CUDA events around its
launch alone, from the profiling entry point, averaged over --iters forwards after --warmup), so it has no pack launch.  Bytes and TF32 MMA operations come from the shapes (3 MMA passes in tc3x); the
floors are bytes over the data-sheet HBM rate and MMA operations over a TF32 rate measured in the same run with a
large torch matmul (TF32 on).  The weight bytes each row tile streams from L2 (192-row tiles for mlp, 128-row
tiles for the single-layer chains and the front chain with its sibling) are reported as an implied L2 rate.
The same chains at V = 20k, whose inputs stay resident in the 50 MB L2, give the time per row without HBM latency.

    python bench_chain.py [--root DIR] [--iters 100] [--warmup 10] [--json FILE]

--root imports the package from another checkout (to compare two builds in one session, one process each).
Prints the card, its power limit and SM clocks (a read-only nvidia-smi query), one table, one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys

HBM_TBS = 3.35            # H100 SXM data sheet, HBM3
PASSES = 3                # tc3x: lo*hi + hi*lo + hi*hi
KC = 16                   # K columns per weight stage
K = C = 128


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi: n/a"
    except (OSError, subprocess.SubprocessError):
        return "nvidia-smi: n/a"


def chain_model(name, V):
    """(HBM bytes, TF32 MMA flops, L2 weight bytes) of one call; weights hi + lo, 16 * N * 8 bytes per K stage."""
    if name == "from_basis":
        layers, rows_in, rows_out = [(K, C)], K, C
    elif name == "pq":
        layers, rows_in, rows_out = [(C, 2 * C)], C, 2 * C
    elif name == "front":  # evecs in; x_diffuse, P and Q out
        layers, rows_in, rows_out = [(K, C), (C, C), (C, C)], K, 3 * C
    elif name == "to_basis":  # evecs, x and mass in; a K x C result (no weights)
        return 4 * V * (K + C + 1), 2 * V * K * C * PASSES, 0
    else:  # mlp: 3 sources + residual in, C out
        layers, rows_in, rows_out = [(3 * C, C), (C, C), (C, C)], 4 * C, C
    hbm = 4 * V * (rows_in + rows_out)
    flops = 2 * V * sum(k * n for k, n in layers) * PASSES
    # several layers, every one 128 wide, no sibling: three consumer warpgroups share each weight stage over 192-row tiles
    tile = 192 if name == "mlp" else 128
    tiles = (V + tile - 1) // tile
    l2w = tiles * sum(((k + KC - 1) // KC) * KC * n * 8 for k, n in layers)
    return hbm, flops, l2w


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(os.path.abspath(__file__)))
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", help="also write the result line to this file")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    import diffusion_net_b200 as dn
    from diffusion_net_b200 import _lib, ops

    assert torch.cuda.is_available(), "bench_chain.py needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dn.set_engine("tc3x")
    lib = _lib.load()
    eng = _lib.ENGINE_TC3X
    card = gpu_info()

    def timed(fn, iters, warm):
        for _ in range(warm):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    # the TF32 tensor-core rate this card sustains now (cuBLAS, 8192^3)
    torch.backends.cuda.matmul.allow_tf32 = True
    a = torch.randn(8192, 8192, device=dev)
    b = torch.randn(8192, 8192, device=dev)
    mm_ms = timed(lambda: torch.mm(a, b), 20, 3)
    tf32_tflops = 2 * 8192 ** 3 / (mm_ms * 1e-3) / 1e12
    del a, b

    g = torch.Generator(device=dev).manual_seed(0)

    def rnd(*shape, scale=1.0):
        return torch.randn(*shape, device=dev, generator=g) * scale

    rows = []
    for V in (200_000, 20_000):
        ws = ops.workspace(V, 2 * C, 2 * C, dev)
        st = ops._stream()
        evecs, spec = rnd(V, K), rnd(K, C, scale=0.1)
        xd, x, feat = rnd(V, C), rnd(V, C), rnd(V, C)
        out_c, out_2c, hid = torch.empty(V, C, device=dev), torch.empty(V, 2 * C, device=dev), torch.empty(V, C, device=dev)
        w_pq = rnd(2 * C, C, scale=C ** -0.5)
        w_mlp = [rnd(C, 3 * C, scale=(3 * C) ** -0.5), rnd(C, C, scale=C ** -0.5), rnd(C, C, scale=C ** -0.5)]
        b_mlp = [rnd(C, scale=0.1) for _ in range(3)]

        def call_fb():
            _lib.check(lib.dn_from_basis(spec.data_ptr(), evecs.data_ptr(), None, V, K, C, out_c.data_ptr(),
                                         ws.data_ptr(), ws.numel(), eng, st), "dn_from_basis")

        pq_args = (_lib.ptr_array([xd.data_ptr()]), _lib.int_array([C]), 1, _lib.ptr_array([w_pq.data_ptr()]),
                   None, _lib.int_array([C, 2 * C]), 1, None, None, V, None, out_2c.data_ptr())

        def call_pq():
            _lib.check(lib.dn_mini_mlp_fwd(*pq_args, ws.data_ptr(), ws.numel(), eng, st), "dn_mini_mlp_fwd")

        mlp_args = (_lib.ptr_array([x.data_ptr(), xd.data_ptr(), feat.data_ptr()]), _lib.int_array([C, C, C]), 3,
                    _lib.ptr_array([w.data_ptr() for w in w_mlp]), _lib.ptr_array([b.data_ptr() for b in b_mlp]),
                    _lib.int_array([3 * C, C, C, C]), 3, None, x.data_ptr(), V, None, out_c.data_ptr())

        def call_mlp():
            _lib.check(lib.dn_mini_mlp_fwd(*mlp_args, ws.data_ptr(), ws.numel(), eng, st), "dn_mini_mlp_fwd")

        mass = torch.rand(V, device=dev, generator=g) + 0.5
        out_kc = torch.empty(K, C, device=dev)

        def call_tb():
            _lib.check(lib.dn_to_basis(x.data_ptr(), evecs.data_ptr(), mass.data_ptr(), V, K, C, out_kc.data_ptr(),
                                       ws.data_ptr(), ws.numel(), eng, st), "dn_to_basis")

        # the front chain as the block forward runs it, at the block's shapes (with rotations, MiniMLP 384 -> 128 -> 128)
        n_side = 500 if V == 200_000 else 200
        mass_b, _, evals_b, evecs_b, gX, gY = dn.synthetic.structural_operators(n_side, V // n_side, K, seed=0, device=dev)
        blk = dn.DiffusionNetBlock(C_width=C, mlp_hidden_dims=[C, C], dropout=False)
        blk.load_state_dict(dn.synthetic.block_weights(C, seed=0), strict=True)
        blk = blk.to(dev).eval()
        gops = dn.prepare_operators(gX, gY)
        A_re, A_im = blk.gradient_features.weights()
        lins = blk.mlp.linears()
        front_stage = ops.PROFILE_STAGES.index("from_basis_pq")

        def time_front(iters, warm):
            tot = 0.0
            with torch.no_grad():
                for i in range(warm + iters):
                    prof = []
                    ops.block_forward_raw(x, mass_b, evals_b, evecs_b, gops, blk.diffusion.diffusion_time, A_re, A_im,
                                          [l.weight for l in lins], [l.bias for l in lins], True, profile=prof)
                    if i >= warm:
                        tot += prof[front_stage]
            return tot / iters

        for name, fn in (("from_basis", call_fb), ("pq", call_pq), ("front", None), ("mlp", call_mlp),
                         ("to_basis", call_tb)):
            ms = time_front(args.iters, args.warmup) if fn is None else timed(fn, args.iters, args.warmup)
            hbm, flops, l2w = chain_model(name, V)
            rows.append({
                "chain": name, "V": V, "ms": round(ms, 4), "ns_per_row": round(ms * 1e6 / V, 3),
                "hbm_MB": round(hbm / 1e6, 1), "mma_GFLOP": round(flops / 1e9, 2),
                "TBps": round(hbm / (ms * 1e-3) / 1e12, 3), "TFLOPps": round(flops / (ms * 1e-3) / 1e12, 1),
                "floor_hbm_ms": round(hbm / (HBM_TBS * 1e12) * 1e3, 4),
                "floor_mma_ms": round(flops / (tf32_tflops * 1e12) * 1e3, 4),
                "l2_weight_GB": round(l2w / 1e9, 3), "l2_weight_TBps": round(l2w / (ms * 1e-3) / 1e12, 2),
            })
        del ws
        torch.cuda.empty_cache()

    print("card (name, power limit, max SM clock, SM clock now):", card)
    print("root:", os.path.abspath(args.root))
    print("cuBLAS TF32 8192^3: {:.3f} ms = {:.0f} TFLOP/s (the MMA floor's rate)".format(mm_ms, tf32_tflops))
    hdr = "{:<11}{:>8}{:>9}{:>10}{:>9}{:>10}{:>8}{:>9}{:>11}{:>11}{:>9}{:>9}"
    print(hdr.format("chain", "V", "ms", "ns/row", "HBM MB", "MMA GF", "TB/s", "TFLOP/s", "floor HBM", "floor MMA",
                     "L2w GB", "L2w TB/s"))
    for r in rows:
        print(hdr.format(r["chain"], r["V"], r["ms"], r["ns_per_row"], r["hbm_MB"], r["mma_GFLOP"], r["TBps"],
                         r["TFLOPps"], r["floor_hbm_ms"], r["floor_mma_ms"], r["l2_weight_GB"], r["l2_weight_TBps"]))
    res = {"card": card, "root": os.path.abspath(args.root), "tf32_tflops": round(tf32_tflops, 1), "chains": rows}
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
