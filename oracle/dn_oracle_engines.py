"""The fused inference block forward (dn_block_fwd / _ex / _batched) restated per engine: every tensor-core operand
rounded exactly where the kernels round it, everything else plain arithmetic in the evaluation dtype.

TEST INFRASTRUCTURE ONLY (checker side, like ``dn_oracle``); the product never imports it.

Where the kernels round (diffusion-net_b200/csrc/dn_tc.cu, dn_tc_ptx.cuh):

* TF32 is round-to-nearest, ties away from zero (``cvt.rna``; the activations' ``split_tf32_fast`` adds half a TF32
  ulp to the magnitude bits, the same rounding).  tc3x splits an operand x = hi + lo and issues lo*hi + hi*lo + hi*hi:
  a weight's lo is ``cvt.rna(w - hi)``, an activation's lo is ``x - hi`` of which the MMA reads the top 19 bits (so it
  is truncated to TF32).  tc1x issues hi*hi only.
* bf16 is round-to-nearest-even (``cvt.rn.bf16x2`` for activations, ``__float2bfloat16_rn`` in the pack kernel).  A
  chain whose shapes do not fit the 16-wide bf16 K steps (``tc_chain_plan``) runs single-pass TF32 instead, and to_basis
  runs single-pass TF32 under the bf16 engine.
* The rounded operands: to_basis's A = Phi and B = fl32(m * x); the spectral multiplier S = expf(-lambda t) * sum,
  formed in the pack kernel and packed as from_basis's weight; from_basis's A = Phi; the [P|Q] layer's A = x_diffuse;
  MLP layer 0's A = [x | x_diffuse | features]; every later layer's A = the previous layer's activation after its
  epilogue; every weight.  The gradient-feature gather, the dots and tanh run on SIMT cores in fp32 (plain here).

``block_forward(..., engine=None)`` is ``dn_oracle.diffusion_net_block`` (no rounding).  With ``engine`` it follows
block_fwd_impl's dispatch (which layers run on tensor cores, whether [P|Q] is one layer or P and Q, whether the MiniMLP
is one chain or layer by layer) and rounds accordingly.  ``dtype=np.float32`` evaluates the same computation in fp32
(the floor of the tolerance model, tests/test_gpu_forward.py)."""
from __future__ import annotations

import numpy as np

__all__ = ["tf32_rna", "tf32_rz", "bf16_rn", "block_forward", "net_forward", "EMU_ENGINES", "dispatch"]

EMU_ENGINES = ("simt", "tc3x", "tc1x", "bf16")
MAX_CHAIN_LAYERS = 8          # DN_MAX_LAYERS


def _round_bits(x, bits, mode):
    """x rounded to ``bits`` significant bits (the implicit one included), in x's dtype; exponent range unbounded."""
    x = np.asarray(x)
    m, e = np.frexp(x.astype(np.float64))            # |m| in [0.5, 1)
    s = np.ldexp(np.abs(m), bits)                    # in [2^(bits-1), 2^bits)
    if mode == "rna":
        r = np.floor(s + 0.5)
    elif mode == "rne":
        r = np.rint(s)
    else:                                            # "rz"
        r = np.floor(s)
    return (np.copysign(np.ldexp(r, e - bits), m)).astype(x.dtype)


def tf32_rna(x):
    """cvt.rna.tf32.f32: 11 significant bits, ties away from zero."""
    return _round_bits(x, 11, "rna")


def tf32_rz(x):
    """the TF32 MMA's read of an fp32 register: the top 19 bits (truncation)."""
    return _round_bits(x, 11, "rz")


def bf16_rn(x):
    """cvt.rn.bf16.f32: 8 significant bits, ties to even."""
    return _round_bits(x, 8, "rne")


# ------------------------------------------------------------------------------------------------
# one dense layer in a given tensor-core mode
# ------------------------------------------------------------------------------------------------
def _mm(a, w_t, mode, dt, packed=True):
    """a (V,K) @ w_t (K,N) with both operands rounded as ``mode`` rounds them ("simt": none, "3x", "1x", "bf16");
    ``a`` is rounded as an activation (register split), ``w_t`` as a packed weight (pack kernel split) or, with
    ``packed=False``, as an activation too (to_basis's B image)."""
    a = a.astype(dt, copy=False)
    w_t = w_t.astype(dt, copy=False)
    if mode == "simt":
        return a @ w_t
    if mode == "bf16":
        return bf16_rn(a) @ bf16_rn(w_t)
    ah, wh = tf32_rna(a), tf32_rna(w_t)
    if mode == "1x":
        return ah @ wh
    al = tf32_rz((a - ah).astype(dt))
    wl = (tf32_rna if packed else tf32_rz)((w_t - wh).astype(dt))
    return al @ wh + ah @ wl + ah @ wh


# ------------------------------------------------------------------------------------------------
# dispatch of block_fwd_impl (dn_capi.cu) / tc_chain_plan / chain_supported (dn_tc.cu)
# ------------------------------------------------------------------------------------------------
def _chain_ok(src_widths, layers, bf16):
    """chain_supported: ``layers`` = [(K, N, sibling)]."""
    ks = 16 if bf16 else 8
    n = len(layers)
    if n < 1 or n > MAX_CHAIN_LAYERS or any(w % ks for w in src_widths) or sum(src_widths) != layers[0][0]:
        return False
    for l, (K, N, sib) in enumerate(layers):
        if K % ks or K < ks or N % 16 or N < 16 or N > (128 if n > 1 else 256):
            return False
        if sib and l < 2:
            return False
        if l > 0 and K != (layers[l - 1][0] if sib else layers[l - 1][1]):
            return False
    return True


def _plan(src_widths, layers, passes):
    """tc_chain_plan -> the mode the chain runs in, or None (not a tensor-core chain)."""
    if passes == "bf16" and _chain_ok(src_widths, layers, True):
        return "bf16"
    if _chain_ok(src_widths, layers, False):
        return "1x" if passes in ("1x", "bf16") else "3x"
    return None


def _to_basis_tc(K, C):
    ok = lambda k, c: k % 4 == 0 and 4 <= k <= 128 and c % 16 == 0 and 16 <= c <= 128
    return ok(K, C) or (C > 128 and C % 128 == 0 and ok(K, 128))


def _mlp_modes(src_widths, dims, passes):
    """run_chain over the MiniMLP: one chain when it fits (every layer in the chain's mode), else layer by layer."""
    layers = [(dims[i], dims[i + 1], 0) for i in range(len(dims) - 1)]
    if passes is None:
        return ["simt"] * len(layers), False
    m = _plan(src_widths, layers, passes)
    if m is not None:
        return [m] * len(layers), True
    modes, w = [], list(src_widths)
    for L in layers:
        mm = _plan(w, [L], passes) if len(layers) > 1 else None
        modes.append(mm or "simt")
        w = [L[1]]
    return modes, False


def dispatch(engine, K, C, dims, with_features=True, rot=True):
    """{stage: mode} the block forward reaches on ``engine``: to_basis, from_basis, pq (list: one entry per [P|Q] layer),
    mlp (list per layer), plus the chain layout ('front_fused', 'mlp_fused')."""
    passes = {"simt": None, "tc3x": "3x", "tc1x": "1x", "bf16": "bf16"}[engine]
    tc = passes is not None
    d = {"to_basis": ("3x" if passes == "3x" else "1x") if tc and _to_basis_tc(K, C) else "simt"}
    front = [(K, C, 0)]
    if with_features:
        npq = 2 * C if rot else C
        if rot and (npq > 256 or (tc and npq > 128)):
            front += [(C, C, 0), (C, C, 1)]
        else:
            front += [(C, npq, 0)]
    fused = tc and len(front) > 1 and _plan([K], front, passes) is not None
    if fused:
        modes = [_plan([K], front, passes)] * len(front)
    else:   # each layer its own run_chain: tensor cores when its plan takes it, SIMT otherwise
        modes = [(_plan([K], front[:1], passes) if tc else None)]
        modes += [(_plan([C], [(L[0], L[1], 0)], passes) if tc else None) for L in front[1:]]
        modes = [m or "simt" for m in modes]
    d["from_basis"] = modes[0]
    d["pq"] = modes[1:]
    d["front_fused"] = fused
    nsrc = 3 if with_features else 2
    d["mlp"], d["mlp_fused"] = _mlp_modes([C] * nsrc, dims, passes)
    return d


# ------------------------------------------------------------------------------------------------
# the block and the net
# ------------------------------------------------------------------------------------------------
def _mlp_weights(params):
    ws, bs, i = [], [], 0
    while "mlp.miniMLP_mlp_layer_{:03d}.weight".format(i) in params:
        ws.append(params["mlp.miniMLP_mlp_layer_{:03d}.weight".format(i)])
        bs.append(params["mlp.miniMLP_mlp_layer_{:03d}.bias".format(i)])
        i += 1
    return ws, bs


def block_forward(x_in, mass, evals, evecs, gradX, gradY, params, engine=None, dtype=np.float64,
                  with_gradient_features=True, head=None, perturb=None):
    """One block (optionally with the fused head ``(W, b)``) on one mesh.

    Returns the block output (or the head output).  ``perturb``: a set of named structural errors for
    the sensitivity tests (drop_last_eig, time, swap_re_im, zero_feature, drop_hidden_bias, zero_last_tile)."""
    dt = dtype
    pert = perturb or set()
    f = lambda a: np.asarray(a).astype(dt)
    x, m, lam, phi = f(x_in), f(mass), f(evals), f(evecs)
    V, C = x.shape
    K = phi.shape[1]
    rot = "gradient_features.A.weight" not in params
    ws, bs = _mlp_weights(params)
    ws, bs = [f(w) for w in ws], [f(b) for b in bs]
    dims = [ws[0].shape[1]] + [w.shape[0] for w in ws]
    t = f(params["diffusion.diffusion_time"]).copy()
    if "time" in pert:
        t[0] *= dt(1 + 1e-3)
    if "drop_last_eig" in pert:
        phi = phi.copy()
        phi[:, K - 1] = 0
    if "drop_hidden_bias" in pert and len(bs) > 1:
        bs[0] = bs[0].copy()
        bs[0][0] = 0
    d = dispatch(engine or "simt", K, C, dims, with_gradient_features, rot)
    tb_mode = d["to_basis"]
    # to_basis: Phi^T (m x); the tensor-core kernel forms m * x in fp32 and splits it
    if engine and tb_mode != "simt":
        S_sum = _mm(phi.T, (x * m[:, None]).astype(np.float32).astype(dt), tb_mode, dt, packed=False)
    else:
        S_sum = phi.T @ (x * m[:, None])
    S = (np.exp(-(lam[:, None] * np.maximum(t, dt(1e-8))[None, :])) * S_sum).astype(dt)
    xd = _mm(phi, S, d["from_basis"] if engine else "simt", dt)
    srcs = [x, xd]
    if with_gradient_features:
        if rot:
            A_re, A_im = f(params["gradient_features.A_re.weight"]), f(params["gradient_features.A_im.weight"])
            if "swap_re_im" in pert:
                A_re, A_im = A_im, A_re
        else:
            A_re, A_im = f(params["gradient_features.A.weight"]), None
        pq_modes = d["pq"] if engine else ["simt"]
        P = _mm(xd, A_re.T, pq_modes[0], dt)
        Q = _mm(xd, A_im.T, pq_modes[-1], dt) if rot else None
        gX, gY = gradX.astype(dt), gradY.astype(dt)
        # the commuted gather: Bre = gX P - gY Q, Bim = gY P + gX Q  (= (gX xd) A_re^T - (gY xd) A_im^T, ...)
        bre = gX @ P - (gY @ Q if rot else 0)
        bim = gY @ P + (gX @ Q if rot else 0)
        feats = np.tanh((gX @ xd) * bre + (gY @ xd) * bim).astype(dt)
        if "zero_feature" in pert:
            feats[:, 0] = 0
        srcs.append(feats)
    h = np.concatenate(srcs, axis=1)
    modes = d["mlp"] if engine else ["simt"] * len(ws)
    for i, (w, b) in enumerate(zip(ws, bs)):
        z = (_mm(h, w.T, modes[i], dt) + b).astype(dt)
        h = np.maximum(z, 0) if i + 1 < len(ws) else (z + x).astype(dt)
    out = h
    if head is not None:
        hw, hb = f(head[0]), f(head[1]) if head[1] is not None else None
        out = (h @ hw.T + (hb if hb is not None else 0)).astype(dt)
    if "zero_last_tile" in pert and V % 128:
        out = out.copy()
        out[V - V % 128:] = 0
    return out


def net_forward(x_in, mass, evals, evecs, gradX, gradY, params, n_block, engine=None, dtype=np.float64,
                with_gradient_features=True):
    """DiffusionNet (outputs at vertices) through the blocks of ``block_forward``: first_lin and last_lin run through
    run_chain as single layers (tensor cores when their shapes allow), or last_lin fused into the last block when the
    head fits (<= 8 outputs and a tensor-core MiniMLP chain)."""
    dt = dtype
    f = lambda a: np.asarray(a).astype(dt)
    passes = {None: None, "simt": None, "tc3x": "3x", "tc1x": "1x", "bf16": "bf16"}[engine]

    def lin(x, W, b):
        W = f(W)
        mode = (_plan([x.shape[1]], [(W.shape[1], W.shape[0], 0)], passes) if passes else None) or "simt"
        return (_mm(x, W.T, mode, dt) + f(b)).astype(dt)

    x = lin(f(x_in), params["first_lin.weight"], params["first_lin.bias"])
    hw, hb = params["last_lin.weight"], params["last_lin.bias"]
    for i in range(n_block):
        pre = "block_{}.".format(i)
        bp = {k[len(pre):]: v for k, v in params.items() if k.startswith(pre)}
        last = i + 1 == n_block
        C = x.shape[1]
        dims = [bp["mlp.miniMLP_mlp_layer_000.weight"].shape[1]] + [w.shape[0] for w in _mlp_weights(bp)[0]]
        fuse = last and 1 <= hw.shape[0] <= 8 and dispatch(engine or "simt", evecs.shape[1], C, dims,
                                                           with_gradient_features)["mlp_fused"]
        x = block_forward(x, mass, evals, evecs, gradX, gradY, bp, engine=engine, dtype=dt,
                             with_gradient_features=with_gradient_features, head=(hw, hb) if fuse else None)
        if last and fuse:
            return x
    return lin(x, hw, hb)
