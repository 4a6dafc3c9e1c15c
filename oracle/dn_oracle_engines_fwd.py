"""The training forward's entry points dn_learned_time_diffusion_fwd (and _batched, dn_to_basis_batched,
dn_from_basis_batched), dn_gradient_features_fwd, dn_mini_mlp_fwd and dn_compute_hks restated per engine, each result
with a componentwise error bound that holds for any fp32 accumulation order.

TEST INFRASTRUCTURE ONLY (checker side, like ``dn_oracle_engines`` and ``dn_oracle_engines_bwd``, whose rounding
model and contraction bound this module reuses); the product never imports it.

Each training entry point writes its intermediates (x_spec, [P|Q], the hidden activations), and the backward reads
them.  So every stage is checked on the fp32 values the kernel itself read: x_diffuse on the call's own x_spec_out,
the features on its own pq_out, MiniMLP layer l on its own hidden_out[l - 1].  No rounding flip of one stage then
propagates into the next stage's gold, and the only band left is that of the spectral multiplier S, which the kernel
forms and rounds again when it packs it (``_spread``).

Where the forward rounds, beyond the contractions of ``dn_oracle_engines_bwd``:

* to_basis (to_basis_partials): Phi^T fl32(m * x).  The tensor-core kernel and the SIMT kernel (atb_partial_kernel,
  ``b[j] *= s``) both form the fp32 product m * x before the contraction.  spectral_scale_kernel sums the P partials as
  4 slices, each serially, then pairwise; the batched pack kernel does the same over 8 slices.  x_spec_out is that
  fp32 sum; S = expf(-(lambda * max(t, 1e-8))) * sum is formed from the same register.
* the [P|Q] layer of dn_gradient_features_fwd: one run_chain layer xd [A_re; A_im]^T (W2 / n_split), not transposed.
* the features gather (feat_entry / feat_value, dn_simt.cu): fmaf chains in CSR order, nnz terms for gX and gY, 2 nnz
  for Bre and Bim with rotations (nnz without); arg = fmaf(gX, Bre, gY * Bim); feature = dn_feat_tanh(arg).
* dn_feat_tanh(x) = 1 - __fdividef(2, __expf(2 x) + 1).  Its absolute error ``tanh_error`` is derived from the CUDA C++
  Programming Guide's documented maximum errors (Intrinsic Functions): __expf(y) within 2 + floor(|1.173 y|) ulp,
  __fdividef(x, y) within 2 ulp for |y| in [2^-126, 2^126] (0 above it); the add and the subtraction round once.
* the MiniMLP: run_chain's epilogue, bias, relu, emul (dropout), then on the last layer the residual (fmaf).
* the fused block's head (dn_block_fwd_ex with a dn_head, DiffusionNet.last_lin in the MiniMLP epilogue): fp32 fmaf
  chains over the finished fp32 row, C / 4 terms per lane, a 2-level butterfly over 4 lanes, then + b.
* dn_compute_hks: out[v, s] = sum_k expf(-(lambda_k s)) phi_vk^2.  Each lane runs an fmaf chain over its
  ceil(K / 32) eigenpairs, and a 5-level butterfly over the 32 lanes sums them (hks_warp_kernel and
  hks_generic_kernel alike).  Every term is >= 0, so the bound is relative to the element.

``tree_sum`` restates, bitwise, the fp32 sums of the split-V partials that spectral_scale_kernel (4 slices) and the pack
kernel's spectral job (8 slices) form; the fused block keeps only the partials, so its x_spec is checked on that sum.

``PERTURBATIONS``, ``HEAD_PERTURBATIONS``: named structural errors for the sensitivity tests."""
from __future__ import annotations

import numpy as np

from dn_oracle_engines import _mlp_modes
from dn_oracle_engines_bwd import (C_SAFE, PARTIAL_FLOATS, PASSES, U, _dense, _last_tile, _mode, _split_v, from_basis,
                                   layer_mode, to_basis_mode)

__all__ = ["diffusion_fwd", "tree_sum", "head_fwd", "clamped_time", "to_basis_batched", "from_basis_batched", "features_fwd", "tanh_error",
           "mini_mlp_fwd", "compute_hks", "routes", "mlp_on_tc", "PERTURBATIONS", "HEAD_PERTURBATIONS"]

TIME_MIN = np.float32(1e-8)   # dn_clamp_time
TIME_COL = 4                  # the channel whose time "time_scaled" perturbs (0 .. 3 are the edge times)
PERTURBATIONS = {
    "diffusion": ("drop_eig", "time_scaled", "no_clamp", "drop_last_partial", "x_spec_scaled", "1x_for_bf16",
                  "1x_for_3x"),
    "features": ("swap_re_im", "q_from_re", "drop_last_entry", "drop_gy_bim", "zero_channel", "tanh_2e-16"),
    "mlp": ("drop_hidden_bias", "hidden_before_emul", "residual_last_tile", "relu_last", "dropout_col",
            "wrong_w0_block", "bf16_for_1x"),
    "hks": ("drop_eig", "scale_scaled"),
}
HEAD_PERTURBATIONS = ("head_wrong_bias", "head_drop_col", "head_before_residual")   # head_fwd's, for the fused block
_f = lambda v: None if v is None else np.asarray(v, np.float64)


def _heat(lam, t):
    """exp(-lambda t) for t (C,) and its band: expf within 2 ulp, lambda * t rounded once (its relative error moves
    the exponent by |lambda t| u); an underflow to a denormal or zero is off by at most the smallest denormal."""
    lt = lam[:, None] * t[None, :]
    e = np.exp(-lt)
    return e, e * (np.abs(lt) * U + 2 * U) + 2.0 ** -149


def clamped_time(time, pert=()):
    """``time`` after the call: max(t, 1e-8) in fp32, bitwise."""
    t32 = np.asarray(time, np.float32)
    return t32.copy() if "no_clamp" in pert else np.maximum(t32, TIME_MIN)


def diffusion_fwd(x, mass, evals, evecs, time, engine, x_spec_out=None, sm=132, part_floats=PARTIAL_FLOATS, pert=(),
                  stats=None, split=None, tree=4, cache=None, fb_mode=None):
    """dn_learned_time_diffusion_fwd: {"x_spec": (gold, bound), "time": fp32, "x_diffuse": (gold, bound)}.

    x_diffuse is checked on ``x_spec_out`` (the call's own fp32 sums; the gold's x_spec when None).  One mesh of the
    batched call with ``split`` = its CTA plan's (P, rows per CTA) and ``tree`` = 8.  ``cache``: a dict shared by the
    calls on the same inputs, so that engines whose to_basis rounds alike share its gold.  ``fb_mode``: from_basis's
    mode when it leads a longer chain (the fused block's front, dn_oracle_engines.dispatch)."""
    xv, m, lam, phi = _f(x), _f(mass), _f(evals), _f(evecs)
    K, C = phi.shape[1], xv.shape[1]
    tb = _mode(to_basis_mode(engine, K, C, sm, part_floats), pert)
    key = (tb, "drop_last_partial" in pert)
    if cache is not None and key in cache:
        xs, exs = cache[key]
    else:
        y = (np.asarray(x, np.float32) * np.asarray(mass, np.float32)[:, None]).astype(np.float64)   # fl32(m * x)
        xs, exs = _split_v(phi, y, tb, sm, part_floats, pert=pert, split=split, tree=tree)
        if cache is not None:
            cache[key] = xs, exs
    t = clamped_time(time, pert).astype(np.float64)
    if "time_scaled" in pert:
        t[TIME_COL] *= 1 + 1e-3
    e, ee = _heat(lam, t)
    if "drop_eig" in pert:
        e = e.copy()
        e[K - 1] = 0
    res = {"x_spec": (e * xs, exs) if "x_spec_scaled" in pert else (xs, exs), "time": clamped_time(time, pert)}
    xk = xs if x_spec_out is None else _f(x_spec_out)
    S = e * xk
    eS = np.abs(xk) * ee + U * np.abs(S)
    res["x_diffuse"] = from_basis(S, phi, None, engine, pert=pert, eW=eS, stats=stats, mode=fb_mode)
    return res


def tree_sum(partials, tree):
    """The fp32 sum over the partials (P, ...) as the kernels reduce them: slice s adds partials s, s + tree, ... serially
    from 0, then the ``tree`` slice sums pairwise (dn_internal.h pairwise_sum).  Bitwise, in IEEE fp32."""
    p = np.asarray(partials, np.float32)
    red = [np.zeros(p.shape[1:], np.float32) for _ in range(tree)]
    for q in range(p.shape[0]):
        red[q % tree] = red[q % tree] + p[q]
    while len(red) > 1:
        red = [red[i] + red[i + 1] for i in range(0, len(red), 2)]
    return red[0]


def to_basis_batched(values, mass, evecs, engine, split, sm=132):
    """One mesh of dn_to_basis_batched: Phi^T fl32(m * x) over the planned CTAs, reduce_partials serially."""
    K, C = evecs.shape[1], values.shape[1]
    y = (np.asarray(values, np.float32) * np.asarray(mass, np.float32)[:, None]).astype(np.float64)
    return _split_v(_f(evecs), y, to_basis_mode(engine, K, C, sm, PARTIAL_FLOATS), sm, PARTIAL_FLOATS, split=split)


def from_basis_batched(values, evecs, row_scale, engine):
    """One mesh of dn_from_basis_batched: the pack kernel packs G as given ("plain"), so there is no band."""
    return from_basis(values, evecs, row_scale, engine)


# ------------------------------------------------------------------------------------------------
# gradient features
# ------------------------------------------------------------------------------------------------
EXPF_ULP_PER_ARG = 1.173      # __expf(y): 2 + floor(|1.173 y|) ulp
FDIV_ULP = 2                  # __fdividef(x, y), |y| in [2^-126, 2^126]


def tanh_error(lo, hi):
    """The largest absolute error of dn_feat_tanh(x) over x in [lo, hi] (elementwise), from the documented errors alone.

    With E = exp(2x), t = tanh x:  e = __expf(2x) = E (1 + d1), |d1| <= (2 + floor(1.173 |2x|)) 2^-23 (one ulp of a
    value is at most 2^-23 of it);  s = fl(e + 1) within 2^-24 relative;  q = __fdividef(2, s) within 2 ulp, so 2^-22
    relative;  f = fl(1 - q) within 2^-24 |f|.  Since 2 / (E + 1) = 1 - t and d(2 / (E + 1)) / dE * E = -(1 - t^2) / 2:
        |f - t| <= (1 - t^2) / 2 * |d1| + (2^-24 + 2^-22) (1 - t) + 2^-24 |t|,
    to first order; the factor (1 + 2^-20) covers the second.  Above |s| = 2^126 __fdividef returns 0 while the quotient
    is below 2^-125, and __expf flushes a result below 2^-126 to zero: the 2^-124 covers both.  Each factor is taken at
    its largest over the interval (1 - t^2 at the point nearest 0, 1 - t at lo, |t| and the ulp count at the largest
    |x|)."""
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    amax = np.maximum(np.abs(lo), np.abs(hi))
    amin = np.where((lo <= 0) & (hi >= 0), 0.0, np.minimum(np.abs(lo), np.abs(hi)))
    with np.errstate(invalid="ignore", over="ignore"):
        n_e = 2 + np.floor(EXPF_ULP_PER_ARG * 2 * np.minimum(amax, 1e30))
        d1 = n_e * 2.0 ** -23
        t_near0 = np.tanh(amin)
        T = (d1 * (1 - t_near0 * t_near0) / 2 + (2.0 ** -24 + FDIV_ULP * 2.0 ** -23) * (1 - np.tanh(lo))
             + 2.0 ** -24 * np.tanh(amax))
    return T * (1 + 2.0 ** -20) + 2.0 ** -124


def _pq_weight(A_re, A_im, pert):
    """[A_re ; A_im]^T (C, npq), the layer's weight as it reads it."""
    A_re, A_im = _f(A_re), _f(A_im)
    if A_im is None:
        return A_re.T
    if "swap_re_im" in pert:
        A_re, A_im = A_im, A_re
    if "q_from_re" in pert:
        A_im = A_re
    return np.vstack([A_re, A_im]).T


def features_fwd(gX, gY, x_diffuse, A_re, A_im, engine, pq_out=None, pert=(), stats=None, mode=None):
    """dn_gradient_features_fwd: {"pq": (gold, bound), "features": (gold, bound), "arg": (gold, band)}.  gX, gY:
    scipy.sparse CSR (V, V) on one pattern with fp32 values; A_im None without rotations.  The features are checked on
    ``pq_out`` (the call's own [P|Q]; the gold's when None) and the exact x_diffuse.  ``mode``: the [P|Q] layers' mode
    in the fused block (dn_oracle_engines.dispatch: a front chain's, or P and Q as two layers); the single layer's plan
    when None."""
    import scipy.sparse as sp
    rot = A_im is not None
    xd = _f(x_diffuse)
    V, C = xd.shape
    W = _pq_weight(A_re, A_im, pert)
    npq = W.shape[1]
    mode = _mode(mode or layer_mode(engine, [C], C, npq), pert)
    res = {"pq": _dense(xd, W, mode, stats=stats)}
    pq = res["pq"][0] if pq_out is None else _f(pq_out)
    Pm, Qm = pq[:, :C], (pq[:, C:2 * C] if rot else None)
    gX, gY = gX.tocsr(), gY.tocsr()
    if "drop_last_entry" in pert:       # every row's last CSR entry
        last = np.diff(gX.indptr) > 0
        keep = np.ones(gX.nnz, bool)
        keep[gX.indptr[1:][last] - 1] = False
        r, c = np.repeat(np.arange(V), np.diff(gX.indptr))[keep], gX.indices[keep]
        gX = sp.csr_matrix((gX.data[keep], (r, c)), shape=(V, V))
        gY = sp.csr_matrix((gY.data[keep], (r, c)), shape=(V, V))
    aX, aY = abs(gX), abs(gY)
    nnz = np.diff(gX.indptr)[:, None].astype(np.float64)
    Lg = C_SAFE * U * nnz                            # an fmaf chain of nnz terms
    Lb = C_SAFE * U * nnz * (2 if rot else 1)
    gXx, gYx = gX @ xd, gY @ xd
    egX, egY = Lg * (aX @ np.abs(xd)), Lg * (aY @ np.abs(xd))
    if rot:
        bre, bim = gX @ Pm - gY @ Qm, gY @ Pm + gX @ Qm
        mre = aX @ np.abs(Pm) + aY @ np.abs(Qm)
        mim = aY @ np.abs(Pm) + aX @ np.abs(Qm)
    else:
        bre, bim = gX @ Pm, gY @ Pm
        mre, mim = aX @ np.abs(Pm), aY @ np.abs(Pm)
    ere, eim = Lb * mre, Lb * mim
    if "drop_gy_bim" in pert:
        bim = np.zeros_like(bim)
    # arg = fmaf(gX, Bre, fl(gY * Bim)): the propagated errors of the four sums, the product's rounding, the fma's
    arg = gXx * bre + gYx * bim
    ea = (np.abs(bre) * egX + np.abs(gXx) * ere + egX * ere + np.abs(bim) * egY + np.abs(gYx) * eim + egY * eim)
    ea = ea + U * (np.abs(gYx) + egY) * (np.abs(bim) + eim)
    ea = ea + U * (np.abs(arg) + ea)
    ft = np.tanh(arg)
    slope = 1 - np.tanh(np.maximum(np.abs(arg) - ea, 0.0)) ** 2   # sup of tanh' over the band
    fb = slope * ea + tanh_error(arg - ea, arg + ea)
    if "zero_channel" in pert:
        ft = ft.copy()
        ft[:, 0] = 0
    if "tanh_2e-16" in pert:
        ft = ft + 2.0 ** -16
    res["features"] = (ft, fb)
    res["arg"] = (arg, ea)
    return res


# ------------------------------------------------------------------------------------------------
# MiniMLP
# ------------------------------------------------------------------------------------------------
def mini_mlp_fwd(srcs, weights, biases, drops, residual, engine, hidden=None, pert=(), stats=None):
    """dn_mini_mlp_fwd: {"hidden": [(gold, bound)] per hidden layer, "out": (gold, bound)}.  weights[l] (dims[l + 1],
    dims[l]); biases[l] or None; drops[l] (the dropout multiplier of hidden layer l) or None; residual (V, dims[-1]) or
    None.  Layer l > 0 is checked on ``hidden[l - 1]`` (the call's own activations; the gold's when None)."""
    n = len(weights)
    Ws = [_f(w) for w in weights]
    bs = [_f(b) for b in (biases or [None] * n)]
    D = [_f(d) for d in drops] if drops is not None else [None] * (n - 1)
    widths = [s.shape[1] for s in srcs]
    dims = [sum(widths)] + [w.shape[0] for w in Ws]
    V = srcs[0].shape[0]
    modes, _ = _mlp_modes(widths, dims, PASSES[engine])
    if "drop_hidden_bias" in pert and n > 1 and bs[0] is not None:
        bs[0] = bs[0].copy()
        bs[0][0] = 0
    if "wrong_w0_block" in pert and len(srcs) > 1:
        Ws[0] = Ws[0].copy()
        Ws[0][:, widths[0]:2 * widths[0]] = Ws[0][:, :widths[0]]
    res = {"hidden": [], "out": None}
    a = np.hstack([_f(s) for s in srcs])
    for l in range(n):
        mode = _mode(modes[l], pert)
        last = l + 1 == n
        em = None if last else D[l]
        if em is not None and "dropout_col" in pert and l == n - 2:
            em = em.copy()
            em[:, 0] = 1.0
        if "hidden_before_emul" in pert:
            em = None
        r = None
        if last and residual is not None:
            r = _f(residual)
            if "residual_last_tile" in pert:
                r = r.copy()
                r[_last_tile(V):] = 0
        z = _dense(a, Ws[l].T, mode, bias=bs[l], relu=not last or "relu_last" in pert, emul=em, residual=r, stats=stats)
        if last:
            res["out"] = z
        else:
            res["hidden"].append(z)
            a = z[0] if hidden is None else _f(hidden[l])
    return res


def head_fwd(out, weight, bias, x_in=None, pert=()):
    """The head in the MiniMLP epilogue: (out W^T + b, bound), (V, n_out), on the block output ``out`` the chain
    finished (fp32).  Each element is at most C fmaf roundings, two butterfly adds and the bias add, each within u of
    a partial sum bounded by |W||out| + |b|: 2 (C + 1) u (|W||out| + |b|).  ``x_in``: the residual, for the
    "head_before_residual" perturbation."""
    o, W = _f(out), _f(weight)
    b = np.zeros(W.shape[0]) if bias is None else _f(bias)
    C = W.shape[1]
    bound = 2 * (C + 1) * U * (np.abs(o) @ np.abs(W).T + np.abs(b)[None, :])
    if "head_before_residual" in pert:
        o = o - _f(x_in)
    if "head_drop_col" in pert:
        W = W.copy()
        W[:, C - 1] = 0
    if "head_wrong_bias" in pert:
        b = np.roll(b, -1)
    return o @ W.T + b[None, :], bound


# ------------------------------------------------------------------------------------------------
# heat kernel signature
# ------------------------------------------------------------------------------------------------
def compute_hks(evals, evecs, scales, pert=()):
    """dn_compute_hks: (gold, bound), both (V, S).  Each term e_k phi_k^2 carries expf's 2 ulp, the rounding of
    lambda s (|lambda s| u relative), that of phi^2 and an underflow's smallest denormal; the fmaf chain and the
    butterfly add ceil(K / 32) + 5 roundings of at most u of the element each."""
    lam, phi, s = _f(evals), _f(evecs), _f(scales).copy()
    K = phi.shape[1]
    if "scale_scaled" in pert:
        s[len(s) // 2] *= 1 + 1e-3
    ls = lam[:, None] * s[None, :]                      # (K, S)
    e = np.exp(-ls)
    p2 = phi * phi
    if "drop_eig" in pert:
        p2 = p2.copy()
        p2[:, K - 1] = 0
    out = p2 @ e
    eterm = p2 @ (e * (np.abs(ls) * U + 3 * U) + 2.0 ** -149)
    L = -(-K // 32) + 5
    return out, C_SAFE * L * U * out + eterm + K * 2.0 ** -149


# ------------------------------------------------------------------------------------------------
# routes
# ------------------------------------------------------------------------------------------------
def routes(engine, K, C, dims, nsrc=3, sm=132):
    """The forward route table: {stage: mode} for the diffusion at (K, C), the [P|Q] layer with and without rotations at
    C, and a MiniMLP over ``nsrc`` sources of width C with layer widths ``dims`` ("mlp/fused": one chain)."""
    r = {"diffusion/to_basis": to_basis_mode(engine, K, C, sm, PARTIAL_FLOATS),
         "diffusion/from_basis": layer_mode(engine, [K], K, C),
         "features/pq": layer_mode(engine, [C], C, 2 * C), "features/pq_norot": layer_mode(engine, [C], C, C)}
    modes, fused = _mlp_modes([C] * nsrc, dims, PASSES[engine])
    for l, m in enumerate(modes):
        r["mlp/l%d" % l] = m
    r["mlp/fused"] = fused
    return r


def mlp_on_tc(engine, C, dims, nsrc=3):
    """Whether every MiniMLP layer runs on tensor cores (one chain, or each layer's own plan)."""
    return "simt" not in _mlp_modes([C] * nsrc, dims, PASSES[engine])[0]
