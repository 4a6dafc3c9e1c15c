"""The backward entry points dn_learned_time_diffusion_bwd, dn_from_basis (with row_scale) and dn_mini_mlp_bwd restated
per engine, each result with a componentwise error bound that holds for any fp32 accumulation order.

TEST INFRASTRUCTURE ONLY (checker side, like ``dn_oracle_engines``); the product never imports it.

Where the kernels round (the forward's rounding points, ``dn_oracle_engines``, plus):

* ``atb`` (dn_capi.cu), the weight-gradient contraction out (+)= A^T B with A = dz, B = the layer input, runs the split-V
  to_basis kernel when both operands are contiguous, tc_to_basis_supported(I, J) holds and sm_count * I * J partials
  fit; A is its "basis" operand and B its "values" operand, both split by split_tf32_fast (hi = round-to-nearest TF32,
  lo = x - hi read truncated): ``_mm(A^T, B, packed=False)``.  Under bf16 it is single-pass TF32.  Otherwise the exact
  SIMT kernel.  The partials are summed by reduce_partials in order, the prefilled output added last (accumulate = 1).
* to_basis of dn_learned_time_diffusion_bwd: the same kernel with A = Phi, B = grad_out (no mass), or its 128-column
  slices for C = 256, or SIMT.  spectral_bwd forms dS = expf(-(lambda * max(t, 1e-8))) * G and the time gradient
  sum_k G (-lambda) e x_spec serially (over <= 4 partials, else over their reduction).
* run_chain on one layer (from_basis: A = Phi, W = dS or the values; the MiniMLP dX layers: A = dz, W = W_l read
  transposed): tc_chain_plan picks bf16 where the 16-wide K steps fit, TF32 (single-pass under bf16) where the 8-wide
  ones do, and SIMT otherwise.  A is split as an activation, W by the pack kernel (split_tf32: lo = cvt.rna(w - hi);
  bf16: round to nearest even).  Epilogue in rows_chain_kernel's order: emul (dropout mask), relu mask (m > 0 keeps),
  row_scale.
* layer 0 of dn_mini_mlp_bwd: one w_trans layer per source, reading W0's columns [off, off + width).

The bound.  A product of two rounded operands is exact in fp32 (TF32 x TF32, bf16 x bf16, fp32 x fp32 under fma), so
an element of a contraction with L sequential adds is off by at most L u sum_r |a_r b_r| (u = 2^-23 per add covers a
truncating accumulator), times C_SAFE.  L comes from the real split: rows per CTA (times the passes) plus the partials.
tc3x drops lo x lo: 2^-22 sum |a||b| more.  Each epilogue multiply or add and each stored sum costs one u of its
result.  An intermediate the kernel rounds again (dS, the deeper layers' dz) carries its own bound e_z: the kernel's
fp32 value lies in [z* - e_z, z* + e_z], the gold reads round(z*), and the kernel's rounded operand lies in
[round(z* - e_z), round(z* + e_z)] (rounding is monotone).  That spread is zero unless a rounding boundary falls inside
the band, and it enters downstream as |spread| x |other operand| (``flip`` counts those elements).

``perturb``: named structural errors for the sensitivity tests (PERTURBATIONS)."""
from __future__ import annotations

import numpy as np

from dn_oracle_engines import _mm, _plan, _to_basis_tc, bf16_rn, tf32_rna

__all__ = ["diffusion_bwd", "from_basis", "mini_mlp_bwd", "gradient_features_bwd", "routes", "atb_split",
           "PERTURBATIONS", "ENGINES"]

ENGINES = ("simt", "tc3x", "tc1x", "bf16")
PASSES = {"simt": None, "tc3x": "3x", "tc1x": "1x", "bf16": "bf16"}
U = 2.0 ** -23               # one fp32 operation, any rounding mode
C_SAFE = 2.0
KC = 16                      # to_basis rows per chunk
TILE = 128                   # rows_chain_kernel rows per tile (two consumer warpgroups)
PARTIAL_FLOATS = 16 << 20    # kPartialFloats
PERTURBATIONS = ("drop_last_partial", "drop_eig", "no_clamp", "relu_mask_last_tile", "dropout_col",
                 "row_scale_last_tile", "wrong_w0_block", "accumulate0", "1x_for_bf16", "bf16_for_1x", "1x_for_3x",
                 "drop_dxd", "drop_dq_a_im")


class Stats:
    """Elements of rounded intermediates, and how many of them have a rounding boundary inside their band."""

    def __init__(self):
        self.n, self.flip = 0, 0


def _mode(m, pert):
    if m == "bf16" and "1x_for_bf16" in pert:
        return "1x"
    if m == "1x" and "bf16_for_1x" in pert:
        return "bf16"
    if m == "3x" and "1x_for_3x" in pert:
        return "1x"
    return m


def _spread(z, r, e, mode, stats):
    """How far the operand the kernel reads can lie from the gold's rounding r of z when its fp32 value is in z +- e."""
    if e is None:
        return None
    if mode == "simt":
        return e
    if mode == "3x":        # hi + truncated lo: each within 2^-21 |x| of x
        return e + 2.0 ** -20 * (np.abs(z) + e)
    rnd = tf32_rna if mode == "1x" else bf16_rn
    s = np.maximum(rnd(z + e) - r, r - rnd(z - e))
    if stats is not None:
        stats.n += s.size
        stats.flip += int(np.count_nonzero(s))
    return s


def _contract(a, b, mode, L, ea=None, eb=None, b_packed=True, stats=None):
    """a (M, R) @ b (R, N) as ``mode`` rounds it, with L sequential adds per element: (gold, bound)."""
    if mode in ("1x", "bf16"):    # _mm's single-pass product, its rounded operands kept for the bound
        rnd = tf32_rna if mode == "1x" else bf16_rn
        ra, rb = rnd(a), rnd(b)
        val = ra @ rb
    else:
        val = _mm(a, b, mode, np.float64, packed=b_packed)
        ra, rb = a, b
    aa, ab = np.abs(ra), np.abs(rb)
    mag = aa @ ab
    bound = C_SAFE * L * U * mag
    if mode == "3x":
        bound += 2.0 ** -22 * mag
    da, db = _spread(a, ra, ea, mode, stats), _spread(b, rb, eb, mode, stats)
    if da is not None:
        bound += da @ ab
    if db is not None:
        bound += aa @ db
    if da is not None and db is not None:
        bound += da @ db
    return val, bound


# ------------------------------------------------------------------------------------------------
# routes (dn_capi.cu: atb, to_basis_partials, run_chain) and splits
# ------------------------------------------------------------------------------------------------
def layer_mode(engine, src_widths, K, N):
    """run_chain on one layer: the tensor-core mode tc_chain_plan picks, or "simt"."""
    p = PASSES[engine]
    return (_plan(list(src_widths), [(K, N, 0)], p) if p else None) or "simt"


def atb_mode(engine, I, J, sm, part_floats):
    p = PASSES[engine]
    if p and J <= 128 and _to_basis_tc(I, J) and sm * I * J <= part_floats:   # no column slices
        return "3x" if p == "3x" else "1x"
    return "simt"


def to_basis_mode(engine, K, C, sm, part_floats):
    p = PASSES[engine]
    if p and sm * K * C <= part_floats and _to_basis_tc(K, C):
        return "3x" if p == "3x" else "1x"
    return "simt"


def _plan_row_slices(V, tiles, slice_floats, ws_floats, rnd, sm):
    """plan_row_slices (dn_simt.cu) -> (P, rows per slice)"""
    P = max(1, min((V + 2047) // 2048, max(1, (4 * sm) // tiles)))
    while P * slice_floats > ws_floats and P > 1:
        P -= 1
    rps = -(-V // P)
    rps = max(rnd, -(-rps // rnd) * rnd)
    return max(1, -(-V // rps)), rps


def atb_split(mode, V, I, J, sm, part_floats):
    """(P, rows per partial) of a split-V A^T B: tc_to_basis_partial's CTA split, or the SIMT kernel's row slices."""
    if mode == "simt":
        return _plan_row_slices(V, -(-I // 64) * -(-J // 64), I * J, part_floats, 16, sm)
    chunks = -(-V // KC)
    grid = max(1, min(sm, chunks))
    cpc = max(1, -(-chunks // grid))
    return max(1, -(-chunks // cpc)), cpc * KC


def _split_v(A, B, mode, sm, part_floats, ea=None, pert=(), stats=None, split=None, tree=None):
    """sum_v A[v]^T B[v] as atb / to_basis_partials + reduce_partials compute it: (gold, bound).  ``split``: (P, rows
    per partial) of a planned mesh batch instead of the kernel's own split.  ``tree``: the partials are summed by
    ``tree`` slices, each serially, then pairwise (spectral_scale_kernel: 4, the pack kernel's spectral job: 8) instead
    of serially with the prefilled output added last."""
    V = A.shape[0]
    P, rps = split or atb_split(mode, V, A.shape[1], B.shape[1], sm, part_floats)
    if "drop_last_partial" in pert and P > 1:
        A = A.copy()
        A[(P - 1) * rps:] = 0
    red = P + 1 if tree is None else -(-P // tree) + int(np.log2(tree))
    L = (3 if mode == "3x" else 1) * rps + red
    return _contract(A.T, B, mode, L, ea=None if ea is None else ea.T, b_packed=False, stats=stats)


def _dense(a, W, mode, ea=None, eW=None, bias=None, relu=False, emul=None, relu_mask=None, row_scale=None,
           residual=None, stats=None):
    """one run_chain layer out = a @ W (W (K, N) as the layer reads it), epilogue in rows_chain_kernel's order: bias,
    relu, emul, relu mask, row_scale, residual (fmaf with res_scale = 1)."""
    L = (3 if mode == "3x" else 1) * a.shape[1]
    z, b = _contract(a, W, mode, L, ea=ea, eb=eW, stats=stats)
    if bias is not None:
        z = z + bias[None, :]
        b = b + U * np.abs(z)
    if relu:                     # non-expansive: the band carries over
        z = np.maximum(z, 0.0)
    if emul is not None:
        z = z * emul
        b = b * np.abs(emul) + U * np.abs(z)
    if relu_mask is not None:
        keep = relu_mask > 0
        z, b = np.where(keep, z, 0.0), np.where(keep, b, 0.0)
    if row_scale is not None:
        z = z * row_scale[:, None]
        b = b * np.abs(row_scale)[:, None] + U * np.abs(z)
    if residual is not None:
        z = z + residual
        b = b + U * np.abs(z)
    return z, b + U * np.abs(z)


def _last_tile(V):
    return V - V % TILE if V % TILE else V


# ------------------------------------------------------------------------------------------------
# the entry points
# ------------------------------------------------------------------------------------------------
def from_basis(values, basis, row_scale, engine, pert=(), eW=None, stats=None, mode=None):
    """dn_from_basis: out = row_scale * (basis @ values).  ``mode``: the chain's mode where from_basis is the first
    layer of a longer chain (the fused block's front); its own plan's when None."""
    K, C = values.shape
    mode = _mode(mode or layer_mode(engine, [K], K, C), pert)
    rs = None if row_scale is None else np.asarray(row_scale, np.float64)
    if rs is not None and "row_scale_last_tile" in pert:
        rs = rs.copy()
        rs[_last_tile(len(rs)):] = 1.0
    return _dense(np.asarray(basis, np.float64), np.asarray(values, np.float64), mode, eW=eW, row_scale=rs,
                  stats=stats)


def diffusion_bwd(grad_out, mass, evals, evecs, time, x_spec, engine, sm=132, part_floats=PARTIAL_FLOATS,
                  grad_time_init=None, pert=(), stats=None, split=None, cache=None):
    """dn_learned_time_diffusion_bwd: (grad_x, bound), (grad_time, bound).  ``time`` as passed (unclamped).  One mesh
    of dn_learned_time_diffusion_bwd_batched with ``split`` = its CTA plan's (P, rows per CTA).  ``cache``: a dict
    shared by the calls on the same inputs, so that engines whose to_basis rounds alike share its gold."""
    f = lambda v: np.asarray(v, np.float64)
    g, m, lam, phi, xs = f(grad_out), f(mass), f(evals), f(evecs), f(x_spec)
    V, C = g.shape
    K = phi.shape[1]
    tb = _mode(to_basis_mode(engine, K, C, sm, part_floats), pert)
    key = (tb, "drop_last_partial" in pert)
    if cache is not None and key in cache:
        G, eG = cache[key]
    else:
        G, eG = _split_v(phi, g, tb, sm, part_floats, split=split)
        if cache is not None:
            cache[key] = G, eG
    t32 = np.asarray(time, np.float32)
    t = f(t32 if "no_clamp" in pert else np.maximum(t32, np.float32(1e-8)))
    lt = lam[:, None] * t[None, :]
    e = np.exp(-lt)
    # expf is within 2 ulp, lambda * t rounded once (its relative error moves the exponent by |lambda t| u);
    # an underflow to a denormal or zero is off by at most the smallest denormal
    ee = e * (np.abs(lt) * U + 2 * U) + 2.0 ** -149
    if "drop_eig" in pert:
        e = e.copy()
        e[K - 1] = 0
    dS = e * G
    edS = np.abs(e) * eG + np.abs(G) * ee + U * np.abs(dS)
    terms = G * (-lam[:, None]) * e * xs
    gt0 = np.zeros(C) if grad_time_init is None else f(grad_time_init)
    gt = gt0 + terms.sum(0)
    egt = (np.abs(lam[:, None] * xs) * (np.abs(e) * eG + np.abs(G) * ee)).sum(0) \
        + C_SAFE * (K + 4) * U * np.abs(terms).sum(0) + U * np.abs(gt)
    gx, egx = from_basis(dS, phi, m, engine, pert=pert, eW=edS, stats=stats)
    return (gx, egx), (gt, egt)


def mini_mlp_bwd(grad_out, srcs, weights, hidden, drop_masks, engine, sm=132, grad_w_init=None, has_bias=None,
                 pert=(), stats=None, grad_b_init=0.0):
    """dn_mini_mlp_bwd.  weights[l] (dims[l + 1], dims[l]); hidden[l] the saved activation of layer l < n - 1 (its
    relu mask is hidden > 0); drop_masks[l] or None.  Returns {"src": [(g, bound)], "w": [...], "b": [... or None]}."""
    f = lambda v: None if v is None else np.asarray(v, np.float64)
    part = PARTIAL_FLOATS // 2
    n = len(weights)
    Ws = [f(w) for w in weights]
    H = [f(h) for h in hidden]
    D = [f(d) for d in drop_masks] if drop_masks is not None else [None] * (n - 1)
    widths = [s.shape[1] for s in srcs]
    dims = [sum(widths)] + [w.shape[0] for w in Ws]
    V = grad_out.shape[0]
    res = {"src": [None] * len(srcs), "w": [None] * n, "b": [None] * n}
    dz, edz = f(grad_out), None
    for l in range(n - 1, -1, -1):
        nout, nin = dims[l + 1], dims[l]
        init = np.zeros((nout, nin)) if grad_w_init is None or "accumulate0" in pert else f(grad_w_init[l])
        ins = [(H[l - 1], 0)] if l > 0 else [(f(s), o) for s, o in zip(srcs, np.cumsum([0] + widths[:-1]))]
        gw, ew = init.copy(), np.zeros((nout, nin))
        for x, off in ins:
            mode = _mode(atb_mode(engine, nout, x.shape[1], sm, part), pert)
            v, b = _split_v(dz, x, mode, sm, part, ea=edz, pert=pert, stats=stats)
            sl = slice(off, off + x.shape[1])
            gw[:, sl] += v
            ew[:, sl] = b + U * np.abs(gw[:, sl])
        res["w"][l] = (gw, ew)
        if has_bias is None or has_bias[l]:
            P, rps = _plan_row_slices(V, -(-nout // 32), nout, part, 1, sm)
            L = -(-rps // 8) + 8 + P + 1
            b0 = 0.0 if "accumulate0" in pert else grad_b_init
            gb = b0 + dz.sum(0)
            res["b"][l] = (gb, C_SAFE * L * U * np.abs(dz).sum(0) + (0 if edz is None else edz.sum(0)) + U * np.abs(gb))
        if l > 0:
            mode = _mode(layer_mode(engine, [nout], nout, nin), pert)
            mask = H[l - 1]
            if "relu_mask_last_tile" in pert:
                mask = mask.copy()
                mask[_last_tile(V):] = 1.0
            em = D[l - 1]
            if em is not None and "dropout_col" in pert and l == n - 1:
                em = em.copy()
                em[:, 0] = 1.0
            dz, edz = _dense(dz, Ws[l], mode, ea=edz, emul=em, relu_mask=mask, stats=stats)
        else:
            off = 0
            for q, w in enumerate(widths):
                o = 0 if ("wrong_w0_block" in pert and q == 1) else off
                mode = _mode(layer_mode(engine, [nout], nout, w), pert)
                res["src"][q] = _dense(dz, Ws[0][:, o:o + w], mode, ea=edz, stats=stats)
                off += w
    return res


def routes(engine, V, K, C, dims, sm=132):
    """The route table: {contraction: mode} for the diffusion backward at (V, K, C) and a MiniMLP backward over three
    sources of width C with layer widths ``dims`` (dims[0] = 3 C)."""
    r = {"diffusion/to_basis": to_basis_mode(engine, K, C, sm, PARTIAL_FLOATS),
         "diffusion/from_basis": layer_mode(engine, [K], K, C),
         "features/dx": layer_mode(engine, [C, C], 2 * C, C), "features/dx_norot": layer_mode(engine, [C], C, C),
         "features/atb": atb_mode(engine, C, C, sm, PARTIAL_FLOATS // 4)}
    part = PARTIAL_FLOATS // 2
    for l in range(len(dims) - 1):
        nout, nin = dims[l + 1], dims[l]
        ins = [nin] if l > 0 else [C, C, C]
        ms = sorted({atb_mode(engine, nout, w, sm, part) for w in ins})
        r["mlp/atb%d" % l] = ms[0] if len(ms) == 1 else "mixed:" + "/".join(ms)
        r["mlp/dx%d" % l] = layer_mode(engine, [nout], nout, nin) if l > 0 else layer_mode(engine, [nout], nout, C)
    return r


def gradient_features_bwd(gX, gY, grad_features, x_diffuse, pq, features, A_re, A_im, engine, sm=132,
                          grad_A_init=None, pert=(), stats=None):
    """dn_gradient_features_bwd.  gX, gY: scipy.sparse (V, V) on one pattern; pq = [P | Q] (P alone without rotations);
    A_im None without rotations.  Returns (grad_x, bound), (grad_A_re, bound), (grad_A_im, bound) or None.

    The gather (features_bwd_local) and its transpose run on SIMT in fp32: a row's gathered sums have 2 nnz + 2 adds,
    dd = dfeat (1 - f^2), U = dd x the gathered sums, and dxd / dP / dQ sum 2 nnz + 2 terms of a column.  grad_x is one
    run_chain layer over the sources (dP | dQ) with [A_re ; A_im] stacked along K and dxd its residual (fmaf); on SIMT
    (simt_layer) two passes, the second adding the first's stored output: 2 more roundings.  grad_A_re += dP^T xd and
    grad_A_im += dQ^T xd are atb over kPartialFloats / 4."""
    f = lambda v: np.asarray(v, np.float64)
    rot = A_im is not None
    d, xd, ft, pqv = f(grad_features), f(x_diffuse), f(features), f(pq)
    V, C = xd.shape
    Pm, Qm = pqv[:, :C], (pqv[:, C:2 * C] if rot else None)
    aX, aY = abs(gX), abs(gY)
    pat = (aX + aY).tocsr()
    Lr = C_SAFE * U * (2 * np.diff(pat.indptr) + 2)[:, None]
    Lc = C_SAFE * U * (2 * np.diff(pat.tocsc().indptr) + 2)[:, None]
    if rot:
        a_s = [gX @ Pm - gY @ Qm, gY @ Pm + gX @ Qm]
        m_s = [aX @ np.abs(Pm) + aY @ np.abs(Qm), aY @ np.abs(Pm) + aX @ np.abs(Qm)]
    else:
        a_s, m_s = [gX @ Pm, gY @ Pm], [aX @ np.abs(Pm), aY @ np.abs(Pm)]
    a_s += [gX @ xd, gY @ xd]
    m_s += [aX @ np.abs(xd), aY @ np.abs(xd)]
    dd = d * (1 - ft * ft)
    edd = C_SAFE * U * np.abs(d) * (ft * ft + 3 * np.abs(1 - ft * ft))
    Us = [dd * a for a in a_s]
    eUs = [np.abs(dd) * Lr * m + np.abs(a) * edd + U * np.abs(u) for a, m, u in zip(a_s, m_s, Us)]
    aU = [np.abs(u) for u in Us]
    gXt, gYt, aXt, aYt = gX.T.tocsr(), gY.T.tocsr(), aX.T.tocsr(), aY.T.tocsr()

    def tsum(i, j, sign):
        v = gXt @ Us[i] + sign * (gYt @ Us[j])
        e = Lc * (aXt @ aU[i] + aYt @ aU[j]) + aXt @ eUs[i] + aYt @ eUs[j]
        return v, e

    dxd, edxd = tsum(0, 1, 1)
    dP, edP = tsum(2, 3, 1)
    dQ, edQ = (gXt @ Us[3] - gYt @ Us[2], Lc * (aXt @ aU[3] + aYt @ aU[2]) + aXt @ eUs[3] + aYt @ eUs[2]) if rot \
        else (None, None)
    # grad_x = dxd + dP A_re (+ dQ A_im)
    if rot:
        mode = _mode(layer_mode(engine, [C, C], 2 * C, C), pert)
        a, ea, W = np.hstack([dP, dQ]), np.hstack([edP, edQ]), np.vstack([f(A_re), f(A_im)])
        if "drop_dq_a_im" in pert:
            W = W.copy()
            W[C:] = 0
    else:
        mode = _mode(layer_mode(engine, [C], C, C), pert)
        a, ea, W = dP, edP, f(A_re)
    z, b = _contract(a, W, mode, (3 if mode == "3x" else 1) * a.shape[1] + 2, ea=ea, stats=stats)
    if "drop_dxd" not in pert:
        z = z + dxd
        b = b + edxd
    gx = (z, b + U * np.abs(z))
    part = PARTIAL_FLOATS // 4
    out = [gx]
    for i, (dm, edm) in enumerate([(dP, edP)] + ([(dQ, edQ)] if rot else [])):
        init = np.zeros((C, C)) if grad_A_init is None or "accumulate0" in pert else f(grad_A_init[i])
        amode = _mode(atb_mode(engine, C, C, sm, part), pert)
        v, e = _split_v(dm, xd, amode, sm, part, ea=edm, pert=pert, stats=stats)
        g = init + v
        out.append((g, e + U * np.abs(g)))
    return out[0], out[1], (out[2] if rot else None)
