"""The fused inference block (block_fwd_impl behind dn_block_fwd, dn_block_fwd_ex and dn_block_fwd_batched) checked stage
by stage, element by element, on every engine, against the per-element golds and bounds of
oracle/dn_oracle_engines_fwd.py: |ours - gold| <= bound.

block_fwd_impl carves its intermediates from the caller's workspace (``regions``), and only S on the tensor-core front
(formed in the pack launch), the MiniMLP's hidden activations inside one chain and, with a head, the block output stay
on chip.  So each stage is checked on the fp32 values the block itself left for the next one, as the training entry
points are (tests/test_gpu_forward_engines.py): the workspace is filled with a NaN sentinel before the call, and the
split-V partials, S (where it is written), x_diffuse, [P|Q] and the features are read back from it.

* to_basis: the kernel's own partials summed in fp32 in the reducing kernel's order (``F.tree_sum``: 4 slices in
  spectral_scale_kernel, 8 in the pack kernel on the tensor-core front).  That emulation is pinned bitwise to
  dn_learned_time_diffusion_fwd's x_spec_out on the same inputs, then checked against the x_spec gold.
* x_diffuse on that sum; [P|Q] on the block's own x_diffuse, with the front's mode (``E.dispatch``); the features on
  the block's own x_diffuse and [P|Q].
* The MiniMLP output is bitwise dn_mini_mlp_fwd's on the block's own (x_in, x_diffuse, features); that call's hidden
  layers and output are checked per element.
* The head in the MiniMLP epilogue (dn_block_fwd_ex) against out W^T + b in fp64 on the block output the same call
  stored; with out = NULL it is bitwise the same.
* Mesh batches (dn_block_fwd_batched): each mesh's stages as above over its own partials, padding rows of x_diffuse
  exactly 0."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from test_gpu_backward_engines import BATCH_CASES, ENGINE_ID, Report, _dev, _nan_buf, _sm, _stream, lib  # noqa: F401
from test_gpu_forward import CASES, _block
from test_gpu_forward_engines import diffusion_fwd_inputs, feat_inputs, run_diffusion_fwd, run_mini_mlp_fwd

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle_engines as E  # noqa: E402  (checker only)
import dn_oracle_engines_bwd as B  # noqa: E402  (checker only)
import dn_oracle_engines_fwd as F  # noqa: E402  (checker only)

ENGINES = B.ENGINES
TC_ENGINES = ("tc3x", "tc1x", "bf16")
HEAD_N_OUT = (1, 5, 8)
SENTINEL = -1          # int32 view of the workspace fill (every byte 0xff: a NaN)

# the benchmark's shapes at V = 200 037 (393 x 509), C = 128 and 256 with rotations: (n, m, K, C, kw, hidden, variant)
BIG = {"v200037_c128": ((393, 509, 128, 128, {}, None, None), ("tc3x", "bf16")),
       "v200037_c256": ((393, 509, 128, 256, {}, None, None), ("tc3x", "bf16"))}


def regions(V, K, C, with_features, rot):
    """{name: (float offset, floats)} of the scratch block_fwd_impl (dn_capi.cu) carves from the front of its workspace
    with Bump::take, in its order: S (K x C), xd (V x C), with gradient features pq (V x npq) and feat (V x C), then the
    split-V partials (kPartialFloats); each take rounds up to 256 bytes.  "end": where the packed weights begin."""
    npq = 2 * C if rot else C
    sizes = [("S", K * C), ("xd", V * C)] + ([("pq", V * npq), ("feat", V * C)] if with_features else [])
    sizes.append(("partial", B.PARTIAL_FLOATS))
    r, off = {}, 0
    for name, n in sizes:
        r[name] = (off, n)
        off += (n * 4 + 255) // 256 * 64
    r["end"] = (off, 0)
    return r


def _nan_ws(lib, V, K, width, extra=0):
    """A workspace of the size ops.workspace gives the block, every byte 0xff."""
    n = lib.dn_workspace_bytes(V, K, width) + extra + 4096
    return torch.full(((n + 255) // 256 * 64,), SENTINEL, dtype=torch.int32, device="cuda")


class Block:
    """One block's inputs (fp32, host and device) and its parameters as block_fwd_impl reads them."""

    def __init__(self, x, mass, evals, evecs, gX, gY, params, wgf, gops, time=None):
        self.x, self.mass, self.evals, self.evecs = (np.ascontiguousarray(a, dtype=np.float32)
                                                     for a in (x, mass, evals, evecs))
        self.gX, self.gY, self.gops, self.wgf = gX, gY, gops, wgf
        self.V, self.C = self.x.shape
        self.K = self.evecs.shape[1]
        self.rot = wgf and "gradient_features.A.weight" not in params
        f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
        self.time = f32(params["diffusion.diffusion_time"] if time is None else time)
        if wgf:
            self.A_re = f32(params["gradient_features.A_re.weight" if self.rot else "gradient_features.A.weight"])
            self.A_im = f32(params["gradient_features.A_im.weight"]) if self.rot else None
        else:
            self.A_re = self.A_im = None
        ws, bs = E._mlp_weights(params)
        self.weights, self.biases = [f32(w) for w in ws], [f32(b) for b in bs]
        self.dims = [self.weights[0].shape[1]] + [w.shape[0] for w in self.weights]
        self.d = {k: _dev(getattr(self, k)) for k in ("x", "mass", "evals", "evecs")}
        self.d_w = [_dev(w) for w in self.weights]
        self.d_b = [_dev(b) for b in self.biases]
        self.d_are = _dev(self.A_re) if wgf else None
        self.d_aim = _dev(self.A_im) if self.rot else None

    def dispatch(self, engine):
        return E.dispatch(engine, self.K, self.C, self.dims, self.wgf, self.rot)

    def call(self, lib, engine, batch=None, head=None, store_out=True):
        """The block on a NaN-filled workspace: (out or None, head_out or None, workspace as float32, clamped time)."""
        from diffusion_net_b200 import _lib as L
        V, K, C = self.V, self.K, self.C
        extra = 0 if batch is None else batch.n_meshes * K * C * 8
        ws = _nan_ws(lib, V, K, max(C, max(self.dims[1:])), extra)
        t = _dev(self.time)
        # (the pointer arrays stay alive in locals until the call returns, as in ops.block_forward_raw)
        wp, bp = L.ptr_array([w.data_ptr() for w in self.d_w]), L.ptr_array([b.data_ptr() for b in self.d_b])
        dm = L.int_array(self.dims)
        prm = L.dn_block_params(t.data_ptr(), self.d_are.data_ptr() if self.wgf else None,
                                self.d_aim.data_ptr() if self.rot else None, int(self.wgf), int(self.rot),
                                len(self.weights), wp, bp, dm)
        out = _nan_buf(V, C) if store_out else None
        csr = ctypes.byref(self.gops.csr[0]) if self.wgf else None
        a = [self.d[k].data_ptr() for k in ("x", "mass", "evals", "evecs")]
        hout = hd = None
        if head is not None:
            hw, hb = head
            hout = _nan_buf(V, hw.shape[0])
            hd = L.dn_head(hw.data_ptr(), hb.data_ptr(), int(hw.shape[0]), hout.data_ptr(), int(hw.shape[0]))
        tail = (out.data_ptr() if store_out else None, ws.data_ptr(), ws.numel() * 4, ENGINE_ID[engine], _stream())
        if head is not None:
            rc = lib.dn_block_fwd_ex(*a, csr, ctypes.byref(prm), ctypes.byref(batch.desc) if batch else None,
                                     ctypes.byref(hd), V, K, C, *tail)
        elif batch is not None:
            rc = lib.dn_block_fwd_batched(*a, csr, ctypes.byref(prm), ctypes.byref(batch.desc), V, K, C, *tail)
        else:
            rc = lib.dn_block_fwd(*a, csr, ctypes.byref(prm), V, K, C, *tail)
        torch.cuda.synchronize()
        assert rc == 0, (engine, rc)
        return out, hout, ws.view(torch.float32), t


def _region(wsf, reg, name, shape=None):
    off, n = reg[name]
    r = wsf[off:off + n]
    return r if shape is None else r.view(*shape)


def check_carve(rep, wsf, reg, rows, engine, tc_front):
    """Fails loudly if ``regions`` drifted from block_fwd_impl: every row of xd, pq and feat below V finite, the
    alignment gaps still the sentinel, and S the sentinel where the front forms it in the pack launch."""
    bits = wsf.view(torch.int32)
    for name in ("xd", "pq", "feat"):
        if name not in reg:
            continue
        off, n = reg[name]
        for r0, r1, width in rows(name):
            if not bool(torch.isfinite(wsf[off + r0 * width:off + r1 * width]).all()):
                rep.misses.append("{} {}: rows below V are not finite (does regions() match block_fwd_impl?)".format(
                    engine, name))
    names = [k for k in reg if k != "end"]
    for name in names:
        off, n = reg[name]
        end = off + (n * 4 + 255) // 256 * 64
        if not bool((bits[off + n:end] == SENTINEL).all()):
            rep.misses.append("{} {}: the alignment gap after it was written".format(engine, name))
    if tc_front and not bool((_region(bits, reg, "S") == SENTINEL).all()):
        rep.misses.append("{}: S was written to the workspace on a tensor-core front".format(engine))


def tc_front(d, engine):
    return engine != "simt" and d["from_basis"] != "simt" and all(m != "simt" for m in d["pq"])


def spectral_checks(rep, blk, engine, wsf, reg, sm, t_after, label="", mesh=None):
    """x_spec on the block's own partials, the time clamp and, where it is written, S, for one mesh (``mesh``: its
    (first, end) partial and the plan's split in a batch).  Returns the x_spec sum and diffusion_fwd's golds."""
    K, C = blk.K, blk.C
    d = blk.dispatch(engine)
    front = tc_front(d, engine)
    part = _region(wsf, reg, "partial")
    if mesh is None:
        tb = B.to_basis_mode(engine, K, C, sm, B.PARTIAL_FLOATS)
        P = B.atb_split(tb, blk.V, K, C, sm, B.PARTIAL_FLOATS)[0]
        p0, p1, split, tree = 0, P, None, (8 if front else 4)
        if P * K * C < B.PARTIAL_FLOATS and not bool(torch.isnan(part[P * K * C])):
            rep.misses.append("{}: more than the modelled {} split-V partials were written".format(engine, P))
    else:
        (p0, p1), split = mesh
        tree = 8
    parts = part[p0 * K * C:p1 * K * C].view(p1 - p0, K, C).cpu().numpy()
    if not np.isfinite(parts).all():
        rep.misses.append("{}{}: a modelled split-V partial is not finite".format(engine, label))
    xs = F.tree_sum(parts, tree)
    gold = F.diffusion_fwd(blk.x, blk.mass, blk.evals, blk.evecs, blk.time, engine, x_spec_out=xs, sm=sm, split=split,
                           tree=tree, fb_mode=d["from_basis"])
    rep("{}{} x_spec".format(engine, label), xs, gold["x_spec"])
    if not np.array_equal(t_after.view(np.int32), gold["time"].view(np.int32)):
        rep.misses.append("{}: time after the call is not max(t, 1e-8f) bitwise".format(engine))
    if not front and mesh is None:
        lam, t = blk.evals.astype(np.float64), gold["time"].astype(np.float64)
        e, ee = F._heat(lam, t)
        x64 = xs.astype(np.float64)
        S = e * x64
        rep("{}{} S".format(engine, label), _region(wsf, reg, "S", (K, C)), (S, np.abs(x64) * ee + F.U * np.abs(S)))
    return xs, gold


@pytest.fixture(scope="module")
def dn():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import diffusion_net_b200 as d
    d._lib.load()
    return d


def single_block(dn, spec):
    run, x, host_ops, params, wgf = _block(dn, spec)
    mass, evals, evecs, gX, gY = host_ops
    gops = dn.ops.prepare_operators(*run.ops)
    if spec[6] == "permuted":
        gops.build_patches()
        assert gops._patches, "the permuted mesh did not get patches"
    gX32 = gX.astype(np.float32).astype(np.float64)
    gY32 = gY.astype(np.float32).astype(np.float64)
    return Block(x, mass, evals, evecs, gX32, gY32, params, wgf, gops)


def pin_x_spec(rep, lib, blk, engine, parts_fn):
    """tree_sum over the partials of dn_learned_time_diffusion_fwd (spectral_scale's 4 slices) is its x_spec_out."""
    rc, _, xs_ref, _ = run_diffusion_fwd(lib, engine, blk.x, blk.mass, blk.evals, blk.evecs, blk.time)
    assert rc == 0, (engine, rc)
    want = xs_ref.cpu().numpy()
    got = F.tree_sum(parts_fn(), 4)
    if not np.array_equal(got.view(np.int32), want.view(np.int32)):
        rep.misses.append("{}: the 4-slice tree sum of the block's partials is not dn_learned_time_diffusion_fwd's "
                          "x_spec_out bitwise ({} of {} differ)".format(engine, int((got != want).sum()), got.size))


def stage_checks(rep, lib, blk, engine, sm, heads=True):
    V, K, C = blk.V, blk.K, blk.C
    d = blk.dispatch(engine)
    reg = regions(V, K, C, blk.wgf, blk.rot)
    out, _, wsf, t = blk.call(lib, engine)
    front = tc_front(d, engine)
    npq = 2 * C if blk.rot else C
    check_carve(rep, wsf, reg, lambda name: [(0, V, npq if name == "pq" else C)], engine, front)
    _, gold = spectral_checks(rep, blk, engine, wsf, reg, sm, t.cpu().numpy())
    P = B.atb_split(B.to_basis_mode(engine, K, C, sm, B.PARTIAL_FLOATS), V, K, C, sm, B.PARTIAL_FLOATS)[0]
    pin_x_spec(rep, lib, blk, engine,
               lambda: _region(wsf, reg, "partial")[:P * K * C].view(P, K, C).cpu().numpy())
    xd = _region(wsf, reg, "xd", (V, C))
    rep(engine + " x_diffuse", xd, gold["x_diffuse"])
    srcs = [blk.x, xd.cpu().numpy()]
    if blk.wgf:
        pq = _region(wsf, reg, "pq", (V, npq))
        feat = _region(wsf, reg, "feat", (V, C))
        g = F.features_fwd(blk.gX, blk.gY, srcs[1], blk.A_re, blk.A_im, engine, pq_out=pq.cpu().numpy(),
                           mode=d["pq"][0])
        rep(engine + " pq", pq, g["pq"])
        rep(engine + " features", feat, g["features"])
        srcs.append(feat.cpu().numpy())
    mlp_checks(rep, lib, blk, engine, srcs, out, slice(0, V))
    rep.nan_rows(engine + " out", out, V)
    if heads and engine != "simt" and d["mlp_fused"]:
        for n_out in HEAD_N_OUT:
            head_checks(rep, lib, blk, engine, n_out, [(0, V)])


def mlp_checks(rep, lib, blk, engine, srcs, out, rows):
    """out is bitwise dn_mini_mlp_fwd on the block's own sources; that call checked per element on ``rows`` (a batch's
    padding rows read whatever the gather left there, so they are not compared)."""
    rc, hid, out2 = run_mini_mlp_fwd(lib, engine, srcs, blk.weights, blk.biases, None, blk.x)
    assert rc == 0, (engine, rc)
    V = blk.V
    sl = lambda a: a[rows]
    a, b = sl(out[:V].cpu().numpy()), sl(out2[:V].cpu().numpy())
    if not np.array_equal(a.view(np.int32), b.view(np.int32)):
        rep.misses.append("{}: the block output is not dn_mini_mlp_fwd's on its own sources bitwise ({} elements "
                          "differ)".format(engine, int((a != b).sum())))
    hid_h = [h[:V].cpu().numpy() for h in hid]
    g = F.mini_mlp_fwd([sl(s) for s in srcs], blk.weights, blk.biases, None, sl(blk.x), engine,
                       hidden=[sl(h) for h in hid_h])
    for l, h in enumerate(hid_h):
        rep("{} hidden{}".format(engine, l), sl(h), g["hidden"][l])
    rep(engine + " out", b, g["out"])


def head_checks(rep, lib, blk, engine, n_out, meshes, batch=None):
    rs = np.random.RandomState(100 + n_out)
    W = np.asarray(rs.randn(n_out, blk.C) / np.sqrt(blk.C), np.float32)
    b = np.asarray(rs.randn(n_out), np.float32)
    hw, hb = _dev(W), _dev(b)
    out, hout, _, _ = blk.call(lib, engine, batch=batch, head=(hw, hb))
    _, hout0, _, _ = blk.call(lib, engine, batch=batch, head=(hw, hb), store_out=False)
    V = blk.V
    lbl = "{} head{}".format(engine, n_out)
    for r0, r1 in meshes:
        rep(lbl, hout[r0:r1], F.head_fwd(out[r0:r1].cpu().numpy(), W, b))
    rep.nan_rows(lbl, hout, V)
    rep.nan_rows(lbl + " out", out, V)
    if not torch.equal(hout.view(torch.int32), hout0.view(torch.int32)):
        rep.misses.append("{}: head_out with out = NULL differs from head_out with out stored".format(lbl))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_block_stages(dn, lib, name):
    blk = single_block(dn, CASES[name])
    sm = _sm(lib)
    rep = Report("block_stages/" + name)
    for engine in ENGINES:
        stage_checks(rep, lib, blk, engine, sm)
    rep.done()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BIG))
def test_block_stages_200k(dn, lib, name):
    """The benchmark's block shapes at V = 200 037 on the engines the benchmark runs; the head at n_out = 8 where the
    MiniMLP is one chain (C = 128)."""
    spec, engines = BIG[name]
    blk = single_block(dn, spec)
    sm = _sm(lib)
    rep = Report("block_stages/" + name)
    for engine in engines:
        stage_checks(rep, lib, blk, engine, sm, heads=False)
        if blk.dispatch(engine)["mlp_fused"]:
            head_checks(rep, lib, blk, engine, 8, [(0, blk.V)])
    rep.done()


# ---- mesh batches ----------------------------------------------------------------------------------------------------
def batch_block(dn, rows, K, C):
    """A ragged MeshBatch of the training tests' diffusion inputs with a random gradient pattern per mesh (the diagonal
    and 6 random neighbours per row), and one block's parameters."""
    import scipy.sparse as sp
    meshes, items, grads = [], [], []
    for i, v in enumerate(rows):
        mi = diffusion_fwd_inputs(v, K, C, seed=31 + i)
        rs = np.random.RandomState(200 + i)
        r = np.repeat(np.arange(v), 7)
        c = np.concatenate([np.arange(v)[:, None], rs.randint(0, v, (v, 6))], axis=1).ravel()
        gX, gY, a = feat_inputs(r, c, v, C, True, seed=300 + i)
        idx = torch.from_numpy(np.stack([a["rows"], a["cols"]]))
        coo = lambda vals: torch.sparse_coo_tensor(idx, torch.from_numpy(vals), (v, v)).coalesce().cuda()
        meshes.append(mi)
        grads.append((gX, gY))
        items.append(dict(mass=_dev(mi[1]), evals=_dev(mi[2]), evecs=_dev(mi[3]), gradX=coo(a["gx"]),
                          gradY=coo(a["gy"])))
    mb = dn.MeshBatch(items)
    params = {k: v.numpy() for k, v in dn.synthetic.block_weights(C, seed=7).items()}
    x = mb.pack([torch.from_numpy(mi[0]).cuda() for mi in meshes]).cpu().numpy()
    blk = Block(x, mb.mass.cpu().numpy(), mb.evals.cpu().numpy(), mb.evecs.cpu().numpy(), sp.block_diag([g[0] for g in grads]),
                sp.block_diag([g[1] for g in grads]), params, True, mb.gops, time=meshes[0][4])
    blk.d["evals"], blk.d["mass"], blk.d["evecs"] = mb.evals, mb.mass, mb.evecs
    return mb, meshes, grads, blk


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(BATCH_CASES))
def test_block_stages_batched(dn, lib, case):
    """dn_block_fwd_batched and dn_block_fwd_ex with a head over a ragged batch: each mesh's stages on its own partials
    (the pack kernel's 8-slice tree over the mesh's CTAs), x_diffuse's padding rows exactly 0."""
    rows, K, C = BATCH_CASES[case]
    sm = _sm(lib)
    mb, meshes, grads, blk = batch_block(dn, rows, K, C)
    V = mb.V
    tb = mb._tb_rows.cpu().numpy().reshape(-1, 2)
    cb = mb._cta_begin.cpu().numpy()
    split = (len(tb), int((tb[:, 1] - tb[:, 0]).max()))
    rb = list(mb.row_begin)
    reg = regions(V, K, C, True, True)
    rep = Report("block_stages_batched/" + case)
    for engine in TC_ENGINES:
        d = blk.dispatch(engine)
        out, _, wsf, t = blk.call(lib, engine, batch=mb)
        spans = lambda name: [(rb[b], rb[b] + n, 2 * C if name == "pq" else C) for b, n in enumerate(rows)]
        check_carve(rep, wsf, reg, spans, engine, True)
        xd = _region(wsf, reg, "xd", (V, C))
        pq = _region(wsf, reg, "pq", (V, 2 * C))
        feat = _region(wsf, reg, "feat", (V, C))
        # the batched training forward's x_spec_out is the same 8-slice sum of the same partials
        xs_ref = torch.full((len(rows) * K, C), float("nan"), device="cuda")
        xd_ref = torch.full((V, C), float("nan"), device="cuda")
        ws2 = _nan_ws(lib, V, K, 2 * C, len(rows) * K * C * 8)
        rc = lib.dn_learned_time_diffusion_fwd_batched(blk.d["x"].data_ptr(), mb.mass.data_ptr(), mb.evals.data_ptr(),
                                                       mb.evecs.data_ptr(), _dev(blk.time).data_ptr(),
                                                       ctypes.byref(mb.desc), V, K, C, xd_ref.data_ptr(),
                                                       xs_ref.data_ptr(), ws2.data_ptr(), ws2.numel() * 4,
                                                       ENGINE_ID[engine], _stream())
        torch.cuda.synchronize()
        assert rc == 0, (engine, rc)
        xs_ref = xs_ref.cpu().numpy()
        for b, n in enumerate(rows):
            r0, r1 = rb[b], rb[b] + n
            mesh_blk = _MeshView(blk, meshes[b], grads[b])
            xs, gold = spectral_checks(rep, mesh_blk, engine, wsf, reg, sm, t.cpu().numpy(),
                                       label=" mesh {}".format(b), mesh=((cb[b], cb[b + 1]), split))
            want = xs_ref[b * K:(b + 1) * K]
            if not np.array_equal(xs.view(np.int32), want.view(np.int32)):
                rep.misses.append("{} mesh {}: the 8-slice sum of the block's partials is not "
                                  "dn_learned_time_diffusion_fwd_batched's x_spec_out bitwise".format(engine, b))
            rep("{} x_diffuse mesh {}".format(engine, b), xd[r0:r1], gold["x_diffuse"])
            if not bool((xd[r1:rb[b + 1]] == 0).all()):
                rep.misses.append("{} mesh {}: padding rows of x_diffuse are not exactly 0".format(engine, b))
            g = F.features_fwd(grads[b][0], grads[b][1], xd[r0:r1].cpu().numpy(), blk.A_re, blk.A_im, engine,
                               pq_out=pq[r0:r1].cpu().numpy(), mode=d["pq"][0])
            rep("{} pq mesh {}".format(engine, b), pq[r0:r1], g["pq"])
            rep("{} features mesh {}".format(engine, b), feat[r0:r1], g["features"])
        mask = np.zeros(V, bool)
        for b, n in enumerate(rows):
            mask[rb[b]:rb[b] + n] = True
        mlp_checks(rep, lib, blk, engine, [blk.x, xd.cpu().numpy(), feat.cpu().numpy()], out, mask)
        rep.nan_rows(engine + " out", out, V)
        for n_out in HEAD_N_OUT:
            head_checks(rep, lib, blk, engine, n_out, [(rb[b], rb[b] + n) for b, n in enumerate(rows)], batch=mb)
    rep.done()


class _MeshView:
    """One mesh of a batch block, as spectral_checks reads it."""

    def __init__(self, blk, mi, grads):
        self.x, self.mass, self.evals, self.evecs = mi[0], mi[1], mi[2], mi[3]
        self.time, self.K, self.C, self.V = blk.time, blk.K, blk.C, mi[0].shape[0]
        self.dispatch = blk.dispatch
