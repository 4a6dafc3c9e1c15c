"""The fused classification head (ops.linear_nll, DiffusionNet.forward_nll / forward_batch_nll) against fp64 torch.

Gold: ``log_softmax`` + ``nll_loss(reduction='none')`` and autograd in float64 (on the CPU; the two largest cases
evaluate the same float64 expressions on the GPU to keep the suite's run time down).

Bounds, componentwise, from the unit roundoff and the contraction lengths.  Each engine rounds the operands of every
tensor-core product: u_p = 2^-22 for tc3x (the dropped low x low term), 2^-11 for tc1x (TF32), 2^-8 for bf16; sums
are fp32 (u = 2^-24).  A contraction of length L of terms a_i b_i is then off by at most (2 u_p + L u) sum |a_i b_i|:
  logits   E[r, n] = (2 u_p + (C + 1) u) (|X| |W|^T + |b|)[r, n],  e_r = max_n E[r, n]
  lse      e_r + (n_class + 8) u + u |lse|              (the fp32 sum of exponentials and its log)
  nll      2 e_r + (n_class + 8) u + 2 u (|lse| + |z_label|)
  dZ       D = |g| P (exp(2 e_r + (n_class + 12) u) - 1)  (P the fp64 softmax)
  dX       D |W| + (2 u_p + (n_class + 1) u) (|dZ| + D) |W|
  dW, db   D^T |X| + (2 u_p + (R + 1) u) (|dZ| + D)^T |X|,  and the same with |X| -> 1 for db
all times a safety factor 2.  argmax must equal the fp64 argmax wherever the fp64 top-two gap exceeds 4 e_r."""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle_torch as T  # noqa: E402  (checker only)

pytestmark = pytest.mark.gpu

D = torch.float64
U = 2.0 ** -24
U_PROD = {"tc3x": 2.0 ** -22, "tc1x": 2.0 ** -11, "bf16": 2.0 ** -8}
TC_ENGINES = ["tc3x", "tc1x", "bf16"]
SAFETY = 2.0

# (R, C, n_class): every n_class, C and R of the issue's grid, each crossed with the others' edge values
CASES = sorted(set(
    [(129, 64, n) for n in (1, 2, 8, 15, 16, 17, 127, 128, 129, 260)]
    + [(129, c, 17) for c in (16, 48, 64, 128, 256)] + [(127, c, 260) for c in (16, 48, 128, 256)]
    + [(r, 48, 129) for r in (1, 127, 128, 129, 6890)] + [(1, 256, 6890), (300, 16, 6890)]))
BIG = [(6890, 256, 6890), (200000, 128, 260)]


@pytest.fixture(scope="module")
def dn():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import diffusion_net_b200 as dn_
    yield dn_
    dn_.set_engine("tc3x")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _inputs(R, C, n, seed=0, scale=1.0, ignore_every=0):
    g = _gen(seed)
    x = torch.randn(R, C, generator=g)
    w = torch.randn(n, C, generator=g) / C ** 0.5 * scale
    b = torch.randn(n, generator=g) * 0.1 * scale
    lab = torch.randint(0, n, (R,), generator=g)
    if ignore_every:
        lab[::ignore_every] = -100
    gr = torch.rand(R, generator=g) + 0.5
    return x, w, b, lab, gr


def _gold(x, w, b, lab, gr, ignore_index=-100, device="cpu"):
    """fp64 nll, argmax, gradients and the ingredients of the bounds."""
    x64, w64, b64 = (t.to(device, D).requires_grad_(True) for t in (x, w, b))
    lab_d = lab.to(device)
    z = x64 @ w64.t() + b64
    logp = torch.log_softmax(z, dim=-1)
    nll = F.nll_loss(logp, lab_d, reduction='none', ignore_index=ignore_index)
    (nll * gr.to(device, D)).sum().backward()
    with torch.no_grad():
        P = logp.exp()
        keep = (lab_d != ignore_index).to(D)
        onehot = torch.zeros_like(P)
        ok = lab_d != ignore_index
        onehot[ok] = F.one_hot(lab_d[ok], P.shape[1]).to(D)
        dz = (gr.to(device, D) * keep)[:, None] * (P - onehot)
        ax = (x64.abs() @ w64.abs().t() + b64.abs()).max(dim=1).values
        top = torch.topk(z, min(2, z.shape[1]), dim=1).values
        gap = top[:, 0] - top[:, 1] if z.shape[1] > 1 else torch.full_like(top[:, 0], float("inf"))
        lse = torch.logsumexp(z, dim=1)
        zl = torch.where(ok, z.gather(1, lab_d.clamp(0, z.shape[1] - 1)[:, None])[:, 0], torch.zeros_like(lse))
    return dict(nll=nll.detach(), argmax=z.argmax(dim=1), gx=x64.grad, gw=w64.grad, gb=b64.grad, P=P, dz=dz, ax=ax,
                gap=gap, lse=lse, zl=zl, x=x64.detach(), w=w64.detach(), gr=gr.to(device, D) * keep)


def _check(engine, G, nll, pred, gx, gw, gb, what):
    up = U_PROD[engine]
    R, C = G["x"].shape
    n = G["w"].shape[0]
    dev = G["x"].device
    e = (2 * up + (C + 1) * U) * G["ax"]
    b_nll = SAFETY * (2 * e + (n + 8) * U + 2 * U * (G["lse"].abs() + G["zl"].abs()))
    err = (nll.to(dev, D) - G["nll"]).abs()
    assert bool((err <= b_nll).all()), "{} nll: worst err/bound {:.3g}".format(what, float((err / b_nll).max()))
    sure = G["gap"] > 4 * e
    assert bool((pred.to(dev)[sure] == G["argmax"][sure]).all()), "{} argmax".format(what)
    Dm = G["gr"][:, None] * G["P"] * torch.expm1(2 * e + (n + 12) * U)[:, None]
    A = G["dz"].abs() + Dm
    b_gx = SAFETY * (Dm @ G["w"].abs() + (2 * up + (n + 1) * U) * (A @ G["w"].abs()))
    b_gw = SAFETY * (Dm.t() @ G["x"].abs() + (2 * up + (R + 1) * U) * (A.t() @ G["x"].abs()))
    b_gb = SAFETY * (Dm.sum(0) + (2 * up + (R + 1) * U) * A.sum(0))
    for name, ours, gold, bound in (("grad_x", gx, G["gx"], b_gx), ("grad_w", gw, G["gw"], b_gw),
                                    ("grad_b", gb, G["gb"], b_gb)):
        err = (ours.to(dev, D) - gold).abs()
        bound = bound + 1e-30
        assert bool((err <= bound).all()), "{} {}: worst err/bound {:.3g}".format(what, name,
                                                                               float((err / bound).max()))


def _run(dn, x, w, b, lab, gr, ignore_index=-100):
    xc, wc, bc = (t.cuda().requires_grad_(True) for t in (x, w, b))
    nll, pred = dn.ops.linear_nll(xc, wc, bc, lab.cuda(), ignore_index)
    (nll * gr.cuda()).sum().backward()
    torch.cuda.synchronize()
    return nll.detach(), pred, xc.grad, wc.grad, bc.grad


_GOLD = {}


def _gold_cached(key, *args, device="cpu"):
    if key not in _GOLD:
        _GOLD.clear()
        _GOLD[key] = _gold(*args, device=device)
    return _GOLD[key]


# ---- 1. the op against fp64 ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=lambda c: "R{}_C{}_n{}".format(*c))
@pytest.mark.parametrize("engine", TC_ENGINES)
def test_linear_nll_vs_fp64(dn, case, engine):
    dn.set_engine(engine)
    R, C, n = case
    args = _inputs(R, C, n, seed=R + C + n, ignore_every=7 if R > 7 else 0)
    G = _gold_cached(case, *args)
    _check(engine, G, *_run(dn, *args), "{} {}".format(engine, case))


@pytest.mark.parametrize("case", BIG, ids=lambda c: "R{}_C{}_n{}".format(*c))
def test_linear_nll_vs_fp64_dataset_scale(dn, case):
    """The sampling_invariance head (6890 vertices and classes, C 256) and 200k rows of the 260-class head, tc3x."""
    dn.set_engine("tc3x")
    R, C, n = case
    args = _inputs(R, C, n, seed=3)
    G = _gold(*args, device="cuda")
    _check("tc3x", G, *_run(dn, *args), "tc3x {}".format(case))


@pytest.mark.parametrize("engine", TC_ENGINES)
def test_linear_nll_large_logits(dn, engine):
    """Logits scaled to about +-1e4: the online log-sum-exp must rescale, never overflow."""
    dn.set_engine(engine)
    args = _inputs(300, 64, 300, seed=11, scale=3e3)
    G = _gold(*args)
    assert float(G["ax"].max()) > 1e4
    out = _run(dn, *args)
    assert torch.isfinite(out[0]).all()
    _check(engine, G, *out, "{} large".format(engine))


# ---- 2. edge semantics ---------------------------------------------------------------------------------------------
def test_ignore_index_rows_and_all_ignored(dn):
    dn.set_engine("tc3x")
    x, w, b, lab, gr = _inputs(200, 32, 10, seed=5)
    lab[::3] = 7 - 100            # a custom ignore_index
    nll, pred, gx, gw, gb = _run(dn, x, w, b, lab, gr, ignore_index=-93)
    ign = (lab == -93).cuda()
    assert bool((nll[ign] == 0).all()) and bool((gx[ign] == 0).all())
    G = _gold(x, w, b, lab, gr, ignore_index=-93)
    _check("tc3x", G, nll, pred, gx, gw, gb, "ignore")
    # every row ignored: the mean is torch's (0 / 0 = nan) and every gradient is 0
    lab_all = torch.full((200,), -100, dtype=torch.int64)
    xc, wc, bc = (t.cuda().requires_grad_(True) for t in (x, w, b))
    nll, _ = dn.ops.linear_nll(xc, wc, bc, lab_all.cuda())
    loss = nll.sum() / (lab_all.cuda() != -100).sum()
    ref = F.nll_loss(torch.log_softmax(x.to(D) @ w.to(D).t() + b.to(D), -1), lab_all)
    assert torch.isnan(loss).item() and torch.isnan(ref).item()
    nll.sum().backward()
    assert not xc.grad.any() and not wc.grad.any() and not bc.grad.any()


def test_element_csr_built_once_per_element_array(dn):
    _, faces = dn.synthetic.torus_mesh(9, 11, seed=1)
    faces = faces.cuda()
    V = int(faces.max()) + 1
    a = dn.ops.cached_element_csr(faces, V)
    assert dn.ops.cached_element_csr(faces, V) is a
    rowptr, ent = a
    counts = torch.bincount(faces.reshape(-1), minlength=V)
    assert torch.equal(rowptr[1:] - rowptr[:-1], counts.to(torch.int32))
    x = torch.randn(V, 16, device="cuda", requires_grad=True)
    y = dn.ops.element_mean(x, faces)
    assert torch.allclose(y, x[faces].mean(dim=1), rtol=1e-6, atol=1e-6)
    g = torch.randn_like(y)
    y.backward(g)
    x2 = x.detach().clone().requires_grad_(True)
    x2[faces].mean(dim=1).backward(g)
    assert torch.allclose(x.grad, x2.grad, rtol=1e-6, atol=1e-6)


def test_out_of_range_label_and_nan_row(dn):
    """A label outside [0, n_class) gives a NaN row and NaN gradients, a NaN feature row a NaN row; no device fault."""
    dn.set_engine("tc3x")
    x, w, b, lab, gr = _inputs(300, 48, 20, seed=6)
    base = _run(dn, x, w, b, lab, gr)
    lab2 = lab.clone()
    lab2[17] = 20
    lab2[40] = -5
    nll, pred, gx, gw, gb = _run(dn, x, w, b, lab2, gr)
    bad = torch.zeros(300, dtype=torch.bool, device="cuda")
    bad[17] = bad[40] = True
    assert bool(torch.isnan(nll[bad]).all()) and torch.equal(nll[~bad], base[0][~bad])
    assert bool(torch.isnan(gx[bad]).all()) and torch.isnan(gw).any() and torch.isnan(gb).any()
    assert torch.equal(gx[~bad], base[2][~bad])
    x3 = x.clone()
    x3[5, 3] = float("nan")
    nll, pred, gx, gw, gb = _run(dn, x3, w, b, lab, gr)
    assert torch.isnan(nll[5]).item()
    keep = torch.ones(300, dtype=torch.bool, device="cuda")
    keep[5] = False
    assert torch.equal(nll[keep], base[0][keep]) and torch.equal(pred[keep], base[1][keep])
    torch.cuda.synchronize()


# ---- 3. determinism, 4. launch counts and the tensor-core route ---------------------------------------------------
def test_bitwise_deterministic_and_launch_counts(dn):
    dn.set_engine("tc3x")
    lib = dn._lib.load()
    counts = set()
    for (R, C, n) in [(129, 64, 8), (6890, 128, 260), (1000, 256, 6890)]:
        args = _inputs(R, C, n, seed=9)
        runs = []
        for _ in range(2):
            c0 = lib.dn_kernel_launch_count()
            runs.append(_run(dn, *args))
            counts.add(lib.dn_kernel_launch_count() - c0)
        for a, b_ in zip(*runs):
            assert torch.equal(a, b_)
    assert counts == {4}, counts        # 1 forward + 3 backward, whatever R and n_class are


def _strict_report():
    import diffusion_net_b200 as dn_
    dn_.set_engine("tc3x")
    res = {}
    for case in CASES + [(6890, 256, 6890)]:
        args = _inputs(*case, seed=1)
        try:
            _run(dn_, *args)
            res["R{}_C{}_n{}".format(*case)] = "ok"
        except RuntimeError as e:
            res["R{}_C{}_n{}".format(*case)] = str(e)
    print(json.dumps(res))


def test_every_case_on_tensor_cores_under_strict_tc(dn):
    env = dict(os.environ, DN_STRICT_TC="1")
    code = "import sys; sys.path.insert(0, {!r}); sys.path.insert(0, {!r}); import test_gpu_linear_nll as t; " \
           "t._strict_report()".format(ROOT, os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert all(v == "ok" for v in res.values()), res


# ---- 5. net level ---------------------------------------------------------------------------------------------------
def _net(dn, C, K, C_out, outputs_at, seed=0):
    torch.manual_seed(seed)
    net = dn.DiffusionNet(C_in=16, C_out=C_out, C_width=C, N_block=2, dropout=False, outputs_at=outputs_at,
                          last_activation=lambda x: torch.nn.functional.log_softmax(x, dim=-1)).cuda().train()
    with torch.no_grad():
        for n_, p_ in net.named_parameters():
            if n_.endswith("diffusion_time"):
                p_.uniform_(1e-3, 0.3)
    return net


def _edges(faces):
    e = torch.cat([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]], 0)
    return torch.unique(torch.sort(e, dim=1).values, dim=0)


@pytest.mark.parametrize("outputs_at", ["vertices", "faces", "edges"])
def test_forward_nll_vs_fp64(dn, outputs_at):
    dn.set_engine("tc3x")
    n, m, K, C, C_out = 20, 24, 32, 64, 12
    mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=2, device="cuda")
    _, faces = dn.synthetic.torus_mesh(n, m, seed=2)
    faces = faces.cuda()
    edges = _edges(faces)
    net = _net(dn, C, K, C_out, outputs_at)
    V = mass.shape[0]
    x = torch.randn(V, 16, generator=_gen(4)).cuda()
    rows = {"vertices": V, "faces": faces.shape[0], "edges": edges.shape[0]}[outputs_at]
    lab = torch.randint(0, C_out, (rows,), generator=_gen(5))
    lab[::9] = -100
    lab = lab.cuda()
    kw = dict(L=L, evals=evals, evecs=evecs, gradX=gX, gradY=gY, edges=edges, faces=faces)
    loss, pred = net.forward_nll(x, mass, labels=lab, **kw)
    loss.backward()
    grads = {k: p_.grad.clone() for k, p_ in net.named_parameters()}
    with torch.no_grad():
        logits = net(x, mass, **kw)              # log_softmax of the logits: same argmax
    # fp64 oracle composition
    prm = {k: v.detach().cpu().to(D).requires_grad_(True) for k, v in net.state_dict().items()}
    m64, e64, v64 = (t.cpu().to(D).unsqueeze(0) for t in (mass, evals, evecs))
    h = torch.addmm(prm["first_lin.bias"], x.cpu().to(D), prm["first_lin.weight"].t()).unsqueeze(0)
    for b in range(2):
        bp = {k[len("block_%d." % b):]: v for k, v in prm.items() if k.startswith("block_%d." % b)}
        h = T.block_forward(h, m64, e64, v64, [gX.cpu().to(D)], [gY.cpu().to(D)], bp)
    z = torch.addmm(prm["last_lin.bias"], h[0], prm["last_lin.weight"].t())
    if outputs_at != "vertices":
        el = (faces if outputs_at == "faces" else edges).cpu()
        z = z[el].mean(dim=1)
    gold = F.nll_loss(torch.log_softmax(z, -1), lab.cpu(), ignore_index=-100)
    gold.backward()
    # test_gpu_backward.py's fp32 bounds: 1e-5 on outputs, 5e-5 on parameter gradients (relative to the largest)
    assert abs(loss.item() - gold.item()) <= 1e-5 * abs(gold.item())
    for k, p_ in prm.items():
        if k not in grads:
            continue
        err = (grads[k].cpu().to(D) - p_.grad).abs().max().item()
        assert err <= 5e-5 * p_.grad.abs().max().item() + 1e-12, (k, err)
    top = torch.topk(z.detach(), 2, dim=1).values
    sure = (top[:, 0] - top[:, 1] > 1e-4).cuda()
    assert torch.equal(pred[sure], logits.argmax(-1)[sure])
    with pytest.raises(ValueError):
        _net(dn, C, K, C_out, "global_mean").forward_nll(x, mass, labels=lab, **kw)


# ---- 6. mesh batches, 7. graphs ------------------------------------------------------------------------------------
def _meshes(dn, shapes, K):
    out = []
    for i, (n, m) in enumerate(shapes):
        mass, L, evals, evecs, gX, gY = dn.synthetic.structural_operators(n, m, K, seed=i, device="cuda")
        _, faces = dn.synthetic.torus_mesh(n, m, seed=i)
        out.append(dict(mass=mass, evals=evals, evecs=evecs, gradX=gX, gradY=gY, faces=faces.cuda()))
    return out


@pytest.mark.parametrize("outputs_at", ["vertices", "faces"])
def test_forward_batch_nll_matches_per_mesh(dn, outputs_at):
    dn.set_engine("tc3x")
    K, C, C_out = 32, 64, 9
    meshes = _meshes(dn, [(9, 11), (14, 10), (7, 8)], K)
    mb = dn.MeshBatch(meshes)
    net = _net(dn, C, K, C_out, outputs_at)
    xs = [torch.randn(it["mass"].shape[0], 16, generator=_gen(20 + i)).cuda() for i, it in enumerate(meshes)]
    key = "faces" if outputs_at == "faces" else "mass"
    labs = [torch.randint(0, C_out, (it[key].shape[0],), generator=_gen(30 + i)).cuda() for i, it in enumerate(meshes)]
    net.zero_grad()
    loss_b, preds = net.forward_batch_nll(mb, xs, labs)
    loss_b.sum().backward()
    gb = {k: p_.grad.clone() for k, p_ in net.named_parameters()}
    net.zero_grad()
    for i, it in enumerate(meshes):
        l1, p1 = net.forward_nll(xs[i], it["mass"], evals=it["evals"], evecs=it["evecs"], gradX=it["gradX"],
                                 gradY=it["gradY"], faces=it["faces"], labels=labs[i])
        assert abs(l1.item() - loss_b[i].item()) <= 1e-5 * abs(l1.item()), i
        l1.backward()
    for k, p_ in net.named_parameters():
        err = (p_.grad - gb[k]).abs().max().item()
        assert err <= 5e-5 * p_.grad.abs().max().item() + 1e-12, (k, err)
    if outputs_at == "vertices":
        # padding rows carry ignore_index: the batch-layout input on padding rows changes nothing, bitwise
        x_lay = mb.pack(xs)
        pad = torch.ones(mb.V, dtype=torch.bool, device="cuda")
        for r0, n in zip(mb.row_begin, mb.n_rows):
            pad[r0:r0 + n] = False
        assert pad.any()
        x2 = x_lay.clone()
        x2[pad] = 1e3
        with torch.no_grad():
            a, pa = net.forward_batch_nll(mb, x_lay, labs)
            b_, pb = net.forward_batch_nll(mb, x2, labs)
        assert torch.equal(a, b_) and all(torch.equal(u, v) for u, v in zip(pa, pb))
    # per-mesh label lengths are checked, also where the total is right
    swapped = [labs[1], labs[0]] + labs[2:]
    if swapped[0].shape != labs[0].shape:
        with pytest.raises(ValueError):
            net.forward_batch_nll(mb, xs, swapped)


@pytest.mark.parametrize("outputs_at", ["vertices", "faces"])
def test_graphed_train_steps(dn, outputs_at):
    """Face outputs also capture the element mean and its cached vertex -> face CSR."""
    dn.set_engine("tc3x")
    K, C, C_out = 32, 64, 260
    meshes = _meshes(dn, [(12, 13), (9, 10)], K)
    mb = dn.MeshBatch(meshes)
    net = _net(dn, C, K, C_out, outputs_at)
    xs = [torch.randn(it["mass"].shape[0], 16, generator=_gen(40 + i)).cuda() for i, it in enumerate(meshes)]
    key = "faces" if outputs_at == "faces" else "mass"
    labs = [torch.randint(0, C_out, (it[key].shape[0],), generator=_gen(50 + i)).cuda()
            for i, it in enumerate(meshes)]
    it = meshes[0]

    def single(net_, x_, l_):
        return net_.forward_nll(x_, it["mass"], evals=it["evals"], evecs=it["evecs"], gradX=it["gradX"],
                                gradY=it["gradY"], faces=it["faces"], labels=l_)[0]

    def batched(net_, xs_, ls_):
        return net_.forward_batch_nll(mb, xs_, ls_)[0].sum()

    for fn, inputs in ((single, (xs[0], labs[0])), (batched, (xs, labs))):
        net.zero_grad()
        fn(net, *inputs).backward()
        ref = {k: p_.grad.clone() for k, p_ in net.named_parameters()}
        step = dn.graphs.GraphedTrainStep(net, fn, inputs)
        dn.graphs.GraphedTrainStep.zero_grads(net)
        step.replay()
        torch.cuda.synchronize()
        for k, p_ in net.named_parameters():
            assert torch.equal(p_.grad, ref[k]), (fn.__name__, k)


# ---- 8. refusals ---------------------------------------------------------------------------------------------------
def test_simt_engine_takes_the_composed_path(dn):
    x, w, b, lab, gr = _inputs(300, 48, 20, seed=12)
    G = _gold(x, w, b, lab, gr)
    dn.set_engine("simt")
    try:
        lib = dn._lib.load()
        xc = x.cuda()
        nll = torch.empty(300, device="cuda")
        c0 = lib.dn_kernel_launch_count()
        rc = lib.dn_linear_nll_fwd(xc.data_ptr(), w.cuda().data_ptr(), None, lab.cuda().data_ptr(), 300, 48, 20, -100,
                                   nll.data_ptr(), torch.empty(300, dtype=torch.int64, device="cuda").data_ptr(),
                                   nll.data_ptr(), dn._lib.ENGINE_SIMT, None)
        assert rc == -2 and lib.dn_kernel_launch_count() == c0
        wc = w.cuda()
        need = lib.dn_linear_nll_workspace_bytes(300, 48, 20)
        ws = torch.empty(need, dtype=torch.uint8, device="cuda")
        gx, gw = torch.empty_like(xc), torch.empty_like(wc)
        rc = lib.dn_linear_nll_bwd(xc.data_ptr(), wc.data_ptr(), None, lab.cuda().data_ptr(), nll.data_ptr(),
                                   nll.data_ptr(), 300, 48, 20, -100, gx.data_ptr(), gw.data_ptr(), None,
                                   ws.data_ptr(), need, dn._lib.ENGINE_SIMT, None)
        assert rc == -2 and lib.dn_kernel_launch_count() == c0
        out, pred = dn.ops.linear_nll(xc, w.cuda(), b.cuda(), lab.cuda())
        err = (out.cpu().to(D) - G["nll"]).abs().max().item()
        assert err <= 1e-5 * G["nll"].abs().max().item()
    finally:
        dn.set_engine("tc3x")


def test_c_abi_refusals_enqueue_nothing(dn):
    lib = dn._lib.load()
    R, C, n = 300, 64, 50
    x, w, b, lab, gr = (t.cuda() for t in _inputs(R, C, n, seed=13))
    out = torch.empty(R, device="cuda")
    am = torch.empty(R, dtype=torch.int64, device="cuda")
    P = lambda t: t.data_ptr()  # noqa: E731
    tc = dn._lib.ENGINE_TC3X
    c0 = lib.dn_kernel_launch_count()
    for (RR, CC, nn_) in [(R, 40, n), (R, 272, n), (0, C, n), (R, C, 0)]:
        rc = lib.dn_linear_nll_fwd(P(x), P(w), P(b), P(lab), RR, CC, nn_, -100, P(out), P(am), P(out), tc, None)
        assert rc in (-1, -2), (RR, CC, nn_, rc)
    need = lib.dn_linear_nll_workspace_bytes(R, C, n)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    gx, gw, gbias = torch.empty_like(x), torch.empty_like(w), torch.empty_like(b)
    rc = lib.dn_linear_nll_bwd(P(x), P(w), P(b), P(lab), P(out), P(gr), R, C, n, -100, P(gx), P(gw), P(gbias), P(ws),
                               need - 8, tc, None)
    assert rc == -3
    assert lib.dn_kernel_launch_count() == c0
