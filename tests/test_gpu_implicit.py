"""Implicit heat diffusion on the GPU (diffusion_method='implicit_dense': the fp64 block Jacobi-PCG of dn_implicit.cu
behind ops.ImplicitDiffusionFn) against what the live reference computed (tests/golden/implicit_small.npz) and against
the fp64 sparse-direct oracle (oracle/dn_oracle_implicit.implicit_diffusion) at user sizes.

Gold is computed from the fp32-rounded L and mass the GPU sees, promoted to fp64: rounding L to fp32 breaks L 1 = 0 by
about eps_32 |L_vv|, which at large t moves the solution by more than the 1e-5 bound.  The spill check runs on the CPU;
everything else needs an H100."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from conftest import GOLDEN, ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import dn_oracle_implicit as OI  # noqa: E402  (checker only)
from ref_import import _cotan_laplacian, _vertex_areas  # noqa: E402

import diffusion_net_b200 as dn  # noqa: E402

gpu = pytest.mark.gpu
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.mark.skipif(shutil.which(NVCC) is None and not os.path.exists(NVCC), reason="nvcc not found")
def test_implicit_kernels_do_not_spill(tmp_path):
    flags = [f for f in dn._lib.NVCC_FLAGS if f != "-shared"]
    cmd = [NVCC] + flags + ["-Xptxas", "-v", "-c", os.path.join(dn._lib._CSRC, "dn_implicit.cu"), "-o",
                            str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [l for l in (r.stdout + r.stderr).splitlines() if "spill stores" in l]
    assert len(lines) == 8                      # one per column-count instantiation
    for l in lines:
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", l)
        assert m and m.group(1) == "0" and m.group(2) == "0", l


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    dn._lib.load()
    return torch.device("cuda")


def _np(t):
    return t.detach().cpu().numpy()


def _close(mine, gold, tol=1e-5):
    mine, gold = np.asarray(mine, dtype=np.float64), np.asarray(gold, dtype=np.float64)
    err = np.abs(mine - gold).max() / max(np.abs(gold).max(), 1e-30)
    assert err <= tol, err
    return err


def _sparse(rows, cols, vals, V, device):
    idx = torch.from_numpy(np.stack((rows, cols)).astype(np.int64))
    return torch.sparse_coo_tensor(idx, torch.from_numpy(vals), (V, V)).coalesce().to(device)


# ---------------------------------------------------------------------------------------------------------------
# reference fixture
# ---------------------------------------------------------------------------------------------------------------
def _fixture(tag, device):
    fx = load_golden("implicit_small")
    f = lambda k: fx["{}:{}".format(tag, k)]
    V = f("mass").shape[0]
    L = _sparse(f("L_rows"), f("L_cols"), f("L_vals"), V, device)
    gx = _sparse(f("gradX_idx")[0], f("gradX_idx")[1], f("gradX_vals"), V, device)
    gy = _sparse(f("gradY_idx")[0], f("gradY_idx")[1], f("gradY_vals"), V, device)
    return fx, f, L, torch.from_numpy(f("mass")).to(device), gx, gy


@gpu
@pytest.mark.parametrize("form", ["2d", "3d"])
@pytest.mark.parametrize("tag", ["torus", "patch"])
def test_learned_time_diffusion_matches_reference(cuda, tag, form):
    _, f, L, mass, _, _ = _fixture(tag, cuda)
    ltd = dn.LearnedTimeDiffusion(8, method="implicit_dense").to(cuda)
    with torch.no_grad():
        ltd.diffusion_time.copy_(torch.from_numpy(f("time_raw")))
    x = torch.from_numpy(f("x")).to(cuda)
    g = torch.from_numpy(f("g")).to(cuda)
    if form == "3d":                                   # the reference's form: (B, V, C) with a (B, V, V) sparse stack
        x, g, Lb, mb = x.unsqueeze(0), g.unsqueeze(0), torch.stack([L]), mass.unsqueeze(0)
    else:
        Lb, mb = L, mass
    x.requires_grad_(True)
    y = ltd(x, Lb, mb, None, None)
    (y * g).sum().backward()
    # the clamp write-back is the reference's, bit for bit
    assert np.array_equal(_np(ltd.diffusion_time), f("time_clamped32"))
    _close(_np(y).reshape(f("y64").shape), f("y64"))
    _close(_np(x.grad).reshape(f("gx64").shape), f("gx64"))
    _close(_np(ltd.diffusion_time.grad), f("gt64"))


@gpu
@pytest.mark.parametrize("eig", ["none", "empty"])
@pytest.mark.parametrize("outputs_at", ["vertices", "faces"])
@pytest.mark.parametrize("tag", ["torus", "patch"])
def test_net_matches_reference(cuda, tag, outputs_at, eig):
    fx, f, L, mass, gx, gy = _fixture(tag, cuda)
    net = dn.DiffusionNet(C_in=3, C_out=4, C_width=8, N_block=2, dropout=False, outputs_at=outputs_at,
                          diffusion_method="implicit_dense")
    net.load_state_dict({k[2:]: torch.from_numpy(v) for k, v in fx.items() if k.startswith("p:")}, strict=True)
    net = net.to(cuda)
    V = mass.shape[0]
    evals, evecs = (None, None) if eig == "none" else (torch.zeros(0, device=cuda), torch.zeros(V, 0, device=cuda))
    x = torch.from_numpy(f("net_x")).to(cuda)
    faces = torch.from_numpy(f("faces")).to(cuda)
    kw = dict(L=L, evals=evals, evecs=evecs, gradX=gx, gradY=gy, faces=faces)
    with torch.no_grad():                              # inference: the composed path, the head applied separately
        y0 = net(x, mass, **kw)
    y = net(x, mass, **kw)
    (y * torch.from_numpy(f("net_gout:" + outputs_at)).to(cuda)).sum().backward()
    _close(_np(y0), f("net_out:" + outputs_at))
    _close(_np(y), f("net_out:" + outputs_at))
    for k, p in net.named_parameters():
        _close(_np(p.grad), f("net_grad:{}:{}".format(outputs_at, k)), tol=1e-4)


# ---------------------------------------------------------------------------------------------------------------
# user sizes against the fp64 sparse-direct oracle
# ---------------------------------------------------------------------------------------------------------------
def _operators(verts, faces):
    """L (fp32-rounded, scipy fp64) and mass (fp32-rounded, fp64) of the mesh, normalised to unit max radius."""
    v = verts.numpy().astype(np.float64)
    v = v - v.mean(0)
    v /= np.linalg.norm(v, axis=1).max()
    f = faces.numpy()
    L = sp.csr_matrix(_cotan_laplacian(v, f, denom_eps=1e-10)).astype(np.float32).astype(np.float64)
    m = _vertex_areas(v, f)
    m = (m + 1e-8 * m.mean()).astype(np.float32).astype(np.float64)
    return L, m


def _to_torch(L, m, device):
    Lc = L.tocoo()
    return (_sparse(Lc.row, Lc.col, Lc.data.astype(np.float32), L.shape[0], device),
            torch.from_numpy(m.astype(np.float32)).to(device))


def _checkpoint_times(C):
    """Learned diffusion times of the reference's shipped human-segmentation checkpoint (all four blocks)."""
    with np.load(os.path.join(GOLDEN, "human_seg_xyz_4x128_f16.npz")) as z:
        t = np.concatenate([z[k].astype(np.float32) for k in sorted(z.files) if k.endswith("diffusion_time")])
    return np.resize(t, C)


def _run(ltd, x, Lt, mt, g):
    x = x.clone().requires_grad_(True)
    y = ltd(x, Lt, mt, None, None)
    its = int(dn.ops.implicit_last_status[1])
    (y * g).sum().backward()
    return y, x.grad, ltd.diffusion_time.grad.clone(), its


@gpu
def test_torus_20k_checkpoint_times_against_oracle(cuda):
    C = 128
    L, m = _operators(*dn.synthetic.torus_mesh(100, 200, seed=0))
    t = _checkpoint_times(C)
    rs = np.random.RandomState(0)
    x = rs.randn(2, L.shape[0], C).astype(np.float32)
    g = rs.randn(2, L.shape[0], C).astype(np.float32)
    gold_y, gold_gx, gold_gt = OI.implicit_diffusion(x, m, L, t, grad_out=g)      # gold_gt: (2, C), per input
    Lt, mt = _to_torch(L, m, cuda)
    ltd = dn.LearnedTimeDiffusion(C, method="implicit_dense").to(cuda)
    with torch.no_grad():
        ltd.diffusion_time.copy_(torch.from_numpy(t))
    xt, gt_ = torch.from_numpy(x).to(cuda), torch.from_numpy(g).to(cuda)
    y, gx, gtime, its = _run(ltd, xt[0], Lt, mt, gt_[0])                     # 2-D
    print("20k torus, C = 128, 2-D: {} forward iterations".format(its))
    _close(_np(y), gold_y[0])
    _close(_np(gx), gold_gx[0])
    _close(_np(gtime), gold_gt[0])
    ltd.diffusion_time.grad = None
    y, gx, gtime, its = _run(ltd, xt, torch.stack([Lt, Lt]), torch.stack([mt, mt]), gt_)   # (B = 2, V, C)
    print("20k torus, C = 128, (2, V, C): {} forward iterations (last mesh)".format(its))
    _close(_np(y), gold_y)
    _close(_np(gx), gold_gx)
    _close(_np(gtime), gold_gt.sum(0))


CASES = {
    "torus1200_c12": (lambda: dn.synthetic.torus_mesh(30, 40, seed=1), 12),
    "torus1200_c64": (lambda: dn.synthetic.torus_mesh(30, 40, seed=1), 64),
    "torus1200_c256": (lambda: dn.synthetic.torus_mesh(30, 40, seed=1), 256),
    "patch80_c12": (lambda: dn.synthetic.patch_mesh(8, 10, seed=2), 12),
}


@gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_widths_and_tiny_meshes_against_oracle(cuda, case):
    make, C = CASES[case]
    L, m = _operators(*make())
    t = _checkpoint_times(C)
    t[::7] = 0.5                                       # the long times of the distribution's tail
    rs = np.random.RandomState(3)
    x = rs.randn(L.shape[0], C).astype(np.float32)
    g = rs.randn(L.shape[0], C).astype(np.float32)
    gold = OI.implicit_diffusion(x, m, L, t, grad_out=g)
    Lt, mt = _to_torch(L, m, cuda)
    ltd = dn.LearnedTimeDiffusion(C, method="implicit_dense").to(cuda)
    with torch.no_grad():
        ltd.diffusion_time.copy_(torch.from_numpy(t))
    y, gx, gtime, its = _run(ltd, torch.from_numpy(x).to(cuda), Lt, mt, torch.from_numpy(g).to(cuda))
    print("{}: {} forward iterations".format(case, its))
    for mine, want in zip((y, gx, gtime), gold):
        _close(_np(mine), want)


@gpu
def test_two_calls_are_bitwise_equal(cuda):
    C = 128
    L, m = _operators(*dn.synthetic.torus_mesh(60, 80, seed=4))
    Lt, mt = _to_torch(L, m, cuda)
    t = _checkpoint_times(C)
    rs = np.random.RandomState(5)
    x = torch.from_numpy(rs.randn(L.shape[0], C).astype(np.float32)).to(cuda)
    g = torch.from_numpy(rs.randn(L.shape[0], C).astype(np.float32)).to(cuda)
    outs = []
    for _ in range(2):
        ltd = dn.LearnedTimeDiffusion(C, method="implicit_dense").to(cuda)
        with torch.no_grad():
            ltd.diffusion_time.copy_(torch.from_numpy(t))
        outs.append(_run(ltd, x, Lt, mt, g))
    a, b = outs
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]) and a[3] == b[3]


# ---------------------------------------------------------------------------------------------------------------
# errors, refusals, memoisation
# ---------------------------------------------------------------------------------------------------------------
def _small_net(cuda, N_block=2, C=16):
    torch.manual_seed(0)
    net = dn.DiffusionNet(C_in=3, C_out=4, C_width=C, N_block=N_block, dropout=False,
                          diffusion_method="implicit_dense").to(cuda)
    with torch.no_grad():
        for b in net.blocks:
            b.diffusion.diffusion_time.fill_(0.05)
    return net


@gpu
def test_errors_and_refusals(cuda, monkeypatch):
    _, f, L, mass, gx, gy = _fixture("torus", cuda)
    ltd = dn.LearnedTimeDiffusion(8, method="implicit_dense").to(cuda)
    with torch.no_grad():
        ltd.diffusion_time.copy_(torch.from_numpy(f("time_raw")))
    x = torch.from_numpy(f("x")).to(cuda)
    monkeypatch.setattr(dn.ops, "IMPLICIT_MAX_ITER", 2)
    with pytest.raises(RuntimeError, match="did not converge"):
        ltd(x, L, mass, None, None)
    monkeypatch.undo()
    assert int(dn.ops.implicit_last_status[0]) > 0
    y = ltd(x, L, mass, None, None)                      # an ordinary status return: the next solve runs normally
    _close(_np(y), f("y64"))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ltd(x.cpu(), L, mass, None, None)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ltd(x, L.cpu(), mass, None, None)
    net = _small_net(cuda)
    with pytest.raises(NotImplementedError):
        dn.graphs.GraphedNet(net)
    with pytest.raises(NotImplementedError):
        dn.graphs.GraphedBatch(net, None)
    with pytest.raises(NotImplementedError):
        dn.graphs.GraphedTrainStep(net, lambda n, *a: n(*a).sum(), (x[:, :3], mass))
    with pytest.raises(NotImplementedError):
        net.forward_batch(None, [x[:, :3]])


@gpu
def test_laplacian_csr_is_built_once_per_mesh(cuda, monkeypatch):
    _, f, L, mass, gx, gy = _fixture("patch", cuda)
    built = []
    orig = dn.ops.LaplacianCSR.__init__

    def counting(self, Lm):
        built.append(1)
        orig(self, Lm)

    monkeypatch.setattr(dn.ops.LaplacianCSR, "__init__", counting)
    net = _small_net(cuda, N_block=4)
    x = torch.from_numpy(f("net_x")).to(cuda)
    for _ in range(2):                                   # 4 blocks, two forwards and a backward: one CSR
        net(x, mass, L=L, gradX=gx, gradY=gy).sum().backward()
    assert len(built) == 1
    assert dn.ops.prepare_laplacian(L) is dn.ops.prepare_laplacian(L)
    Lb = torch.stack([L, L])
    with torch.no_grad():
        net(x.unsqueeze(0).expand(2, -1, -1).contiguous(), mass.expand(2, -1).contiguous(), L=Lb,
            gradX=torch.stack([gx, gx]), gradY=torch.stack([gy, gy]))
    assert len(built) == 3                               # the stack: one CSR per mesh, once
