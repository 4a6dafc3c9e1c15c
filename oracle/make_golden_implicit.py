"""Generate ``tests/golden/implicit_small.npz`` by running the UNMODIFIED reference's implicit diffusion here (build
container only; needs /root/reference):

    python oracle/make_golden_implicit.py

For two small seeded meshes -- the 12 x 16 jittered torus (``torus``) and the open patch with an unreferenced vertex and
a zero-area face of ``make_golden_ops.ops_patch_mesh`` (``patch``) -- the operators come from the reference's own
``get_operators(..., k_eig=0)`` (no eigenbasis: the implicit method does not need one).  Recorded per mesh, under
``<mesh>:``:
  * inputs: L (COO rows / cols / fp32 values), mass, gradX / gradY, faces, x (V, 8), the raw diffusion times spanning
    1e-8 .. 0.5 with one negative entry, an upstream gradient g;
  * ``LearnedTimeDiffusion(8, method='implicit_dense')`` on (1, V, 8) in fp32 and in fp64 (the fp32 inputs promoted,
    so the gold is the exact solution for the operators the GPU sees): the output, the clamped time the forward wrote
    back, and the reference-autograd gradients of sum(g * y) with respect to x and the time;
  * a 2-block ``DiffusionNet(3, 4, C_width=8, diffusion_method='implicit_dense')`` in fp64 with evals / evecs None, for
    outputs_at 'vertices' and 'faces': its seeded raw parameters (``p:<name>``, shared by both meshes), its input, the
    output and the gradients of sum(gout * out) with respect to every parameter.
The fixture is data only.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import diffusion_net_b200.synthetic as syn  # noqa: E402

C = 8
TIMES = np.array([-1.6e-5, 1e-8, 3e-6, 1e-4, 2e-3, 3e-2, 0.15, 0.5], dtype=np.float32)
OUTPUTS_AT = ("vertices", "faces")


def meshes():
    from make_golden_ops import ops_patch_mesh
    return {"torus": syn.torus_mesh(12, 16, seed=0), "patch": ops_patch_mesh()}


def _np(t):
    return t.detach().cpu().numpy()


def main():
    from ref_import import import_reference
    ref = import_reference()
    out = {}
    torch.manual_seed(0)
    net0 = ref.layers.DiffusionNet(C_in=3, C_out=4, C_width=C, N_block=2, dropout=False,
                                   diffusion_method="implicit_dense")
    with torch.no_grad():
        for i, b in enumerate(net0.blocks):
            b.diffusion.diffusion_time.copy_(torch.from_numpy(np.roll(TIMES, 3 * i)))
    params = {k: v.detach().clone() for k, v in net0.state_dict().items()}
    for k, v in params.items():
        out["p:" + k] = _np(v)
    for tag, (verts, faces) in meshes().items():
        frames, mass, L, evals, evecs, gradX, gradY = ref.geometry.get_operators(verts, faces, k_eig=0)
        L, gradX, gradY = L.coalesce(), gradX.coalesce(), gradY.coalesce()
        V = mass.shape[0]
        rs = np.random.RandomState(1 if tag == "torus" else 2)
        x = rs.randn(V, C).astype(np.float32)
        g = rs.randn(V, C).astype(np.float32)
        rec = {"L_rows": _np(L.indices()[0]), "L_cols": _np(L.indices()[1]), "L_vals": _np(L.values()).astype(np.float32),
               "mass": _np(mass).astype(np.float32), "faces": _np(faces), "x": x, "g": g, "time_raw": TIMES,
               "gradX_idx": _np(gradX.indices()), "gradX_vals": _np(gradX.values()).astype(np.float32),
               "gradY_idx": _np(gradY.indices()), "gradY_vals": _np(gradY.values()).astype(np.float32)}
        for dt, sfx in ((torch.float32, "32"), (torch.float64, "64")):
            ltd = ref.layers.LearnedTimeDiffusion(C, method="implicit_dense").to(dt)
            with torch.no_grad():
                ltd.diffusion_time.copy_(torch.from_numpy(TIMES))
            xt = torch.from_numpy(x).to(dt).unsqueeze(0).requires_grad_(True)
            y = ltd(xt, L.to(dt).unsqueeze(0), mass.to(dt).unsqueeze(0), None, None)
            (y * torch.from_numpy(g).to(dt).unsqueeze(0)).sum().backward()
            rec["y" + sfx] = _np(y[0])
            rec["time_clamped" + sfx] = _np(ltd.diffusion_time)
            rec["gx" + sfx] = _np(xt.grad[0])
            rec["gt" + sfx] = _np(ltd.diffusion_time.grad)
        xn = rs.randn(V, 3).astype(np.float32)
        rec["net_x"] = xn
        for oa in OUTPUTS_AT:
            net = ref.layers.DiffusionNet(C_in=3, C_out=4, C_width=C, N_block=2, dropout=False, outputs_at=oa,
                                          diffusion_method="implicit_dense").double()
            net.load_state_dict({k: v.double() for k, v in params.items()})
            d = torch.float64
            y = net(torch.from_numpy(xn).to(d), mass.to(d), L=L.to(d), evals=None, evecs=None, gradX=gradX.to(d),
                    gradY=gradY.to(d), faces=faces)
            gout = torch.from_numpy(np.random.RandomState(3).randn(*y.shape)).to(d)
            (y * gout).sum().backward()
            rec["net_out:" + oa] = _np(y)
            rec["net_gout:" + oa] = _np(gout)
            for k, p in net.named_parameters():
                rec["net_grad:{}:{}".format(oa, k)] = _np(p.grad)
        out.update({"{}:{}".format(tag, k): v for k, v in rec.items()})
    path = os.path.join(ROOT, "tests", "golden", "implicit_small.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
