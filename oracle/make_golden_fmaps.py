"""Generate ``tests/golden/fmaps_small.*.npz`` by running the UNMODIFIED reference functional-map model here (build container
only; needs /root/reference):

    python oracle/make_golden_fmaps.py

``experiments/functional_correspondence/fmaps_model.py`` is imported as it lies (it imports the reference
``diffusion_net`` package, loaded first through ``ref_import`` and its stubs).  Two different small seeded meshes, shape
x a 12 x 16 jittered torus and shape y a 162-vertex perturbed icosphere, get their operators from the reference's own
``get_operators(..., k_eig=48)``.  Recorded:
  * per shape, under ``x:`` / ``y:``: verts, faces, mass, evals, evecs, gradX / gradY (COO, fp32);
  * ``p:<key>``: the shipped ``faust_xyz.pth`` weights as float16; the reference runs on exactly these rounded weights;
  * the model in eval mode (no dropout masks) in fp64 (weights and operators promoted): ``C64`` (n x n), ``feat1_64``,
    ``feat2_64``; in fp32 ``C32`` and, as scalars max|x32 - x64| / max|x64|, the reference's own fp32 errors
    ``err32:C``, ``err32:feat1``, ``err32:feat2``;
  * ``C_gt`` (seeded) and ``grad:<key>``: the fp64 autograd gradient of mean((C_pred - C_gt)^2) for every parameter of
    at most 384 entries (biases, diffusion times, first_lin.weight), which pins ``dn_oracle_fmaps.model_torch``, the fp64
    gold of every gradient, to the reference; ``gradfloor:<key>`` for every parameter: the reference's own fp32 error
    on its gradient, max|g32 - g64| / max|g64|, with the fp32 run fed the fp64 run's upstream gradient
    2 (C64 - C_gt) / n^2;
  * the evaluation's pointwise map (functional_correspondence.py:194-196) from the fp32 run: ``map`` (the reference's
    ``find_knn(..., k=1, method='cpu_kd')``), ``map_target`` (the fp32 points it searched, evecs_x[:, :30] C^T) and, per
    query, the fp64 squared distances to the best and second-best target (``map_d1`` / ``map_d2``).
The fixture is stored in four parts, ``conftest.load_golden`` merges them: the weights of first_lin and blocks 0-1
(``params_a``), the other weights (``params_b``), the meshes and the outputs, each about 0.5 MB.  The fixture is data only.
"""
from __future__ import annotations

import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import diffusion_net_b200.synthetic as syn  # noqa: E402

FMAPS_MODEL = "/root/reference/experiments/functional_correspondence/fmaps_model.py"
CKPT = "/root/reference/experiments/functional_correspondence/pretrained_models/faust_xyz.pth"
K_EIG = 48
N_FMAP = 30


def _np(t):
    return t.detach().cpu().numpy()


def import_fmaps_model():
    from ref_import import import_reference
    import_reference()
    spec = importlib.util.spec_from_file_location("fmaps_model", FMAPS_MODEL)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    from ref_import import import_reference
    import dn_oracle_fmaps as OF
    ref = import_reference()
    fm = import_fmaps_model()
    out = {}
    shapes = {}
    for tag, (verts, faces) in (("x", syn.torus_mesh(12, 16, seed=0)), ("y", syn.icosphere_mesh(2, seed=1))):
        verts = torch.as_tensor(np.asarray(verts), dtype=torch.float32)
        faces = torch.as_tensor(np.asarray(faces), dtype=torch.int64)
        frames, mass, L, evals, evecs, gradX, gradY = ref.geometry.get_operators(verts, faces, k_eig=K_EIG)
        gradX, gradY = gradX.coalesce(), gradY.coalesce()
        shapes[tag] = [verts, faces, frames, mass, L, evals, evecs, gradX, gradY, None,
                       torch.arange(verts.shape[0])]
        out.update({tag + ":verts": _np(verts), tag + ":faces": _np(faces), tag + ":mass": _np(mass).astype(np.float32),
                    tag + ":evals": _np(evals).astype(np.float32), tag + ":evecs": _np(evecs).astype(np.float32),
                    tag + ":gradX_idx": _np(gradX.indices()), tag + ":gradX_vals": _np(gradX.values()).astype(np.float32),
                    tag + ":gradY_idx": _np(gradY.indices()), tag + ":gradY_vals": _np(gradY.values()).astype(np.float32)})
    sd = torch.load(CKPT, map_location="cpu")
    sd16 = {k: v.to(torch.float16) for k, v in sd.items()}
    out.update({"p:" + k: _np(v) for k, v in sd16.items()})
    C_gt = np.random.RandomState(5).randn(N_FMAP, N_FMAP) * 0.2
    out["C_gt"] = C_gt
    for dt, sfx in ((torch.float64, "64"), (torch.float32, "32")):
        model = fm.FunctionalMapCorrespondenceWithDiffusionNetFeatures(n_feat=128, input_features="xyz")
        model.load_state_dict({k: v.to(dt) for k, v in sd16.items()}, strict=True)
        model = model.to(dt).eval()
        cast = lambda t: t.to(dt) if torch.is_tensor(t) and t.is_floating_point() else t
        s1 = [cast(t) for t in shapes["x"]]
        s2 = [cast(t) for t in shapes["y"]]
        C_pred, feat1, feat2 = model(s1, s2)
        res = {"C": _np(C_pred[0]), "feat1": _np(feat1), "feat2": _np(feat2)}
        if dt == torch.float64:
            out["C64"], out["feat1_64"], out["feat2_64"] = res["C"], res["feat1"], res["feat2"]
        else:
            out["C32"] = res["C"]
            for k, v in res.items():
                g = out[k + "_64"] if k != "C" else out["C64"]
                out["err32:" + k] = np.float64(np.abs(v - g).max() / np.abs(g).max())
        if dt == torch.float64:
            loss = torch.mean(torch.square(C_pred.squeeze(0) - torch.from_numpy(C_gt)))
            loss.backward()
            out["loss64"] = np.float64(loss.item())
            grads64 = {k: _np(p.grad) for k, p in model.named_parameters()}
            out.update({"grad:" + k: g for k, g in grads64.items() if g.size <= 384})
        else:
            # the reference's own fp32 gradient error, under the fp64 run's upstream gradient G = 2 (C64 - C_gt) / n^2
            G = torch.from_numpy(2 * (out["C64"] - C_gt) / N_FMAP ** 2).float()
            (C_pred[0] * G).sum().backward()
            for k, p in model.named_parameters():
                g64 = grads64[k]
                out["gradfloor:" + k] = np.float64(np.abs(_np(p.grad) - g64).max() / np.abs(g64).max())
            with torch.no_grad():                                       # functional_correspondence.py:194-196
                evec1_on_2 = s1[6][:, :N_FMAP] @ C_pred.squeeze(0).transpose(0, 1)
                _, labels = ref.geometry.find_knn(s2[6][:, :N_FMAP], evec1_on_2, k=1, method='cpu_kd')
            out["map"] = _np(labels).reshape(-1).astype(np.int64)
            out["map_target"] = _np(evec1_on_2)
            _, d1, d2 = OF.nearest_neighbor(_np(s2[6][:, :N_FMAP]), _np(evec1_on_2))
            out["map_d1"], out["map_d2"] = d1, d2
    first = ("p:feature_extractor.first_lin.", "p:feature_extractor.block_0.", "p:feature_extractor.block_1.")
    parts = {"params_a": {k: v for k, v in out.items() if k.startswith(first)},
             "params_b": {k: v for k, v in out.items() if k.startswith("p:") and not k.startswith(first)},
             "meshes": {k: v for k, v in out.items() if k.startswith(("x:", "y:"))},
             "outputs": {k: v for k, v in out.items() if not k.startswith(("p:", "x:", "y:"))}}
    for name, arrs in parts.items():
        path = os.path.join(ROOT, "tests", "golden", "fmaps_small.{}.npz".format(name))
        np.savez_compressed(path, **arrs)
        print(path, os.path.getsize(path), "bytes,", len(arrs), "arrays")


if __name__ == "__main__":
    main()
