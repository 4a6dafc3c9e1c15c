"""Generate the operator-construction fixture by running the UNMODIFIED reference's ``get_operators`` here (build
container only; needs /root/reference):

    python oracle/make_golden_ops.py

``tests/golden/op_cache_patch/<sha1>_0.npz`` -- the cache entry the reference writes (geometry.py:526-568) for
``ops_patch_mesh()``, k_eig = 32: a jittered open grid patch (boundary vertices) plus
  * one unreferenced vertex (no face: NaN normal after the wiggle -> the random-normal path, geometry.py:137-141; a zero
    Laplacian row, so an eigenpair of the eps-regularised problem sits at eps / (eps * mean mass)), and
  * one zero-area face on three coincident new vertices (NaN normals that the wiggle repairs, geometry.py:128-135; every
    cotangent is 0 / (0 + denom_eps), the denom_eps path of the Laplacian; explicit zeros in L's pattern).
(potpourri3d's cotan_laplacian / vertex_areas are the numpy restatements in ``ref_import.py``.)  The existing fixtures
are not regenerated.
"""
from __future__ import annotations

import os
import shutil
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import diffusion_net_b200.synthetic as syn  # noqa: E402

K_EIG = 32


def ops_patch_mesh():
    """(verts fp32, faces int64) of the fixture: 22 x 22 patch + 3 coincident vertices in one face + 1 unreferenced."""
    v, f = syn.patch_mesh(22, 22, seed=11)
    v, f = v.numpy(), f.numpy()
    V = v.shape[0]
    extra = np.array([[0.5, 0.5, 0.4]] * 3 + [[1.3, -0.2, 0.1]], dtype=np.float32)
    verts = np.concatenate((v, extra), 0)
    faces = np.concatenate((f, np.array([[V, V + 1, V + 2]], dtype=np.int64)), 0)
    return torch.from_numpy(verts), torch.from_numpy(faces)


def main():
    from ref_import import import_reference
    dn = import_reference()
    verts, faces = ops_patch_mesh()
    out = os.path.join(ROOT, "tests", "golden", "op_cache_patch")
    shutil.rmtree(out, ignore_errors=True)
    os.makedirs(out)
    with tempfile.TemporaryDirectory() as tmp:
        dn.geometry.get_operators(verts, faces, k_eig=K_EIG, op_cache_dir=tmp)
        files = sorted(os.listdir(tmp))
        assert len(files) == 1, files
        shutil.copy(os.path.join(tmp, files[0]), os.path.join(out, files[0]))
    print(files[0], os.path.getsize(os.path.join(out, files[0])))


if __name__ == "__main__":
    main()
