"""Generate ``tests/golden/rotations.npz`` from the UNMODIFIED reference's rotation helpers (build container only; needs
/root/reference):

    python oracle/make_golden_rotations.py

For each of 16 fixed seeds s:
  * ``R[s]``: ``diffusion_net.utils.random_rotation_matrix(np.random.RandomState(s))`` (float64), and ``u[s]`` the three
    uniforms it drew, ``RandomState(s).rand(3)`` (the function's first and only draw);
  * ``Ry[s]``: the matrix ``random_rotate_points_y`` multiplies by, read off as ``random_rotate_points_y(I)`` in float64
    after ``torch.manual_seed(s)``, and ``uy[s]`` the uniform it drew, ``torch.rand(1, dtype=float64)`` after the same
    seed.
The fixture is data only: tests/test_rotations.py rebuilds every matrix from its uniforms with
``batch.rotation_from_uniforms``.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "rotations.npz")
SEEDS = list(range(16))


def main():
    sys.path.insert(0, HERE)
    from ref_import import import_reference
    ref = import_reference()
    utils = ref.utils
    R, u, Ry, uy = [], [], [], []
    for s in SEEDS:
        R.append(utils.random_rotation_matrix(np.random.RandomState(s)))
        u.append(np.random.RandomState(s).rand(3))
        torch.manual_seed(s)
        Ry.append(utils.random_rotate_points_y(torch.eye(3, dtype=torch.float64)).numpy())
        torch.manual_seed(s)
        uy.append(torch.rand(1, dtype=torch.float64).numpy())
    np.savez(OUT, seeds=np.asarray(SEEDS, np.int64), R=np.stack(R), u=np.stack(u), Ry=np.stack(Ry), uy=np.stack(uy))
    print("wrote", OUT)


if __name__ == "__main__":
    main()
