"""The random rotations of ``batch.random_rotations`` (CPU): the reference's two constructions rebuilt from the
uniforms they drew (tests/golden/rotations.npz, made by oracle/make_golden_rotations.py from the unmodified
``random_rotation_matrix`` and ``random_rotate_points_y``), and the properties every draw must have."""
import os

import numpy as np
import pytest
import torch

from conftest import ROOT

import diffusion_net_b200 as dn

GOLD = os.path.join(ROOT, "tests", "golden", "rotations.npz")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def test_uniform_rotation_matches_the_reference_from_its_uniforms(gold):
    R = dn.batch.rotation_from_uniforms(torch.from_numpy(gold["u"])).numpy()
    assert R.shape == gold["R"].shape
    assert np.abs(R - gold["R"]).max() <= 1e-6


def test_y_rotation_matches_the_reference_from_its_uniform(gold):
    R = dn.batch.rotation_from_uniforms(torch.from_numpy(gold["uy"]), axis="y").numpy()
    assert np.abs(R - gold["Ry"]).max() <= 1e-6
    assert np.array_equal(R[:, 1], np.tile([0.0, 1.0, 0.0], (len(R), 1)))    # y is fixed


@pytest.mark.parametrize("axis", [None, "y"])
def test_draws_are_proper_rotations(axis):
    g = torch.Generator().manual_seed(0)
    R = dn.batch.random_rotations(512, axis=axis, generator=g, device="cpu")
    assert R.dtype == torch.float32 and R.shape == (512, 3, 3)
    R64 = R.double()
    assert (R64 @ R64.transpose(1, 2) - torch.eye(3, dtype=torch.float64)).abs().max() < 1e-6
    assert (torch.linalg.det(R64) - 1).abs().max() < 1e-6
    again = dn.batch.random_rotations(512, axis=axis, generator=torch.Generator().manual_seed(0), device="cpu")
    assert torch.equal(R, again)


def test_uniform_draws_cover_so3():
    """Haar-uniform rotations map a fixed unit vector uniformly onto the sphere: the image of e_z has mean ~0 and
    second moment ~I/3 (4096 draws; bounds 5 standard errors)."""
    R = dn.batch.random_rotations(4096, generator=torch.Generator().manual_seed(1), device="cpu").double()
    v = R[:, 2, :]                                   # e_z @ R
    se = 1.0 / np.sqrt(3 * 4096)
    assert v.mean(0).abs().max() < 5 * se
    assert (v.t() @ v / 4096 - torch.eye(3, dtype=torch.float64) / 3).abs().max() < 5 * 0.3 / np.sqrt(4096)


def test_refusals():
    with pytest.raises(ValueError, match="axis"):
        dn.batch.random_rotations(2, axis="x", device="cpu")
    with pytest.raises(ValueError, match=r"\(n, 3\)"):
        dn.batch.rotation_from_uniforms(torch.rand(4, 2))
