"""Seeded synthetic meshes and operator tuples for benchmarks and parity tests.

The reference ships no data (SURVEY.md section 8d); these generators build inputs
with the statistics the reference's own ``get_operators()`` produces on a
jittered torus, without needing the reference at run time:

* ``torus_mesh``       -- the Tier-G mesh (verts, faces), for callers that have
                          the reference precompute available (build container).
* ``structural_operators`` -- Tier-S: the same 7-nnz/row sparsity pattern, random
                          gradient values, M-orthonormal random eigenbasis.  Gives
                          an operator tuple in exactly the layout
                          ``diffusion_net.geometry.get_operators`` returns
                          (geometry.py:289-296): ``mass (V)``, ``L`` sparse,
                          ``evals (K)``, ``evecs (V,K)``, ``gradX``/``gradY``
                          coalesced sparse COO (V,V) sharing one pattern.
"""
from __future__ import annotations

import numpy as np
import torch


def torus_mesh(n, m, seed=0, jit=0.25, R=1.0, r=0.4):
    """n x m jittered grid on a torus; vertex id = i*m + j; V = n*m, F = 2nm."""
    rs = np.random.RandomState(seed)
    ju = rs.rand(n, m)
    jv = rs.rand(n, m)
    ii, jj = np.meshgrid(np.arange(n), np.arange(m), indexing="ij")
    u = 2 * np.pi * (ii + jit * (ju - 0.5)) / n
    v = 2 * np.pi * (jj + jit * (jv - 0.5)) / m
    x = (R + r * np.cos(v)) * np.cos(u)
    y = (R + r * np.cos(v)) * np.sin(u)
    z = r * np.sin(v)
    verts = np.stack((x, y, z), axis=-1).reshape(-1, 3).astype(np.float32)
    vid = lambda a, b: ((a % n) * m + (b % m))
    f1 = np.stack((vid(ii, jj), vid(ii + 1, jj), vid(ii + 1, jj + 1)), axis=-1).reshape(-1, 3)
    f2 = np.stack((vid(ii, jj), vid(ii + 1, jj + 1), vid(ii, jj + 1)), axis=-1).reshape(-1, 3)
    faces = np.concatenate((f1, f2), axis=0).astype(np.int64)
    return torch.from_numpy(verts), torch.from_numpy(faces)


def patch_mesh(n, m, seed=0, jit=0.25, height=0.15):
    """n x m jittered open grid patch (a disk-like mesh with a boundary) over [0, 1] x [0, m/n], with a smooth height
    field; vertex id = i*m + j; V = n*m, F = 2(n-1)(m-1)."""
    rs = np.random.RandomState(seed)
    ii, jj = np.meshgrid(np.arange(n), np.arange(m), indexing="ij")
    h = 1.0 / (n - 1)
    x = (ii + jit * (rs.rand(n, m) - 0.5) * (ii > 0) * (ii < n - 1)) * h
    y = (jj + jit * (rs.rand(n, m) - 0.5) * (jj > 0) * (jj < m - 1)) * h
    z = height * np.sin(2.1 * x + 0.3) * np.cos(3.3 * y - 0.2)
    verts = np.stack((x, y, z), axis=-1).reshape(-1, 3).astype(np.float32)
    a, b = ii[:-1, :-1], jj[:-1, :-1]
    vid = lambda p, q: p * m + q
    f1 = np.stack((vid(a, b), vid(a + 1, b), vid(a + 1, b + 1)), axis=-1).reshape(-1, 3)
    f2 = np.stack((vid(a, b), vid(a + 1, b + 1), vid(a, b + 1)), axis=-1).reshape(-1, 3)
    return torch.from_numpy(verts), torch.from_numpy(np.concatenate((f1, f2), 0).astype(np.int64))


def icosphere_mesh(subdiv, seed=0, jit=0.1, bump=0.08):
    """Genus-0 test mesh: a subdivided icosahedron (V = 10 * 4**subdiv + 2) whose vertices are jittered tangentially
    (by ``jit`` of the edge length) and pushed radially by a few smooth bumps of relative height ``bump``.  A sphere's
    Laplace-Beltrami eigenvalues come in clusters of 2l + 1; the perturbation splits each only slightly, so the mesh
    has wide near-degenerate clusters."""
    t = (1.0 + 5 ** 0.5) / 2.0
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
         (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
         (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10),
         (8, 6, 7), (9, 8, 1)]
    verts = [np.array(p, dtype=np.float64) / np.linalg.norm(p) for p in v]
    faces = f
    for _ in range(subdiv):
        mid = {}

        def midpoint(a, b):
            key = (min(a, b), max(a, b))
            if key not in mid:
                p = verts[a] + verts[b]
                verts.append(p / np.linalg.norm(p))
                mid[key] = len(verts) - 1
            return mid[key]
        nf = []
        for a, b, c in faces:
            ab, bc, ca = midpoint(a, b), midpoint(b, c), midpoint(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        faces = nf
    P = np.array(verts)
    rs = np.random.RandomState(seed)
    h = 1.1 / (2 ** subdiv)                                       # about one edge length on the unit sphere
    d = rs.randn(*P.shape) * jit * h
    d -= (d * P).sum(1, keepdims=True) * P                        # tangential jitter
    P = P + d
    P /= np.linalg.norm(P, axis=1, keepdims=True)
    centres = rs.randn(5, 3)
    centres /= np.linalg.norm(centres, axis=1, keepdims=True)
    r = 1.0 + bump * np.exp(-8.0 * (1.0 - P @ centres.T)).sum(1)
    P = P * r[:, None]
    return torch.from_numpy(P.astype(np.float32)), torch.from_numpy(np.array(faces, dtype=np.int64))


def torus_pattern(n, m):
    """(rows, cols) int64, row-sorted then col-sorted: self + 6 torus-grid
    neighbours, the pattern the cotan Laplacian / gradient matrices share."""
    ii, jj = np.meshgrid(np.arange(n), np.arange(m), indexing="ij")
    vid = lambda a, b: ((a % n) * m + (b % m))
    nb = np.stack((vid(ii, jj), vid(ii + 1, jj), vid(ii - 1, jj), vid(ii, jj + 1), vid(ii, jj - 1),
                   vid(ii + 1, jj + 1), vid(ii - 1, jj - 1)), axis=-1).reshape(n * m, 7)
    nb = np.sort(nb, axis=1)
    rows = np.repeat(np.arange(n * m, dtype=np.int64), 7)
    return rows, nb.reshape(-1).astype(np.int64)


def structural_operators(n, m, k_eig, seed=0, device="cpu", permute=False):
    """Tier-S operator tuple ``(mass, L, evals, evecs, gradX, gradY)`` (fp32).

    ``permute=True`` applies a random vertex relabelling (worst-case gather
    locality for the sparse-gradient kernel)."""
    V = n * m
    g = torch.Generator().manual_seed(1234 + seed)
    rows, cols = torus_pattern(n, m)
    nnz = rows.shape[0]
    sigma = 0.12 * float(np.sqrt(V))
    vx = torch.randn(nnz, generator=g) * sigma
    vy = torch.randn(nnz, generator=g) * sigma
    # rows of a gradient operator annihilate constants: remove the row mean
    # (values are still in unpermuted row-major order here, 7 per row)
    vx = (vx.view(V, 7) - vx.view(V, 7).mean(dim=1, keepdim=True)).reshape(-1)
    vy = (vy.view(V, 7) - vy.view(V, 7).mean(dim=1, keepdim=True)).reshape(-1)
    if permute:
        perm = np.random.RandomState(seed).permutation(V).astype(np.int64)
        rows, cols = perm[rows], perm[cols]
    idx = torch.from_numpy(np.stack((rows, cols)))
    gradX = torch.sparse_coo_tensor(idx, vx, (V, V)).coalesce()
    gradY = torch.sparse_coo_tensor(idx, vy, (V, V)).coalesce()
    L = torch.sparse_coo_tensor(idx, torch.randn(nnz, generator=g), (V, V)).coalesce()
    mass = (8.0 / V) * (0.5 + torch.rand(V, generator=g))
    q, _ = torch.linalg.qr(torch.randn(V, k_eig, generator=g, dtype=torch.float64))
    evecs = (q / mass.double().sqrt()[:, None]).float()       # Phi^T M Phi = I
    evals = (200.0 * torch.arange(k_eig, dtype=torch.float32) / k_eig)
    out = (mass, L, evals, evecs.contiguous(), gradX, gradY)
    return tuple(t.to(device) for t in out)


def block_weights(C, seed=0, with_gradient_rotations=True, with_gradient_features=True,
                  mlp_hidden_dims=None, t_lo=1e-3, t_hi=0.3):
    """Seeded DiffusionNetBlock parameters under the reference state_dict names
    (layers.py:38,110-113,150-155); nn.Linear default init ranges, and
    ``diffusion_time ~ U(t_lo, t_hi)`` (default init 0 makes diffusion a pure
    projection; shipped checkpoints span 3e-6..0.47, SURVEY.md section 2 row 15)."""
    g = torch.Generator().manual_seed(4321 + seed)
    hid = [C, C] if mlp_hidden_dims is None else list(mlp_hidden_dims)
    p = {}
    p["diffusion.diffusion_time"] = t_lo + (t_hi - t_lo) * torch.rand(C, generator=g)

    def lin(n_out, n_in):
        bound = 1.0 / np.sqrt(n_in)
        return (torch.rand(n_out, n_in, generator=g) * 2 - 1) * bound

    if with_gradient_features:
        if with_gradient_rotations:
            p["gradient_features.A_re.weight"] = lin(C, C)
            p["gradient_features.A_im.weight"] = lin(C, C)
        else:
            p["gradient_features.A.weight"] = lin(C, C)
    sizes = [(3 if with_gradient_features else 2) * C] + hid + [C]
    for i in range(len(sizes) - 1):
        p["mlp.miniMLP_mlp_layer_{:03d}.weight".format(i)] = lin(sizes[i + 1], sizes[i])
        p["mlp.miniMLP_mlp_layer_{:03d}.bias".format(i)] = (
            (torch.rand(sizes[i + 1], generator=g) * 2 - 1) / np.sqrt(sizes[i]))
    return p
