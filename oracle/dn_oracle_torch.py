"""torch-CPU restatement of the reference DiffusionNetBlock forward, used as the *timed CPU arm*
(``bench.py`` ``cpu_baseline`` / ``--impl reference``) on the GPU box, where /root/reference does
not exist.  TEST/BENCH INFRASTRUCTURE ONLY -- never imported by the product package.

It issues the same torch ops the reference does on CPU tensors (``torch.matmul`` dense GEMMs,
``torch.mm`` on sparse COO operands, ``stack``/``cat`` copies, elementwise exp/tanh/relu), so its
run time on the host cores is what the reference's own CPU PyTorch path costs.  Parity status:
PINNED -- ``tests/test_oracle.py::test_torch_port_matches_reference`` checks it against the
live-reference fixtures in ``tests/golden``.  Citations are to /root/reference/src/diffusion_net/.
"""
from __future__ import annotations

import torch


def to_basis(values, basis, massvec):
    """geometry.py:572-583."""
    return torch.matmul(basis.transpose(-2, -1), values * massvec.unsqueeze(-1))


def from_basis(values, basis):
    """geometry.py:586-598 (real branch)."""
    return torch.matmul(basis, values)


def block_forward(x_in, mass, evals, evecs, gradX, gradY, params, with_gradient_features=True, relu_masks=None,
                  pre_acts=None, diffuse=None):
    """layers.py:200-241 for a batched input (B,V,C); gradX/gradY sparse COO (B,V,V) or lists of (V,V).

    Test hooks (not reference behaviour): ``pre_acts`` (a list) receives every hidden layer's pre-activation;
    ``relu_masks`` (one bool tensor per hidden layer) replaces ``relu(h)`` by ``h * mask`` so that a gradient can be
    checked under a GIVEN activation pattern -- the gradient of ReLU is discontinuous at 0, and an fp32 forward may
    land on the other side of a kink than the fp64 one for pre-activations of order 1e-7.  ``diffuse`` (a callable
    ``(x_in, t) -> x_diffuse`` with t already clamped) replaces the spectral diffusion, so that a test can compose the
    block around another solve of the heat equation (the implicit method, layers.py:69-84); ``evals`` / ``evecs`` are
    then not read."""
    t = torch.clamp(params["diffusion.diffusion_time"], min=1e-8)                  # layers.py:48-49
    if diffuse is not None:
        x_diffuse = diffuse(x_in, t)
    else:
        x_spec = to_basis(x_in, evecs, mass)                                       # :59
        coefs = torch.exp(-evals.unsqueeze(-1) * t.unsqueeze(0))                   # :62-63
        x_diffuse = from_basis(coefs * x_spec, evecs)                              # :64-67
    feats = [x_in, x_diffuse]
    if with_gradient_features:
        grads = []
        for b in range(x_in.shape[0]):                                             # :217-222
            gx = torch.mm(gradX[b], x_diffuse[b])
            gy = torch.mm(gradY[b], x_diffuse[b])
            grads.append(torch.stack((gx, gy), dim=-1))
        v = torch.stack(grads, dim=0)                                              # :223
        lin = lambda w, a: torch.matmul(a, w.t())
        if "gradient_features.A.weight" in params:                                 # :125-126
            A = params["gradient_features.A.weight"]
            b_re, b_im = lin(A, v[..., 0]), lin(A, v[..., 1])
        else:                                                                      # :122-123
            A_re, A_im = params["gradient_features.A_re.weight"], params["gradient_features.A_im.weight"]
            b_re = lin(A_re, v[..., 0]) - lin(A_im, v[..., 1])
            b_im = lin(A_re, v[..., 1]) + lin(A_im, v[..., 0])
        feats.append(torch.tanh(v[..., 0] * b_re + v[..., 1] * b_im))              # :128-130
    h = torch.cat(feats, dim=-1)                                                   # :229/:232
    i = 0
    while "mlp.miniMLP_mlp_layer_{:03d}.weight".format(i) in params:               # layers.py:140-164
        w = params["mlp.miniMLP_mlp_layer_{:03d}.weight".format(i)]
        b = params["mlp.miniMLP_mlp_layer_{:03d}.bias".format(i)]
        h = torch.addmm(b, h.reshape(-1, h.shape[-1]), w.t()).reshape(h.shape[:-1] + (w.shape[0],))
        if "mlp.miniMLP_mlp_layer_{:03d}.weight".format(i + 1) in params:
            if pre_acts is not None:
                pre_acts.append(h.detach())
            h = torch.relu(h) if relu_masks is None else h * relu_masks[i].to(h.dtype).reshape(h.shape)
        i += 1
    return h + x_in                                                                # :239
