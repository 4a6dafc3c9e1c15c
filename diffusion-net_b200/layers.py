"""Drop-in mirror of ``diffusion_net.layers`` (reference ``src/diffusion_net/layers.py``) whose
per-block hot path runs the hand-written sm_90a kernels behind the C-ABI.

Same class names, constructor kwargs, forward signatures, exceptions and state_dict keys as the
reference (SURVEY.md section 8b), so shipped ``.pth`` checkpoints load with ``strict=True`` and
experiment scripts only change their import.  CUDA float32 tensors only -- there is no CPU path.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops


class LearnedTimeDiffusion(nn.Module):
    """Per-channel learned-time heat diffusion (reference layers.py:17-90).

    ``spectral``: ``evecs @ (exp(-evals t^T) * (evecs^T (mass * x)))``.  ``implicit_dense``: per channel
    ``(M + t_c L)^-1 M x_c``, which the reference forms as a dense (B, C, V, V) Cholesky; here a sparse fp64 block
    conjugate-gradient solve on L's CSR (ops.ImplicitDiffusionFn), exact at any size and needing no eigenbasis
    (evals / evecs may be None).  L: sparse (V, V) for 2-D x, (B, V, V) for 3-D x, or a list of per-mesh Laplacians."""

    def __init__(self, C_inout, method='spectral'):
        super(LearnedTimeDiffusion, self).__init__()
        self.C_inout = C_inout
        self.diffusion_time = nn.Parameter(torch.Tensor(C_inout))  # (C), reference layers.py:38
        self.method = method  # one of ['spectral', 'implicit_dense']
        nn.init.constant_(self.diffusion_time, 0.0)

    def forward(self, x, L, mass, evals, evecs):
        if x.shape[-1] != self.C_inout:  # reference layers.py:51-54
            raise ValueError(
                "Tensor has wrong shape = {}. Last dim shape should have number of channels = {}".format(
                    x.shape, self.C_inout))
        if self.method == 'spectral':
            ops._require_cuda(x, mass, evals, evecs, self.diffusion_time)
            # the clamp of layers.py:48-49 happens inside the kernel, in place on the Parameter's storage
            if x.dim() == 2:
                return ops.DiffusionFn.apply(x, self.diffusion_time, mass, evals, evecs)
            return torch.stack([ops.DiffusionFn.apply(x[b], self.diffusion_time, mass[b], evals[b], evecs[b])
                                for b in range(x.shape[0])], dim=0)
        elif self.method == 'implicit_dense':
            ops._require_cuda(x, mass, self.diffusion_time)
            # the clamp of layers.py:48-49 happens inside the kernel, in place on the Parameter's storage
            if x.dim() == 2:
                lap = ops.prepare_laplacians(L, 1)[0]
                return ops.ImplicitDiffusionFn.apply(x, self.diffusion_time, mass, lap)
            laps = ops.prepare_laplacians(L, x.shape[0])
            return torch.stack([ops.ImplicitDiffusionFn.apply(x[b], self.diffusion_time, mass[b], laps[b])
                                for b in range(x.shape[0])], dim=0)
        else:
            raise ValueError("unrecognized method")


class SpatialGradientFeatures(nn.Module):
    """tanh(Re(conj(z) * A z)) with a learned complex-linear A (reference layers.py:93-130).

    Input ``vectors`` (..., V, C, 2); output (..., V, C)."""

    def __init__(self, C_inout, with_gradient_rotations=True):
        super(SpatialGradientFeatures, self).__init__()
        self.C_inout = C_inout
        self.with_gradient_rotations = with_gradient_rotations
        if self.with_gradient_rotations:
            self.A_re = nn.Linear(self.C_inout, self.C_inout, bias=False)
            self.A_im = nn.Linear(self.C_inout, self.C_inout, bias=False)
        else:
            self.A = nn.Linear(self.C_inout, self.C_inout, bias=False)

    def weights(self):
        if self.with_gradient_rotations:
            return self.A_re.weight, self.A_im.weight
        return self.A.weight, None

    def forward(self, vectors):
        ops._require_cuda(vectors)
        A_re, A_im = self.weights()
        lead = vectors.shape[:-3]
        v = vectors.reshape((-1,) + tuple(vectors.shape[-3:]))
        needs_grad = torch.is_grad_enabled() and (vectors.requires_grad or A_re.requires_grad or
                                                  (A_im is not None and A_im.requires_grad))
        outs = []
        for b in range(v.shape[0]):
            if not needs_grad:
                outs.append(ops.spatial_gradient_features_raw(v[b], A_re, A_im))
            else:
                # standalone differentiable route: dense maps through the row-GEMM kernels,
                # the per-element product/tanh as autograd glue (the block itself uses the fused path)
                g0, g1 = v[b][..., 0].contiguous(), v[b][..., 1].contiguous()
                lin = lambda w, g: ops.mlp_apply([g], [w], [None])
                if A_im is not None:
                    b_re = lin(A_re, g0) - lin(A_im, g1)
                    b_im = lin(A_re, g1) + lin(A_im, g0)
                else:
                    b_re, b_im = lin(A_re, g0), lin(A_re, g1)
                outs.append(torch.tanh(g0 * b_re + g1 * b_im))
        return torch.stack(outs, 0).reshape(lead + outs[0].shape)


FUSE_HEAD = True     # DiffusionNet: compute last_lin in the last block's MiniMLP epilogue when possible (inference)


class MiniMLP(nn.Sequential):
    """[Linear, ReLU, (Dropout .5)]* Linear, with the reference submodule names (layers.py:133-164)."""

    def __init__(self, layer_sizes, dropout=False, activation=nn.ReLU, name="miniMLP"):
        super(MiniMLP, self).__init__()
        self._fused_ok = activation is nn.ReLU
        self._uses_dropout = bool(dropout)
        self._linear_names = []
        for i in range(len(layer_sizes) - 1):
            is_last = (i + 2 == len(layer_sizes))
            if dropout and i > 0:
                self.add_module(name + "_mlp_layer_dropout_{:03d}".format(i), nn.Dropout(p=.5))
            self.add_module(name + "_mlp_layer_{:03d}".format(i), nn.Linear(layer_sizes[i], layer_sizes[i + 1]))
            self._linear_names.append(name + "_mlp_layer_{:03d}".format(i))
            if not is_last:
                self.add_module(name + "_mlp_act_{:03d}".format(i), activation())

    def linears(self):
        return [getattr(self, n) for n in self._linear_names]

    def forward_sources(self, srcs, residual=None):
        """cat(srcs, -1) -> MLP (+ residual) on one mesh, the concat never materialised."""
        lins = self.linears()
        if not self._fused_ok:
            x = torch.cat(srcs, dim=-1)
            for m in self:
                x = ops.mlp_apply([x], [m.weight], [m.bias]) if isinstance(m, nn.Linear) else m(x)
            return x if residual is None else x + residual
        drop_p = 0.5 if (self._uses_dropout and self.training) else 0.0
        return ops.mlp_apply(srcs, [l.weight for l in lins], [l.bias for l in lins], residual=residual,
                             drop_p=drop_p)

    def forward(self, x):
        ops._require_cuda(x)
        lead = x.shape[:-1]
        y = self.forward_sources([x.reshape(-1, x.shape[-1])])
        return y.reshape(lead + (y.shape[-1],))


class DiffusionNetBlock(nn.Module):
    """diffusion -> tangent-gradient features -> MiniMLP -> skip (reference layers.py:167-241)."""

    def __init__(self, C_width, mlp_hidden_dims, dropout=True, diffusion_method='spectral',
                 with_gradient_features=True, with_gradient_rotations=True):
        super(DiffusionNetBlock, self).__init__()
        self.C_width = C_width
        self.mlp_hidden_dims = mlp_hidden_dims
        self.dropout = dropout
        self.with_gradient_features = with_gradient_features
        self.with_gradient_rotations = with_gradient_rotations
        self.diffusion = LearnedTimeDiffusion(self.C_width, method=diffusion_method)
        self.MLP_C = 2 * self.C_width
        if self.with_gradient_features:
            self.gradient_features = SpatialGradientFeatures(
                self.C_width, with_gradient_rotations=self.with_gradient_rotations)
            self.MLP_C += self.C_width
        self.mlp = MiniMLP([self.MLP_C] + self.mlp_hidden_dims + [self.C_width], dropout=self.dropout)

    def _forward_mesh(self, x_in, mass, evals, evecs, gops, fused, head=None, lap=None, out=None):
        A_re = A_im = None
        if self.with_gradient_features:
            A_re, A_im = self.gradient_features.weights()
        if fused:  # inference: one C-ABI call, nothing saved (dn_block_fwd)
            lins = self.mlp.linears()
            return ops.block_forward_raw(x_in, mass, evals, evecs, gops, self.diffusion.diffusion_time, A_re, A_im,
                                         [l.weight for l in lins], [l.bias for l in lins],
                                         self.with_gradient_features, head=head, out=out)
        if head is not None:
            raise ops.HeadNotFused()
        x_diffuse = self.diffusion(x_in, lap, mass, evals, evecs)
        srcs = [x_in, x_diffuse]
        if self.with_gradient_features:
            srcs.append(ops.GradFeaturesFn.apply(x_diffuse, A_re, A_im, gops))
        return self.mlp.forward_sources(srcs, residual=x_in)   # layers.py:229-239

    def _forward_batch(self, batch, x_in):
        """Differentiable block over every mesh of a ``batch.MeshBatch`` (x_in in the batch layout): the per-mesh
        spectral diffusion runs grouped (ops.BatchedDiffusionFn), the implicit one as one solve over every (mesh,
        channel) pair (ops.BatchedImplicitDiffusionFn); the gradient features run on the block-diagonal CSR and the
        MiniMLP row-wise, each once over the whole range.  Padding rows never reach a real row."""
        if self.diffusion.method == 'implicit_dense':
            x_diffuse = ops.BatchedImplicitDiffusionFn.apply(x_in, self.diffusion.diffusion_time, batch)
        else:
            x_diffuse = ops.BatchedDiffusionFn.apply(x_in, self.diffusion.diffusion_time, batch)
        srcs = [x_in, x_diffuse]
        if self.with_gradient_features:
            A_re, A_im = self.gradient_features.weights()
            srcs.append(ops.GradFeaturesFn.apply(x_diffuse, A_re, A_im, batch.gops))
        return self.mlp.forward_sources(srcs, residual=x_in)

    def forward(self, x_in, mass, L, evals, evecs, gradX, gradY, head=None):
        """Reference signature (layers.py:200); ``head=(weight, bias)`` is this package's extension: a linear head fused
        behind the block in inference (returns the head's output; raises ops.HeadNotFused when it cannot be fused)."""
        B = x_in.shape[0]
        if x_in.shape[-1] != self.C_width:  # reference layers.py:204-207
            raise ValueError(
                "Tensor has wrong shape = {}. Last dim shape should have number of channels = {}".format(
                    x_in.shape, self.C_width))
        ops._require_cuda(x_in, mass, evals, evecs)
        implicit = self.diffusion.method == 'implicit_dense'
        if self.diffusion.method not in ('spectral', 'implicit_dense'):
            self.diffusion(x_in, L, mass, evals, evecs)   # raises like the reference would route
        # implicit: the eigenbasis is not used (k_eig = 0 gives None or empty evals / evecs); L's CSR, once per mesh
        laps = ops.prepare_laplacians(L, B) if implicit else [None] * B
        pick = lambda t, b: None if t is None else t[b]
        gops = [None] * B
        if self.with_gradient_features:
            if isinstance(gradX, (list, tuple)):           # pre-split per-mesh operators
                # an element may already be a prepared ops.GradOperators (geometry.get_operators /
                # GradOperators.from_csr): it then stands for the (gradX, gradY) pair and gradY[b] is ignored
                gys = gradY if gradY is not None else [None] * len(gradX)
                gops = [gx if isinstance(gx, ops.GradOperators) else ops.prepare_operators(gx, gy)
                        for gx, gy in zip(gradX, gys)]
            else:
                gops = ops.prepare_operators_batched(gradX, gradY)
        params_need_grad = any(p.requires_grad for p in self.parameters())
        needs_grad = torch.is_grad_enabled() and (x_in.requires_grad or params_need_grad)
        # the fused inference block is spectral: an implicit block runs the composed path (solve, features, MiniMLP)
        fused = (not implicit) and (not needs_grad) and self.mlp._fused_ok and not (self.training and self.dropout)
        if head is not None and not fused:
            raise ops.HeadNotFused()
        if fused:   # every mesh writes its slice of one fresh result: no stacking copy
            n_res = self.C_width if head is None else int(head[0].shape[0])
            res = torch.empty(B, x_in.shape[1], n_res, dtype=torch.float32, device=x_in.device)
            for b in range(B):
                self._forward_mesh(x_in[b], mass[b], pick(evals, b), pick(evecs, b), gops[b], fused, head, laps[b],
                                   out=res[b])
            return res
        outs = [self._forward_mesh(x_in[b], mass[b], pick(evals, b), pick(evecs, b), gops[b], fused, head, laps[b])
                for b in range(B)]
        return torch.stack(outs, dim=0)


def _is_slot(batch):
    from .batch import BatchSlot
    return isinstance(batch, BatchSlot)


class DiffusionNet(nn.Module):

    def __init__(self, C_in, C_out, C_width=128, N_block=4, last_activation=None, outputs_at='vertices',
                 mlp_hidden_dims=None, dropout=True, with_gradient_features=True, with_gradient_rotations=True,
                 diffusion_method='spectral'):
        """Same parameters as the reference ``DiffusionNet`` (layers.py:246-263)."""
        super(DiffusionNet, self).__init__()
        self.C_in = C_in
        self.C_out = C_out
        self.C_width = C_width
        self.N_block = N_block
        self.last_activation = last_activation
        self.outputs_at = outputs_at
        if outputs_at not in ['vertices', 'edges', 'faces', 'global_mean']:
            raise ValueError("invalid setting for outputs_at")
        if mlp_hidden_dims == None:
            mlp_hidden_dims = [C_width, C_width]
        self.mlp_hidden_dims = mlp_hidden_dims
        self.dropout = dropout
        self.diffusion_method = diffusion_method
        if diffusion_method not in ['spectral', 'implicit_dense']:
            raise ValueError("invalid setting for diffusion_method")
        self.with_gradient_features = with_gradient_features
        self.with_gradient_rotations = with_gradient_rotations

        self.first_lin = nn.Linear(C_in, C_width)
        self.last_lin = nn.Linear(C_width, C_out)
        self.blocks = []
        for i_block in range(self.N_block):
            block = DiffusionNetBlock(C_width=C_width, mlp_hidden_dims=mlp_hidden_dims, dropout=dropout,
                                      diffusion_method=diffusion_method,
                                      with_gradient_features=with_gradient_features,
                                      with_gradient_rotations=with_gradient_rotations)
            self.blocks.append(block)
            self.add_module("block_" + str(i_block), self.blocks[-1])

    def _linear(self, lin, x):
        B = x.shape[0]
        return torch.stack([ops.mlp_apply([x[b]], [lin.weight], [lin.bias]) for b in range(B)], 0)

    def forward_batch(self, batch, xs):
        """The net over a ``batch.MeshBatch`` of independent meshes in ONE launch sequence (BASELINE config 4): the
        reference's per-mesh loop (layers.py:217-222, 366-401) with every stage of every block launched once over all
        meshes.  ``xs``: list of per-mesh (V_b, C_in) features, or one tensor already in the batch layout.  Returns the
        list of per-mesh outputs.  Equal to ``[self(x_b, mass_b, ...) for b]`` (tests/test_gpu_parity.py).

        Inference runs the fused block (``dn_block_fwd_batched``).  When autograd is needed or dropout is active the
        blocks run differentiably (``DiffusionNetBlock._forward_batch``): sum or average the per-mesh losses and the
        gradients are the per-mesh gradients accumulated, input gradients reaching each ``x_b``.  Dropout masks are
        drawn over the whole batch layout, one draw per hidden layer per block.  'faces' / 'edges' outputs need the
        batch items to carry ``faces`` / ``edges``.

        An implicit_dense net needs a batch whose items carry 'L'; it runs the differentiable route in inference as well
        (batched solve, gradient features, MiniMLP)."""
        self._check_batch(batch, "forward_batch")
        if _is_slot(batch):
            raise NotImplementedError("forward_batch returns per-mesh lists, and a BatchSlot keeps no host copy of its "
                                      "layout: train on a slot with forward_batch_global_nll or forward_batch_nll")
        elems = None
        if self.outputs_at in ('edges', 'faces'):
            elems = batch.faces if self.outputs_at == 'faces' else batch.edges
            if elems is None:
                raise ValueError("forward_batch with outputs_at='{0}' needs '{0}' in every MeshBatch item".format(
                    self.outputs_at))
        x = self._forward_batch_layout(batch, xs)
        if elems is not None:
            # mean of the per-vertex outputs over each element's corners (as in forward), one gather for the batch
            y = x[elems.view(-1)].view(elems.shape + (x.shape[-1],)).mean(dim=1)
            outs = list(torch.split(y, batch.elem_counts(self.outputs_at)))
        else:
            outs = batch.unpack(x)
        if self.outputs_at == 'global_mean':
            res = []
            for b, o in enumerate(outs):
                m = batch.mass[batch.row_begin[b]:batch.row_begin[b] + batch.n_rows[b]]
                res.append((o * (m / m.sum()).unsqueeze(-1)).sum(dim=-2))
            outs = res
        if self.last_activation != None:
            outs = [self.last_activation(o) for o in outs]
        return outs

    def _forward_batch_layout(self, batch, xs):
        """forward_batch up to last_lin: the (V, C_out) per-vertex output in the batch layout (padding rows included),
        before any remap to elements, global mean or last activation."""
        x = xs if torch.is_tensor(xs) else batch.pack(xs)
        if x.shape[-1] != self.C_in:
            raise ValueError("DiffusionNet was constructed with C_in={}, but x_in has last dim={}".format(
                self.C_in, x.shape[-1]))
        needs_grad = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters()))
        dropout = any(blk.training and blk.dropout for blk in self.blocks)
        if needs_grad or dropout or self.diffusion_method == 'implicit_dense':   # the fused block is spectral
            return ops.mlp_apply([self._forward_batch_blocks(batch, x)], [self.last_lin.weight], [self.last_lin.bias])
        return self._forward_batch_fused(batch, x)

    def _check_batch(self, batch, what):
        """The batch routes run spectral nets on batches with eigenpairs, implicit nets on batches with Laplacians."""
        if self.diffusion_method == 'implicit_dense' and _is_slot(batch):
            raise NotImplementedError("{}: a BatchSlot serves spectral nets only (the implicit solve reads its "
                                      "convergence status on the host)".format(what))
        if self.diffusion_method == 'implicit_dense':
            if batch is None or not batch.has_laplacian:
                raise NotImplementedError("{}: a diffusion_method='implicit_dense' net needs a MeshBatch whose items "
                                          "carry the Laplacian 'L'".format(what))
        elif batch is not None and batch.K == 0:
            raise ValueError("{}: a spectral net needs eigenpairs, and this MeshBatch has none (k_eig = 0)".format(what))

    def _forward_batch_blocks(self, batch, x):
        """The differentiable route of forward_batch from the packed input to the last block's (V, C_width) output."""
        x = ops.mlp_apply([x], [self.first_lin.weight], [self.first_lin.bias])
        for blk in self.blocks:
            x = blk._forward_batch(batch, x)
        return x

    def _forward_batch_fused(self, batch, x):
        """Inference route of forward_batch: one dn_block_fwd_batched per block, last_lin fused behind the last one when
        it can be.  Returns the (V, C_out) output in the batch layout."""
        from . import batch as _batch
        x = ops.mlp_apply([x], [self.first_lin.weight], [self.first_lin.bias])
        fuse_head = FUSE_HEAD and ops.head_fusable(self.C_out)
        head_done = False
        for i_b, blk in enumerate(self.blocks):
            A_re = A_im = None
            if blk.with_gradient_features:
                A_re, A_im = blk.gradient_features.weights()
            lins = blk.mlp.linears()
            args = (batch, x, blk.diffusion.diffusion_time, A_re, A_im, [l.weight for l in lins], [l.bias for l in lins],
                    blk.with_gradient_features)
            if fuse_head and i_b + 1 == len(self.blocks):
                try:
                    x = _batch.block_forward_batched_raw(*args, head=(self.last_lin.weight, self.last_lin.bias))
                    head_done = True
                    break
                except ops.HeadNotFused:
                    pass
            x = _batch.block_forward_batched_raw(*args)
        if not head_done:
            x = ops.mlp_apply([x], [self.last_lin.weight], [self.last_lin.bias])
        return x

    def _head_nll(self, x, labels, elems, csr, ignore_index, label_smoothing=0.0):
        """(per-row nll, pred) of last_lin + log_softmax + nll_loss on the (V, C_width) block output ``x``, on element
        rows (the mean of the corner features) when ``elems`` is given."""
        if elems is not None:
            x = ops.element_mean(x, elems, csr)
        return ops.linear_nll(x, self.last_lin.weight, self.last_lin.bias, labels, ignore_index, label_smoothing)

    def _check_nll_head(self):
        if self.outputs_at == 'global_mean':
            raise ValueError("forward_nll / forward_batch_nll: outputs_at='global_mean' has one output per mesh: use "
                             "forward_global_nll / forward_batch_global_nll")

    def _forward_blocks(self, x_in, mass, L, evals, evecs, gradX, gradY):
        """forward's route on one mesh from x_in [N, C_in] to the last block's [N, C_width] output, differentiable."""
        mass_b = mass.unsqueeze(0)
        evals_b = evals.unsqueeze(0) if evals is not None else None
        evecs_b = evecs.unsqueeze(0) if evecs is not None else None
        Lb = [L] if L is not None else None
        gX = [gradX] if gradX is not None else None
        gY = [gradY] if gradY is not None else None
        x = self._linear(self.first_lin, x_in.unsqueeze(0))
        for b in self.blocks:
            x = b(x, mass_b, Lb, evals_b, evecs_b, gX, gY)
        return x[0]

    def forward_nll(self, x_in, mass, L=None, evals=None, evecs=None, gradX=None, gradY=None, labels=None, edges=None,
                    faces=None, ignore_index=-100, label_smoothing=0.0):
        """Training step of a segmentation / per-vertex classification net on one mesh: ``(loss, pred_labels)`` with
        ``loss = F.nll_loss(F.log_softmax(last_lin(...)), labels, ignore_index=ignore_index)`` (mean over the rows whose
        label is not ignore_index, as torch defines it) and ``pred_labels`` the argmax of the logits.  For nets whose
        ``last_activation`` is log_softmax: it is not applied here, the fused head (ops.linear_nll) replaces last_lin,
        log_softmax and nll_loss, so the (rows, C_out) logits are never formed.  The blocks run as in ``forward``.
        x_in is [N, C] (one mesh); labels int64 per vertex, or per face / edge for outputs_at 'faces' / 'edges' (the
        head then runs on the mean of each element's corner features, equal to the mean of its corner logits).
        A label outside [0, C_out) that is not ignore_index makes the loss NaN instead of a device assert.
        ``label_smoothing``: the smoothed target of ops.linear_nll (the reference's label_smoothing_log_loss)."""
        self._check_nll_head()
        if labels is None:
            raise ValueError("forward_nll needs labels")
        if x_in.dim() != 2 or x_in.shape[-1] != self.C_in:
            raise ValueError("forward_nll takes one mesh: x_in [N, {}], got {}".format(self.C_in, tuple(x_in.shape)))
        ops._require_cuda(x_in, mass, labels)
        elems = None
        if self.outputs_at in ('edges', 'faces'):
            elems = edges if self.outputs_at == 'edges' else faces
            if elems is None:
                raise ValueError("forward_nll with outputs_at='{0}' needs {0}".format(self.outputs_at))
        x = self._forward_blocks(x_in, mass, L, evals, evecs, gradX, gradY)
        nll, pred = self._head_nll(x, labels, elems, None, ignore_index, label_smoothing)
        n_valid = (labels != ignore_index).sum().to(nll.dtype)
        return nll.sum() / n_valid, pred

    def forward_batch_nll(self, batch, xs, labels, ignore_index=-100, label_smoothing=0.0):
        """forward_nll over a ``batch.MeshBatch``: ``labels`` is the list of per-mesh label tensors (per vertex, or per
        face / edge).  Returns ``(losses, preds)``: the (n_meshes,) per-mesh mean losses and the list of per-mesh
        predictions; ``losses.sum().backward()`` accumulates the gradients of the per-mesh loop.  The blocks run on
        forward_batch's differentiable route; padding rows of the batch layout carry ignore_index.

        With outputs_at='vertices', ``labels`` may instead be one (V,) int64 tensor in the batch layout (``ds.pack``,
        ``BatchSlot.pack``); the per-mesh losses are then formed on the device (the mean of the per-row nll over the
        mesh's rows whose label is not ignore_index, NaN for a mesh without one), whatever the padding rows hold, and
        ``preds`` is the (V,) prediction in the batch layout.  This is the route of a ``BatchSlot``.  With outputs_at
        'faces' / 'edges' on a ``BatchSlot`` that holds those elements, ``labels`` is one (E_cap,) int64 tensor in the
        slot's element layout (``BatchSlot.pack_elements``): the head runs on the slot's elements with its gathered
        vertex -> element CSR, and the losses are formed the same way over the element segments, whatever the padding
        elements hold; ``preds`` is (E_cap,)."""
        self._check_nll_head()
        self._check_batch(batch, "forward_batch_nll")
        if torch.is_tensor(labels):
            return self._forward_batch_nll_layout(batch, xs, labels, ignore_index, label_smoothing)
        if _is_slot(batch):
            raise NotImplementedError("forward_batch_nll on a BatchSlot takes the labels as one (V,) tensor in the "
                                      "batch layout (slot.pack(labels)): a slot keeps no host copy of its layout")
        if len(labels) != batch.n_meshes:
            raise ValueError("forward_batch_nll: {} label tensors for {} meshes".format(len(labels), batch.n_meshes))
        x = xs if torch.is_tensor(xs) else batch.pack(xs)
        if x.shape[-1] != self.C_in:
            raise ValueError("DiffusionNet was constructed with C_in={}, but x_in has last dim={}".format(
                self.C_in, x.shape[-1]))
        x = self._forward_batch_blocks(batch, x)
        elems = None
        if self.outputs_at in ('edges', 'faces'):
            elems = batch.faces if self.outputs_at == 'faces' else batch.edges
            if elems is None:
                raise ValueError("forward_batch_nll with outputs_at='{0}' needs '{0}' in every MeshBatch item".format(
                    self.outputs_at))
            counts = batch.elem_counts(self.outputs_at)
            for b, (l, n) in enumerate(zip(labels, counts)):
                if l.shape != (n,):
                    raise ValueError("forward_batch_nll: mesh {} has {} {}, got labels of shape {}".format(
                        b, n, self.outputs_at, tuple(l.shape)))
            lab = torch.cat(list(labels))
        else:
            counts = batch.n_rows
            lab = torch.full((batch.V,), ignore_index, dtype=torch.int64, device=x.device)
            for b, l in enumerate(labels):
                if l.shape != (batch.n_rows[b],):
                    raise ValueError("forward_batch_nll: mesh {} has {} vertices, got labels of shape {}".format(
                        b, batch.n_rows[b], tuple(l.shape)))
                lab[batch.row_begin[b]:batch.row_begin[b] + batch.n_rows[b]] = l
        nll, pred = self._head_nll(x, lab, elems, None, ignore_index, label_smoothing)
        if elems is not None:
            nlls, preds, labs = torch.split(nll, counts), list(torch.split(pred, counts)), labels
        else:
            nlls = [nll[r0:r0 + n] for r0, n in zip(batch.row_begin, batch.n_rows)]
            preds = [pred[r0:r0 + n] for r0, n in zip(batch.row_begin, batch.n_rows)]
            labs = labels
        losses = torch.stack([v.sum() / (l != ignore_index).sum().to(v.dtype) for v, l in zip(nlls, labs)])
        return losses, preds

    def _forward_batch_nll_layout(self, batch, xs, labels, ignore_index, label_smoothing):
        """forward_batch_nll with (V,) labels in the batch layout, or (E_cap,) labels in a slot's element layout:
        per-mesh losses from the device segment tables."""
        elems = csr = None
        if self.outputs_at != 'vertices':
            cap = batch.element_capacity.get(self.outputs_at) if _is_slot(batch) else None
            if cap is None or labels.dim() != 1 or labels.shape[0] != cap:
                err = NotImplementedError if _is_slot(batch) else ValueError
                raise err("forward_batch_nll: labels in the batch layout are per vertex; outputs_at='{0}' takes the "
                          "list of per-mesh labels of a MeshBatch, or ({1},) labels in the element layout of a "
                          "BatchSlot holding '{0}' (ds.slot(n, elements='{0}'), slot.pack_elements)".format(self.outputs_at,
                                                                               "E_cap" if cap is None else cap))
            elems, csr = getattr(batch, self.outputs_at), batch.element_csr(self.outputs_at)
            seg, n = batch.element_segments[self.outputs_at], cap
        else:
            seg, n = batch.segments, batch.V
        if labels.dtype != torch.int64 or tuple(labels.shape) != (n,):
            raise ValueError("forward_batch_nll: labels in the batch layout must be an int64 tensor of shape ({},), "
                             "got {} of shape {}".format(n, labels.dtype, tuple(labels.shape)))
        x = xs if torch.is_tensor(xs) else batch.pack(xs)
        if x.shape[-1] != self.C_in:
            raise ValueError("DiffusionNet was constructed with C_in={}, but x_in has last dim={}".format(
                self.C_in, x.shape[-1]))
        ops._require_cuda(x, labels)
        x = self._forward_batch_blocks(batch, x)
        # padding rows / elements are ignored whatever label they hold (an out-of-range label would make its row NaN)
        rows = torch.arange(n, device=x.device)
        s = seg.tile_seg.long()[rows >> 7]
        sc = s.clamp(min=0)
        real = (s >= 0) & (rows < (seg.begin.long() + seg.rows.long())[sc])
        lab = torch.where(real, labels, torch.full_like(labels, ignore_index))
        # elements: the slot's gathered CSR, never cached_element_csr (a fill rewrites the elements in place)
        nll, pred = self._head_nll(x, lab, elems, csr, ignore_index, label_smoothing)
        # per mesh: sum of nll / number of labelled rows, as the mass-weighted mean with weights (label != ignore)
        w = (lab != ignore_index).to(nll.dtype)
        losses = ops.global_mean_pool(torch.nn.functional.pad(nll[:, None], (0, 3)), w, seg)[:, 0]
        return losses, pred

    def _check_global_head(self, what):
        if self.outputs_at != 'global_mean':
            raise ValueError("{}: needs outputs_at='global_mean', the net has outputs_at='{}' (use forward_nll / "
                             "forward_batch_nll)".format(what, self.outputs_at))

    def forward_global_nll(self, x_in, mass, L=None, evals=None, evecs=None, gradX=None, gradY=None, labels=None,
                           label_smoothing=0.0, ignore_index=-100):
        """Training step of a whole-shape classifier (outputs_at='global_mean') on one mesh: ``(loss, pred)`` with
        ``loss = -sum_j t_j log_softmax(mean_mass(last_lin(...)))_j``, the reference's
        ``utils.label_smoothing_log_loss(net(...), labels, label_smoothing)`` (t: 1 - s on the label, s / (C_out - 1)
        elsewhere; s = 0 is nll_loss), and ``pred`` the 0-d argmax class.  For nets whose ``last_activation`` is
        log_softmax: it is not applied here.  The blocks run as in ``forward``; the mass-weighted mean
        (ops.global_mean_pool) then runs on the block output before the fused head (ops.linear_nll): the mean's weights
        sum to 1, so pooling before last_lin equals the reference's last_lin, mean, log_softmax.  ``labels``: an int64
        tensor of one element.  A label equal to ignore_index gives loss 0 and no gradient."""
        self._check_global_head("forward_global_nll")
        if labels is None or not torch.is_tensor(labels) or labels.dtype != torch.int64 or labels.numel() != 1:
            raise ValueError("forward_global_nll needs labels: an int64 tensor of one element")
        if x_in.dim() != 2 or x_in.shape[-1] != self.C_in:
            raise ValueError("forward_global_nll takes one mesh: x_in [N, {}], got {}".format(self.C_in,
                                                                                            tuple(x_in.shape)))
        ops._require_cuda(x_in, mass, labels)
        x = self._forward_blocks(x_in, mass, L, evals, evecs, gradX, gradY)
        pooled = ops.global_mean_pool(x, mass)
        nll, pred = ops.linear_nll(pooled, self.last_lin.weight, self.last_lin.bias, labels.reshape(1), ignore_index,
                                   label_smoothing)
        return nll[0], pred[0]

    def forward_batch_global_nll(self, batch, xs, labels, label_smoothing=0.0, ignore_index=-100):
        """forward_global_nll over a ``batch.MeshBatch``: ``labels`` an (n_meshes,) int64 tensor or a list of
        one-element int64 tensors.  Returns ``(losses, preds)``, both (n_meshes,); ``losses.sum().backward()``
        accumulates the gradients of the per-mesh loop.  The blocks run on forward_batch's differentiable route, then
        one pool over every mesh (padding rows never read) and one fused head over the n_meshes pooled rows.  An
        implicit_dense net needs a batch whose items carry 'L'."""
        self._check_global_head("forward_batch_global_nll")
        self._check_batch(batch, "forward_batch_global_nll")
        if torch.is_tensor(labels):
            lab = labels
        else:
            if any(not torch.is_tensor(l) or l.numel() != 1 for l in labels):
                raise ValueError("forward_batch_global_nll: labels must be one-element tensors, one per mesh")
            lab = torch.cat([l.reshape(1) for l in labels]) if len(labels) else None
        if lab is None or lab.dtype != torch.int64 or lab.shape != (batch.n_meshes,):
            raise ValueError("forward_batch_global_nll: {} meshes need {} int64 labels, got {}".format(
                batch.n_meshes, batch.n_meshes, tuple(lab.shape) if lab is not None else 0))
        x = xs if torch.is_tensor(xs) else batch.pack(xs)
        if x.shape[-1] != self.C_in:
            raise ValueError("DiffusionNet was constructed with C_in={}, but x_in has last dim={}".format(
                self.C_in, x.shape[-1]))
        ops._require_cuda(x, lab)
        x = self._forward_batch_blocks(batch, x)
        pooled = ops.global_mean_pool(x, batch.mass, batch.segments)
        return ops.linear_nll(pooled, self.last_lin.weight, self.last_lin.bias, lab, ignore_index, label_smoothing)

    def forward(self, x_in, mass, L=None, evals=None, evecs=None, gradX=None, gradY=None, edges=None, faces=None):
        """[N,C] or [B,N,C] in, [N,C_out] or [B,N,C_out] out (reference layers.py:314-407)."""
        if x_in.shape[-1] != self.C_in:
            raise ValueError("DiffusionNet was constructed with C_in={}, but x_in has last dim={}".format(
                self.C_in, x_in.shape[-1]))
        if len(x_in.shape) not in (2, 3):
            raise ValueError("x_in should be tensor with shape [N,C] or [B,N,C]")
        ops._require_cuda(x_in, mass)
        if len(x_in.shape) == 2:
            appended_batch_dim = True
            x_in = x_in.unsqueeze(0)
            mass = mass.unsqueeze(0)
            if evals != None: evals = evals.unsqueeze(0)
            if evecs != None: evecs = evecs.unsqueeze(0)
            # sparse operators stay un-batched: wrapping them in 1-element lists keeps the user's
            # tensor objects (and the CSR prepared from them) alive across blocks and epochs
            if L is not None: L = [L]
            if gradX != None: gradX = [gradX]
            if gradY != None: gradY = [gradY]
            if edges != None: edges = edges.unsqueeze(0)
            if faces != None: faces = faces.unsqueeze(0)
        else:
            appended_batch_dim = False

        x = self._linear(self.first_lin, x_in)
        # last_lin rides in the last block's MiniMLP epilogue when it can (inference, <= 8 outputs, fused tensor-core chain):
        # the C_width-wide output of the last block is then never written (SURVEY.md 8f-1)
        fuse_head = FUSE_HEAD and len(self.blocks) > 0 and ops.head_fusable(self.C_out) and not torch.is_grad_enabled()
        for i_b, b in enumerate(self.blocks):
            if fuse_head and i_b + 1 == len(self.blocks):
                try:
                    x = b(x, mass, L, evals, evecs, gradX, gradY, head=(self.last_lin.weight, self.last_lin.bias))
                    break
                except ops.HeadNotFused:
                    fuse_head = False
            x = b(x, mass, L, evals, evecs, gradX, gradY)
        if not fuse_head:
            x = self._linear(self.last_lin, x)

        # remap to edges / faces / global mean: callers' side of the hot path (SURVEY.md 8f row 1)
        if self.outputs_at in ('edges', 'faces'):
            # mean of the per-vertex outputs over each element's corners
            elems = edges if self.outputs_at == 'edges' else faces
            x_out = torch.stack([x[b][elems[b]].mean(dim=1) for b in range(x.shape[0])], dim=0)
        elif self.outputs_at == 'global_mean':
            # area-weighted mean (discretisation invariant)
            w = mass / mass.sum(dim=-1, keepdim=True)
            x_out = (x * w.unsqueeze(-1)).sum(dim=-2)
        else:
            x_out = x

        if self.last_activation != None:
            x_out = self.last_activation(x_out)
        if appended_batch_dim:
            x_out = x_out.squeeze(0)
        return x_out
