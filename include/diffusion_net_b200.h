/*
 * diffusion_net_b200 -- C ABI of the H100-native (sm_90a) DiffusionNetBlock hot path.
 *
 * The reference (nmwsharp/diffusion-net) is pure Python and has no FFI layer; its
 * boundary is the module API of src/diffusion_net/layers.py plus the operator
 * tuple of geometry.get_operators (SURVEY.md section 8b).  Each entry point below
 * replaces one reference function on that path and is what a reference-side ctypes
 * binding would call (INTEGRATION.md shows the stub).  Conventions:
 *
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless a
 *     name ends in _host; all float data is fp32, row-major, densely packed unless
 *     a leading dimension is given;
 *   - the caller allocates every output and the workspace (dn_workspace_bytes);
 *   - kernels are enqueued on `stream` (a cudaStream_t) and never synchronise;
 *   - return 0 on success, <0 for a DN_ERR_* argument/support error, >0 for a
 *     cudaError_t raised at launch; dn_error_string() explains either;
 *   - no global mutable state: calls on different streams are independent.
 *
 * `engine` selects the arithmetic of the dense contractions:
 *   DN_ENGINE_SIMT  exact fp32 FFMA (debug / gold-on-device, any shape)
 *   DN_ENGINE_TC3X  wgmma tensor cores, error-compensated 3xTF32 (fp32-grade,
 *                   the default product path; <=1e-5 relative vs the reference)
 *   DN_ENGINE_TC1X  wgmma single-pass TF32 (fast, ~5e-4 relative)
 *   DN_ENGINE_BF16  wgmma single-pass bf16 (fp32 accumulate; ~1e-2 relative; layers up to
 *                   128 wide chain on chip, a 256-wide layer runs as its own launch).  Tensors stay fp32 in HBM.
 */
#ifndef DIFFUSION_NET_B200_H
#define DIFFUSION_NET_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DN_ABI_VERSION 5

typedef void* dn_stream_t; /* cudaStream_t */

enum dn_status {
  DN_OK = 0,
  DN_ERR_INVALID_ARGUMENT = -1, /* null pointer, negative size, mismatched dims   */
  DN_ERR_UNSUPPORTED = -2,      /* shape/engine combination not implemented        */
  DN_ERR_WORKSPACE = -3,        /* workspace too small (see dn_workspace_bytes)    */
  DN_ERR_NOT_SM100 = -4         /* tensor-core engine requested on a non-sm_90 GPU */
};

enum dn_engine { DN_ENGINE_SIMT = 0, DN_ENGINE_TC3X = 1, DN_ENGINE_TC1X = 2, DN_ENGINE_BF16 = 3 };

/* Shared-pattern CSR form of the (gradX, gradY) pair.  The reference hands over two
 * coalesced COO tensors with identical, row-sorted sparsity (Re/Im of one complex
 * matrix, geometry.py:381-382; utils.py:50-55).  vals holds (gx, gy) interleaved. */
struct dn_patches;
typedef struct dn_csr {
  const int32_t* rowptr; /* V+1 */
  const int32_t* colidx; /* nnz */
  const float* vals;     /* 2*nnz: gx0, gy0, gx1, gy1, ... */
  int64_t nnz;
  const struct dn_patches* patches; /* optional (NULL): locality structure for the gather kernel, see below */
} dn_csr;

/* Optional locality structure over a dn_csr, built once per mesh (dn_patch_build, host side) for operators that
 * stay resident.  The rows are grouped into patches of graph-adjacent vertices; the fused gradient-features
 * kernel then stages the distinct neighbour rows of a patch in shared memory once (coalesced) and gathers from
 * there, instead of re-fetching every neighbour row through L1/L2 for every vertex that touches it.  Results are
 * bit-identical to the unpatched kernel (same entries, same order, same arithmetic).  The struct lives in host
 * memory like dn_csr; the arrays are device arrays. */
typedef struct dn_patches {
  int32_t n_patches;
  int32_t max_src;         /* largest number of distinct source rows of any patch (sizes the shared memory) */
  const int32_t* tgt_ptr;  /* n_patches+1: the rows of patch p are tgt[tgt_ptr[p] .. tgt_ptr[p+1])           */
  const int32_t* tgt;      /* V: row ids in patch order, every row exactly once                              */
  const int32_t* src_ptr;  /* n_patches+1                                                                    */
  const int32_t* src_rows; /* distinct column ids (= gathered rows) of each patch                            */
  const int32_t* ent_ptr;  /* V+1: the entries of row tgt[i] are [ent_ptr[i], ent_ptr[i+1]) of lcol / vals   */
  const uint8_t* lcol;     /* nnz: index into the patch's src_rows                                           */
  const float* vals;       /* 2*nnz: (gx, gy) in patch order                                                 */
} dn_patches;

/* Parameters of one DiffusionNetBlock, named as in the reference state_dict
 * (layers.py:38, 110-113, 150-155).  nn.Linear layout: weight[n_out][n_in]. */
typedef struct dn_block_params {
  float* diffusion_time;     /* (C)   in/out: overwritten with max(t, 1e-8), layers.py:48-49 */
  const float* A_re;         /* (C,C) gradient_features.A_re.weight, or .A.weight when !rotations */
  const float* A_im;         /* (C,C) gradient_features.A_im.weight, NULL when !rotations        */
  int with_gradient_features;
  int with_gradient_rotations;
  int n_mlp_layers;          /* number of Linear layers in the MiniMLP (reference default 3)      */
  const float* const* mlp_weight_host; /* host array [n_mlp_layers] of device pointers            */
  const float* const* mlp_bias_host;   /* host array [n_mlp_layers] of device pointers            */
  const int* mlp_dims_host;  /* host array [n_mlp_layers+1]: 3C (or 2C), hidden..., C             */
} dn_block_params;

int dn_abi_version(void);
const char* dn_error_string(int code);
/* sm count / compute capability (major*10+minor) / opt-in shared memory per block of `device`. */
int dn_device_query(int device, int* sm_count, int* cc, int64_t* smem_optin_bytes);

/* Number of kernels this library has launched so far in this process (monotonic; bench.py
 * differences it around the timed region). */
int64_t dn_kernel_launch_count(void);

/* Bytes of scratch any call below needs for (V, K, C); 256-byte aligned base required. */
int64_t dn_workspace_bytes(int64_t V, int K, int C);

/* Operator prep: row-sorted COO (int64 rows/cols as in utils.py:55) -> dn_csr arrays.
 * vy may be NULL (single matrix; gy written as 0). */
int dn_csr_from_coo(const int64_t* rows, const int64_t* cols, const float* vx, const float* vy,
                    int64_t nnz, int64_t V, int32_t* rowptr, int32_t* colidx, float* vals,
                    dn_stream_t stream);

/* HOST-side operator prep (every pointer here is a HOST pointer): greedy breadth-first clustering of the CSR
 * pattern into patches of at most max_targets rows whose distinct columns number at most max_src (<= 256).
 * Outputs (caller-allocated): tgt_ptr, src_ptr (V+1 each: worst case one patch per row), tgt (V), src_rows (nnz),
 * ent_ptr (V+1), lcol (nnz), perm (nnz: patch-order entry -> CSR entry, for permuting vals), max_src_out (1).
 * Returns the number of patches, or a negative DN_ERR_* (a row longer than max_src is DN_ERR_UNSUPPORTED). */
int64_t dn_patch_build(int64_t V, const int32_t* rowptr_host, const int32_t* colidx_host, int max_targets,
                       int max_src, int32_t* tgt_ptr_host, int32_t* tgt_host, int32_t* src_ptr_host,
                       int32_t* src_rows_host, int32_t* ent_ptr_host, uint8_t* lcol_host, int32_t* perm_host,
                       int32_t* max_src_out_host);

/* Operator prep from the reference's on-disk cache (geometry.py:548-568 stores gradX/gradY as scipy CSC; the
 * read side is geometry.py:494-519): a CSC matrix is the CSR of its transpose, so the cache arrays are `in`
 * verbatim and this call produces the forward CSR (columns sorted inside every row, deterministic).
 * `in` and the outputs describe square V x V matrices; workspace needs 4*V bytes. */
int dn_csr_transpose(const dn_csr* in, int64_t V, int32_t* rowptr_out, int32_t* colidx_out,
                     float* vals_out, void* workspace, int64_t ws_bytes, dn_stream_t stream);

/* geometry.py:600-628 compute_hks: out(V,S)[v,s] = sum_k exp(-evals[k]*scales[s]) * evecs(V,K)[v,k]^2. */
int dn_compute_hks(const float* evals, const float* evecs, const float* scales, int64_t V, int K,
                   int S, float* out, dn_stream_t stream);

/* geometry.py:572-583 to_basis: out(K,C) = basis(V,K)^T @ (values(V,C) * massvec(V)[:,None]).
 * massvec may be NULL (no weighting; used by the backward pass). */
int dn_to_basis(const float* values, const float* basis, const float* massvec, int64_t V, int K,
                int C, float* out, void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream);

/* geometry.py:586-598 from_basis (real branch): out(V,C) = basis(V,K) @ values(K,C).
 * row_scale (V) optional: out rows multiplied by it (mass, backward pass). */
int dn_from_basis(const float* values, const float* basis, const float* row_scale, int64_t V, int K,
                  int C, float* out, void* workspace, int64_t ws_bytes, int engine,
                  dn_stream_t stream);

/* layers.py:44-67 LearnedTimeDiffusion.forward, method='spectral'.
 * time (C) is clamped in place (layers.py:48-49).  x_spec_out (K,C) optional: the
 * un-scaled spectral coefficients, saved for the backward pass. */
int dn_learned_time_diffusion_fwd(const float* x, const float* mass, const float* evals,
                                  const float* evecs, float* time, int64_t V, int K, int C,
                                  float* x_diffuse, float* x_spec_out, void* workspace,
                                  int64_t ws_bytes, int engine, dn_stream_t stream);

/* Backward of the above w.r.t. x and time (mass/evals/evecs are data, SURVEY.md 8a).
 * grad_time (C) is ACCUMULATED into (+=).  */
int dn_learned_time_diffusion_bwd(const float* grad_out, const float* mass, const float* evals,
                                  const float* evecs, const float* time, const float* x_spec,
                                  int64_t V, int K, int C, float* grad_x, float* grad_time,
                                  void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream);

/* layers.py:216-223: out(V,C,2) with out[v,c,0] = (gradX @ x)[v,c], out[v,c,1] = (gradY @ x)[v,c]. */
int dn_grad_spmm(const dn_csr* grad, const float* x, int64_t V, int C, float* out,
                 dn_stream_t stream);

/* layers.py:117-130 SpatialGradientFeatures.forward on vectors(V,C,2) -> out(V,C). */
int dn_spatial_gradient_features_fwd(const float* vectors, const float* A_re, const float* A_im,
                                     int with_gradient_rotations, int64_t V, int C, float* out,
                                     void* workspace, int64_t ws_bytes, int engine,
                                     dn_stream_t stream);

/* layers.py:216-226 fused: features(V,C) = SpatialGradientFeatures(stack(gradX@x, gradY@x)).
 * The dense maps are applied before the sparse gradient (P = x A_re^T, Q = x A_im^T; the two
 * operators commute by linearity), so the (V,C,2) tensor is never materialised.
 * pq_out (V,2C) optional: P|Q saved for the backward pass (workspace used if NULL). */
int dn_gradient_features_fwd(const dn_csr* grad, const float* x_diffuse, const float* A_re,
                             const float* A_im, int with_gradient_rotations, int64_t V, int C,
                             float* features, float* pq_out, void* workspace, int64_t ws_bytes,
                             int engine, dn_stream_t stream);

/* Backward of dn_gradient_features_fwd.  grad_t is the CSR of the TRANSPOSED pattern
 * (same (gx,gy) values permuted).  grad_x is written; grad_A_re / grad_A_im are ACCUMULATED. */
int dn_gradient_features_bwd(const dn_csr* grad, const dn_csr* grad_t, const float* grad_features,
                             const float* x_diffuse, const float* pq, const float* features,
                             const float* A_re, const float* A_im, int with_gradient_rotations,
                             int64_t V, int C, float* grad_x, float* grad_A_re, float* grad_A_im,
                             void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream);

/* Generic fused affine chain over vertex rows (MiniMLP layers.py:133-164, first_lin/last_lin
 * layers.py:366,373, and the block's cat+MLP+skip layers.py:229-239):
 *   h_0 = concat_s src[s](V, width[s]);  h_{l+1} = act_l(h_l @ W_l^T + b_l) (* dropmask_l);
 *   out = h_L (+ residual).
 * ReLU after every layer but the last.  hidden_out[l] (optional, l < L-1) receives h_{l+1}
 * (post-activation, post-mask) for the backward pass; drop_mask[l] (optional) is a (V, dims[l+1])
 * multiplier applied after the activation (training-mode Dropout(p=.5), layers.py:143-147). */
int dn_mini_mlp_fwd(const float* const* src_host, const int* src_width_host, int nsrc,
                    const float* const* weight_host, const float* const* bias_host,
                    const int* dims_host, int n_layers, const float* const* drop_mask_host,
                    const float* residual, int64_t V, float* const* hidden_out_host, float* out,
                    void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream);

/* Backward of dn_mini_mlp_fwd.  hidden[l] = h_{l+1} saved by the forward.  grad_src[s] written
 * (residual gradient is NOT added here); grad_weight / grad_bias ACCUMULATED. */
int dn_mini_mlp_bwd(const float* grad_out, const float* const* src_host, const int* src_width_host,
                    int nsrc, const float* const* weight_host, const int* dims_host, int n_layers,
                    const float* const* hidden_host, const float* const* drop_mask_host, int64_t V,
                    float* const* grad_src_host, float* const* grad_weight_host,
                    float* const* grad_bias_host, void* workspace, int64_t ws_bytes, int engine,
                    dn_stream_t stream);

/* layers.py:200-241 DiffusionNetBlock.forward for one mesh (eval mode: no dropout, nothing
 * saved).  L is unused by the spectral method and is not passed. */
int dn_block_fwd(const float* x_in, const float* mass, const float* evals, const float* evecs,
                 const dn_csr* grad, const dn_block_params* params, int64_t V, int K, int C,
                 float* out, void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream);

/* Profiling hook: the same launch sequence as dn_block_fwd with CUDA events recorded on `stream` between its stages;
 * SYNCHRONISES on the last event and writes DN_PROFILE_STAGES host floats (milliseconds):
 *   [0] to_basis (split-V partials)  [1] partial reduction + exp(-lambda t) scale when it is a separate launch
 *   (SIMT engine; 0 on the tensor-core path, where it is part of [2])  [2] weight split/pack (+ reduction and scale)
 *   [3] from_basis (+ [P|Q]) chain   [4] sparse gradient gather + inner product + tanh   [5] MiniMLP chain + skip
 * (bench.py reports each stage's roofline from these).  Not for use inside CUDA-graph capture. */
#define DN_PROFILE_STAGES 6
int dn_block_fwd_profile(const float* x_in, const float* mass, const float* evals, const float* evecs,
                         const dn_csr* grad, const dn_block_params* params, int64_t V, int K, int C,
                         float* out, void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream,
                         float* stage_ms_host);

/* Operator construction, the per-vertex part (SURVEY.md 8f-4): geometry.py:198-207 `edge_tangent_vectors` +
 * geometry.py:209-273 `build_grad` on the device, straight into dn_csr arrays.  `edges` is the reference's (2, E) int64
 * tensor (row 0 tails, row 1 tips, any order; self loops are skipped as in :228).  Pass either `edge_tangent` (E, 2)
 * as `build_grad` receives it, or NULL with `verts` (V, 3) and `frames` (V, 3, 3) to have it computed.  Row v of the
 * result holds the entry of v itself followed / surrounded by its neighbours, columns sorted; capacity E + V entries,
 * the actual count is rowptr_out[V] (device).  fp64 2x2 solves like numpy.  workspace: 4 * V bytes. */
int dn_build_grad(const float* verts, const float* frames, const float* edge_tangent, const int64_t* edges, int64_t E,
                  int64_t V, int32_t* rowptr_out, int32_t* colidx_out, float* vals_out, void* workspace,
                  int64_t ws_bytes, dn_stream_t stream);

/* ---- operator construction for triangle meshes (geometry.py:276-392 compute_operators) --------------------------
 * The calls below are fp64 (double) throughout; `faces` is (F, 3) int64 with every index in [0, V).  They are the
 * steps of geometry.compute_operators: Laplacian + mass, frames, then the eigensolver's kernels, then dn_build_grad
 * on the Laplacian's pattern.  None synchronises. */

/* geometry.py:322-329 for meshes: the cotan Laplacian (cot = u.v / (|u x v| + 1e-10) per face corner) as int32 CSR with
 * sorted columns, the pattern of the reference's `L` (the diagonal of every referenced vertex and both directions of
 * every face edge, duplicates summed, explicit zeros kept; exactly symmetric), and the lumped mass (barycentric areas
 * + eps * mean).  Capacity of colidx_out / L_vals_out / A_vals_out: 6 F + V; the count is rowptr_out[V].
 * A_vals_out (optional, same pattern) and A_diag_out (optional, V) describe A = M^-1/2 (L + eps I) M^-1/2 =
 * A_vals + diag(A_diag); bound_out (1) receives Gershgorin's upper bound on A's spectrum; nan_out (2) the number of
 * rows of L holding a NaN and of NaN mass entries.  Deterministic.  workspace: 120 F + 12 V + 2048 bytes. */
int dn_mesh_laplacian(const double* verts, const int64_t* faces, int64_t F, int64_t V, double eps, int32_t* rowptr_out,
                      int32_t* colidx_out, double* L_vals_out, double* mass_out, double* A_vals_out, double* A_diag_out,
                      double* bound_out, int32_t* nan_out, void* workspace, int64_t ws_bytes, dn_stream_t stream);

/* geometry.py:101-177 for meshes.  normals_in NULL: unit face normals (divide-eps 1e-6) summed per vertex in face order
 * and normalised into normals_out (V, 3); a vertex whose normal is NaN (no face with a nonzero normal) is counted in
 * n_bad_out (1) -- the caller applies the reference's remedy and calls again.  normals_in given: used as they are.
 * frames_out (V, 3, 3): rows basisX, basisY, normal.  workspace (only without normals_in): 12 F + 8 V + 1024 bytes. */
int dn_vertex_frames(const double* verts, const int64_t* faces, int64_t F, int64_t V, const double* normals_in,
                     double* normals_out, double* frames_out, int32_t* n_bad_out, void* workspace, int64_t ws_bytes,
                     dn_stream_t stream);

/* Eigensolver kernels on row-major V x n fp64 blocks with leading dimension ld (>= n).
 * dn_eig_filter: one step of the scaled Chebyshev recurrence, Y_out = alpha (A Y) + beta Y + gamma Y_prev with A from
 *   dn_mesh_laplacian (Y_prev may be NULL).  Y_out must not alias Y or Y_prev.
 * dn_eig_gram: out (m x n, dense) = X^T Y; split-V partial sums in a fixed order.  workspace: 512 m n bytes.
 * dn_eig_rotate: Z = beta Z + X C, X (V x kd), C (kd x n, ldc); Z must not alias X.  beta = 0 does not read Z.
 * dn_eig_residual_norms: out[c] = || W[:, c] - theta[c] Q[:, c] ||_2.  workspace: 512 n bytes.
 * dn_eig_finalize: out (V x k, dense) = s_i M^-1/2 Y[:, cols[i]], s_i = +-1 making the largest-magnitude entry of each
 *   column positive (lowest row on ties).  workspace: 8 k bytes. */
int dn_eig_filter(const int32_t* rowptr, const int32_t* colidx, const double* A_vals, const double* A_diag, int64_t V,
                  int n, const double* Y, const double* Y_prev, int64_t ld, double alpha, double beta, double gamma,
                  double* Y_out, dn_stream_t stream);
int dn_eig_gram(const double* X, int64_t ldx, const double* Y, int64_t ldy, int64_t V, int m, int n, double* out,
                void* workspace, int64_t ws_bytes, dn_stream_t stream);
int dn_eig_rotate(const double* X, int64_t ldx, const double* C, int64_t ldc, int64_t V, int kd, int n, double beta,
                  double* Z, int64_t ldz, dn_stream_t stream);
int dn_eig_residual_norms(const double* W, int64_t ldw, const double* Q, int64_t ldq, const double* theta, int64_t V,
                          int n, double* out, void* workspace, int64_t ws_bytes, dn_stream_t stream);
int dn_eig_finalize(const double* Y, int64_t ldy, const int32_t* cols, int k, const double* mass, int64_t V, double* out,
                    void* workspace, int64_t ws_bytes, dn_stream_t stream);

/* ---- the same for a batch of small meshes, as one launch sequence ---------------------------------------------------
 * Mesh b owns rows [row_begin[b], row_begin[b + 1]) of every V x n block (V = row_begin[n_meshes]), of mass / A_diag
 * and of one block-diagonal CSR whose column indices are batch-global.  Inside each mesh, starting at its first row,
 * rows are cut into tiles of DN_EIG_TILE_ROWS (what one CTA of a row-parallel kernel owns) and into slices of
 * DN_EIG_SLICE_ROWS (what one partial sum of a reduction over rows covers); the partial sums of a mesh are added in
 * slice order.  So no tile or slice spans two meshes, and a mesh's results do not depend on which other meshes share the
 * batch or on its position in it.  All arrays are device int32, built by the caller; the kernels trust them. */
#define DN_EIG_TILE_ROWS 64
#define DN_EIG_SLICE_ROWS 1024
typedef struct dn_eig_batch {
  int32_t n_meshes;
  int32_t n_tiles;                /* sum over meshes of ceil(V_b / DN_EIG_TILE_ROWS)                    */
  int32_t n_slices;               /* sum over meshes of ceil(V_b / DN_EIG_SLICE_ROWS)                   */
  const int32_t* row_begin;       /* [n_meshes + 1]                                                     */
  const int32_t* tile_mesh;       /* [n_tiles]: mesh of every tile                                      */
  const int32_t* tile_begin;      /* [n_meshes + 1]: the tiles of mesh b are [begin[b], begin[b + 1])   */
  const int32_t* slice_mesh;      /* [n_slices]                                                         */
  const int32_t* slice_begin;     /* [n_meshes + 1]                                                     */
} dn_eig_batch;

/* dn_mesh_laplacian on the union of n_meshes meshes: `verts` (V, 3) is their concatenation, `faces` (F, 3) index the
 * union (each mesh's faces offset by its row_begin, every face inside its own mesh -- the caller checks), row_begin is
 * device int32 [n_meshes + 1].  The outputs are the union's (block-diagonal CSR, batch-global columns), and the rows of
 * every mesh are bitwise what dn_mesh_laplacian gives for that mesh alone: the mass shift eps * mean(mass_b),
 * bound_out[b] and nan_out[2 b], nan_out[2 b + 1] are kept per mesh (bound_out: n_meshes doubles, nan_out: 2 n_meshes
 * ints).  Capacities and workspace as for dn_mesh_laplacian with the union's F and V. */
int dn_mesh_laplacian_batched(const double* verts, const int64_t* faces, int64_t F, int64_t V, int n_meshes,
                              const int32_t* row_begin, double eps, int32_t* rowptr_out, int32_t* colidx_out,
                              double* L_vals_out, double* mass_out, double* A_vals_out, double* A_diag_out,
                              double* bound_out, int32_t* nan_out, void* workspace, int64_t ws_bytes, dn_stream_t stream);

/* The eigensolver's kernels over such a batch; blocks are row-major V x n with leading dimension ld as above.
 * `active` (device int32 [n_meshes], may be NULL = all): nothing of a mesh with active[b] == 0 is read or written, in
 * the blocks or in the per-mesh outputs.  Reductions use no atomics: results are bitwise reproducible.
 * filter: Y_out = alpha[b] (A Y) + beta[b] Y + gamma[b] Y_prev on the rows of mesh b; alpha, beta, gamma are device
 *   arrays of n_meshes doubles; Y_prev may be NULL; Y_out must not alias Y or Y_prev.
 * gram: out[b] (m x n, dense; out is (n_meshes, m, n)) = X_b^T Y_b.  workspace: 8 n_slices m n bytes.
 * rotate: Z_b = beta Z_b + X_b C[b], X (V x kd), C (n_meshes, kd, n) dense; Z must not alias X.
 * residual_norms: out[b][c] = || W_b[:, c] - theta[b][c] Q_b[:, c] ||_2; theta and out are (n_meshes, n).
 *   workspace: 8 n_slices n bytes.
 * finalize: out (V x k, dense) rows of mesh b = s_bi M^-1/2 Y_b[:, cols[b][i]], cols (n_meshes, k) device int32, with
 *   dn_eig_finalize's sign rule inside each mesh.  workspace: 8 n_meshes k bytes. */
int dn_eig_filter_batched(const int32_t* rowptr, const int32_t* colidx, const double* A_vals, const double* A_diag,
                          const dn_eig_batch* batch, int n, const double* Y, const double* Y_prev, int64_t ld,
                          const double* alpha, const double* beta, const double* gamma, const int32_t* active,
                          double* Y_out, dn_stream_t stream);
int dn_eig_gram_batched(const double* X, int64_t ldx, const double* Y, int64_t ldy, const dn_eig_batch* batch, int m, int n,
                        const int32_t* active, double* out, void* workspace, int64_t ws_bytes, dn_stream_t stream);
int dn_eig_rotate_batched(const double* X, int64_t ldx, const double* C, const dn_eig_batch* batch, int kd, int n,
                          double beta, const int32_t* active, double* Z, int64_t ldz, dn_stream_t stream);
int dn_eig_residual_norms_batched(const double* W, int64_t ldw, const double* Q, int64_t ldq, const double* theta,
                                  const dn_eig_batch* batch, int n, const int32_t* active, double* out, void* workspace,
                                  int64_t ws_bytes, dn_stream_t stream);
int dn_eig_finalize_batched(const double* Y, int64_t ldy, const int32_t* cols, int k, const double* mass,
                            const dn_eig_batch* batch, double* out, void* workspace, int64_t ws_bytes, dn_stream_t stream);

/* ---- implicit diffusion (layers.py:69-84, method='implicit_dense') -------------------------------------------------
 * Per channel c: x_diffuse[:, c] = (M + t_c L)^-1 M x[:, c], solved at any size by a Jacobi-preconditioned block
 * conjugate gradient over the C columns (preconditioner m_v + t_c L_vv), with each column's own step lengths, instead of
 * the reference's dense (B, C, V, V) Cholesky.  `L` is the cotan Laplacian as a dn_csr built by dn_csr_from_coo with
 * vy = NULL (the gy half is ignored); it is used as given (symmetric positive semi-definite, as get_operators returns
 * it) and promoted to fp64 like `mass`.  The solver state and every reduction are fp64 SIMT on every device: there is
 * no `engine` argument.  One cooperative launch per call; reductions run in a fixed order without atomics, so results
 * are bitwise reproducible on a given device.  C <= 256 (DN_ERR_UNSUPPORTED above).
 *
 * Convergence is decided on the device, per column: column c stops (its solution is final) once
 * ||r_c||_2 <= rtol ||b_c||_2 (b = M x forward, b = grad_out backward).  `status` (device, 2 + 2C doubles) receives
 * [0] the number of columns that did not converge within max_iter iterations, [1] the largest iteration count,
 * [2 + c] the iterations of column c, [2 + C + c] its final ||r_c|| / ||b_c|| (0 when b_c = 0).  When [0] > 0 the
 * outputs are not written (grad_time is not accumulated); the caller reads `status` to find out.
 * Non-finite data gives NaN, at once: a column whose b_c is not finite, or whose p.q, alpha, r.r or r.z turns
 * non-finite (an inf in the data, a NaN in L), stops with a NaN result: that column of x_diffuse (grad_x) is NaN and
 * grad_time[c] becomes NaN; [2 + c] holds its iterations and [2 + C + c] is NaN.  It does not count in [0].
 *   fwd: time (C) is clamped in place (layers.py:48-49) whether or not the solve converges, as the reference clamps
 *        before solving.
 *   bwd: with A_c = M + t_c L and w_c = A_c^-1 grad_out[:, c]: grad_x = M w, grad_time[c] += -sum_v w[v][c] (L x_diffuse)[v][c]
 *        (ACCUMULATED, fixed order).  `time` is the clamped time the forward left; `x_diffuse` the forward's output.
 * Workspace: dn_implicit_diffusion_workspace_bytes(V, C) (about 32 V C bytes). */
int64_t dn_implicit_diffusion_workspace_bytes(int64_t V, int C);
int dn_implicit_diffusion_fwd(const dn_csr* L, const float* x, const float* mass, float* time, int64_t V, int C,
                              double rtol, int max_iter, float* x_diffuse, double* status, void* workspace,
                              int64_t ws_bytes, dn_stream_t stream);
int dn_implicit_diffusion_bwd(const dn_csr* L, const float* grad_out, const float* mass, const float* time,
                              const float* x_diffuse, int64_t V, int C, double rtol, int max_iter, float* grad_x,
                              float* grad_time, double* status, void* workspace, int64_t ws_bytes, dn_stream_t stream);

/* ---- functional maps (experiments/functional_correspondence/fmaps_model.py:11-40) ----------------------------------
 * A = F_hat, B = G_hat (n x d, the spectral features of shapes x and y), D[i][j] = (evals_x[j] - evals_y[i])^2.  Row i of
 * the functional map C (n x n) solves
 *   S_i c_i = A b_i,   S_i = A A^T + lambda diag(D[i, :]),   b_i = B[i, :]^T,   C[i, :] = c_i^T.
 * One CTA per row forms A A^T and A b_i in fp64 from the exactly promoted fp32 inputs (each a sum over d in increasing
 * order), adds the regulariser, factors S_i by an fp64 Cholesky in shared memory and writes the solution in fp32.
 * 1 <= n <= 128 (DN_ERR_UNSUPPORTED above, before any work is enqueued), any d >= 1, lambda >= 0.  There is no
 * `engine` argument: the arithmetic is fp64 SIMT on every device.
 * A row whose S_i has a non-positive (or NaN) pivot is written as NaN and the call goes on: nothing is read back on the
 * host, so the call can be captured in a CUDA graph.  (The reference's torch.inverse raises on a singular system.)
 *   fwd: 1 launch.
 *   bwd: 2 launches.  With g_i = grad_C[i, :]^T and w_i = S_i^-1 g_i (S_i re-factored, c_i re-solved in fp64):
 *        grad_B = W A,  grad_A = W^T B - sum_i (w_i c_i^T + c_i w_i^T) A  (W has rows w_i^T), OVERWRITTEN, every sum in a
 *        fixed order without atomics (two calls give bitwise-equal results).  No gradient reaches the eigenvalues or
 *        lambda.  Workspace: 16 n^2 bytes.  Rows of a singular S_i make the gradients NaN. */
int dn_fmap_solve_fwd(const float* A, const float* B, const float* evals_x, const float* evals_y, int n, int d,
                      double lambda, float* C, dn_stream_t stream);
int dn_fmap_solve_bwd(const float* A, const float* B, const float* evals_x, const float* evals_y, int n, int d,
                      double lambda, const float* grad_C, float* grad_A, float* grad_B, void* workspace,
                      int64_t ws_bytes, dn_stream_t stream);

/* Exact 1-nearest neighbour (geometry.find_knn(source, target, k=1), functional_correspondence.py:194-196):
 * out_index[s] = argmin_t sum_k (source[s][k] - target[t][k])^2 over the rows of target (Vt x n), n <= 128
 * (DN_ERR_UNSUPPORTED above, and for Vt >= 2^31).  The distance of each pair is one fp32 FMA chain over k in increasing
 * order, in the difference form (no |q|^2 + |t|^2 - 2 q.t expansion, no tensor cores); the Vs x Vt distance matrix is
 * never formed.  Ties go to the lowest target index; a source row whose distances are all NaN or +inf gets index 0.  The
 * result is deterministic and does not depend on the device.  1 launch, or 2 when Vs is too small to fill the GPU and
 * the targets are split into ranges; the workspace (dn_nearest_neighbor_workspace_bytes, 0 when not split) holds the
 * per-range partials. */
int64_t dn_nearest_neighbor_workspace_bytes(int64_t Vs, int64_t Vt, int n);
int dn_nearest_neighbor(const float* source, int64_t Vs, const float* target, int64_t Vt, int n, int64_t* out_index,
                        void* workspace, int64_t ws_bytes, dn_stream_t stream);

/* ---- batches of independent meshes in one launch sequence (BASELINE config 4; SURVEY.md 8e) -------------------
 * The reference loops over the batch dimension with one set of operators per mesh (layers.py:217-222; a DataLoader
 * of batch_size None in every experiment).  Here a batch is ONE vertex range: mesh b occupies rows
 * [row_begin[b], row_begin[b] + n_rows[b]) of every (V, .) array; row_begin[b] is a multiple of 128 (a 128-row tile
 * never straddles two meshes); rows in the padding between meshes carry mass 0, basis 0 and no CSR entries; the CSR
 * is block diagonal with batch-global column indices; evals is (n_meshes, K).  Every per-vertex stage (gather,
 * MiniMLP) then runs as one launch over the whole range, and the per-mesh spectral stages run grouped:
 * to_basis CTAs never cross a mesh (tb_rows), the spectral multiplier is packed once per mesh and the from_basis chain
 * picks its weights per tile (tile_mesh).  Device arrays are built once per batch from dn_mesh_batch_plan's output. */
typedef struct dn_mesh_batch {
  int32_t n_meshes;
  int32_t n_tb_ctas;             /* CTAs of the grouped to_basis launch (<= 1024)                             */
  const int32_t* tile_mesh;      /* device [V / 128]: mesh of every 128-row tile                              */
  const int32_t* tb_rows;        /* device [2 * n_tb_ctas]: row range [begin, end) of each to_basis CTA       */
  const int32_t* mesh_cta_begin; /* device [n_meshes + 1]: the CTAs of mesh b are [begin[b], begin[b+1])      */
} dn_mesh_batch;

/* HOST-side planner (all pointers are HOST pointers): lays n_meshes meshes of n_rows_host[b] vertices out in one
 * row range (each start rounded up to 128) and splits them over about sm_count to_basis CTAs.
 * Outputs (caller-allocated): row_begin_host [n_meshes + 1] (last = padded total V), tile_mesh_host [V / 128],
 * tb_rows_host [2 * 1024], mesh_cta_begin_host [n_meshes + 1].  Returns the number of to_basis CTAs or DN_ERR_*. */
int dn_mesh_batch_plan(int n_meshes, const int32_t* n_rows_host, int sm_count, int32_t* row_begin_host,
                       int32_t* tile_mesh_host, int32_t* tb_rows_host, int32_t* mesh_cta_begin_host);

/* A batch gathered from a device-resident dataset (batch.MeshDataset): the dataset holds every mesh's arrays back to
 * back (no padding, int64 offsets), and one call writes any batch of its meshes in the layout above.  Each "part" is one
 * array, copied mesh by mesh in units (a row, a CSR entry, a face, a mesh) of `width` elements.  `table` (device int64
 * [n_meshes][n_ranges][4]) names for batch mesh b and range r the tuple (src_begin, dst_begin, n, n_dst) in units:
 * units [0, n) of the mesh come from src units [src_begin, src_begin + n) and go to dst units [dst_begin, ...); units
 * [n, n_dst) are padding; only the first min(n, n_dst) source units are written when n > n_dst.  The ops:
 *   DN_GATHER_COPY:    4-byte words copied as they are; padding written as 0 (fp32 rows, interleaved CSR values,
 *                      eigenvalues, and int64 data as word pairs);
 *   DN_GATHER_ADD_I32, DN_GATHER_ADD_I64: int32 / int64 entries plus the mesh's offset o = dst_begin of range
 *                      `offset_range`; padding written as o + n of that range (mesh-local column and vertex indices
 *                      rebased to batch rows, and mesh-local row pointers rebased to batch entries, padding rows empty).
 * Every batch value must fit the element type (the caller checks: a batch is int32-indexed).  `max_units` is the largest
 * n_dst of the part's range over the meshes; it sizes the grid only.  Parts must not overlap in dst.  One launch for up
 * to DN_GATHER_MAX_PARTS parts and 65535 meshes; nothing is read back, so the call never waits on the device. */
#define DN_GATHER_MAX_PARTS 16
enum dn_gather_op { DN_GATHER_COPY = 0, DN_GATHER_ADD_I32 = 1, DN_GATHER_ADD_I64 = 2 };
typedef struct dn_gather_part {
  const void* src;       /* dataset array                                     */
  void* dst;             /* batch array                                       */
  int32_t op;            /* dn_gather_op                                      */
  int32_t width;         /* elements per unit (4-byte words for DN_GATHER_COPY) */
  int32_t range;         /* range of `table` that places this array's units   */
  int32_t offset_range;  /* ADD ops: range whose dst_begin is added           */
  int64_t max_units;
} dn_gather_part;
int dn_batch_gather(const dn_gather_part* parts_host, int n_parts, const int64_t* table, int n_ranges, int n_meshes,
                    dn_stream_t stream);

/* DEVICE-side planner of a fixed-capacity batch slot (batch.BatchSlot): the layout above for the n_meshes dataset
 * meshes ids[b] (device int64), planned in one single-CTA launch that reads nothing back, so it can be captured in a
 * CUDA graph and replayed with new ids.  dataset_sizes (device int64 [n_dataset][4]) gives every dataset mesh's
 * (rows, first row, gradient entries, first entry) in the dataset's concatenated arrays.  The slot's row range is
 * V_cap rows (a multiple of 128) and its to_basis grid n_tb_ctas CTAs; both stay fixed while the batch changes.
 * Written (device arrays of dn_slot_plan):
 *   row_begin, tile_mesh, tb_rows, mesh_cta_begin: dn_mesh_batch_plan's for the same meshes (sm_count as there) on the
 *     batch's rows; tiles past the batch's end map to the last mesh, and CTAs from mesh_cta_begin[n_meshes] up to
 *     n_tb_ctas get the empty range [V, V) (V = row_begin[n_meshes]): no mesh's CTA range holds them;
 *   seg_begin, seg_rows, tile_seg: one global-mean segment per mesh (tile_seg -1 past the batch's end);
 *   table [2 n_meshes][n_ranges][4]: dn_batch_gather's table.  Entry b < n_meshes is batch mesh b, with ranges
 *     0 rows, 1 meshes, 2 row pointers (n_rows + 1 per dataset mesh; the last batch mesh also writes row V), 3 gradient
 *     entries, and every other range empty.  Entry n_meshes + k is piece k of the tail: rows
 *     [V + k tail_rows, V + (k + 1) tail_rows) clipped to V_cap, written as padding (row pointers V + 1 ... V_cap equal
 *     to the batch's entry count), so a gather grid sized by tail_rows covers it;
 *   status [3]: sticky.  A fill whose ids hold an id outside [0, n_dataset) or whose rows or entries exceed V_cap or
 *     entry_cap reads nothing through its ids and is planned with every mesh empty (V = 0, every mesh one empty CTA,
 *     no gathered data), and if status[0] is 0 it records (1 = bad id / 2 = over capacity, first offending position,
 *     the id there).  The caller reads and clears it.
 * Requires 1 <= n_meshes <= 1024, V_cap a multiple of 128 below 2^31 - 256, entry_cap < 2^31,
 * min(1024, sm_count + n_meshes) <= n_tb_ctas <= 1024 (the host planner never uses more CTAs: each mesh gets at most
 * chunks_b sm_count / chunks_total + 1), n_meshes * tail_rows >= V_cap and n_ranges >= 4; DN_ERR_INVALID_ARGUMENT
 * otherwise, before any launch. */
typedef struct dn_slot_plan {
  int32_t* row_begin;        /* [n_meshes + 1]          */
  int32_t* tile_mesh;        /* [V_cap / 128]           */
  int32_t* tb_rows;          /* [2 * n_tb_ctas]         */
  int32_t* mesh_cta_begin;   /* [n_meshes + 1]          */
  int32_t* seg_begin;        /* [n_meshes]              */
  int32_t* seg_rows;         /* [n_meshes]              */
  int32_t* tile_seg;         /* [V_cap / 128]           */
  int64_t* table;            /* [2 n_meshes][n_ranges][4] */
  int64_t* status;           /* [3]                     */
} dn_slot_plan;
int dn_mesh_batch_plan_device(const int64_t* ids, int n_meshes, const int64_t* dataset_sizes, int64_t n_dataset,
                              int sm_count, int64_t V_cap, int64_t entry_cap, int n_tb_ctas, int64_t tail_rows,
                              int n_ranges, const dn_slot_plan* out_host, dn_stream_t stream);

/* The same planner for a slot that also holds element kinds (faces, edges: outputs_at 'faces' / 'edges' training).
 * dataset_sizes is [n_dataset][size_cols], size_cols >= 4 + 2 n_kinds: the four columns above, then for kind q the
 * dataset mesh's (elements, first element) at columns 4 + 2q and 5 + 2q.  With n_kinds = 0 and size_cols = 4 this is
 * dn_mesh_batch_plan_device, bitwise.  For every kind, in the same launch:
 *   begin [n_meshes + 1], count [n_meshes]: batch mesh b's elements are [begin[b], begin[b] + count[b]) of the slot's
 *     element layout of `capacity` elements; every begin is a multiple of 128 (so an element tile belongs to one mesh),
 *     begin[n_meshes] is the padded total; tile_seg [capacity / 128]: the mesh of every element tile, -1 past the
 *     total.  (begin, count, tile_seg) are one global-mean segment per mesh over the element layout;
 *   table range `range` of entry b: (first element, begin[b], count[b], padded count) for the corners, which
 *     dn_batch_gather offsets by (and pads with) dst_begin of range `corner_range` = the mesh's first row, so every
 *     padding corner names a row of the slot; tail piece entries pad [begin[n_meshes], capacity) in pieces of `tail`
 *     elements, their corners row 0;
 *   table range `csr_range` of entry b: (k * first element, c_b, k count[b], k count[b]) for the mesh's vertex -> element
 *     CSR entries, c_b the sum of k count over the earlier meshes: no gaps between meshes, so with the row pointers
 *     gathered through range 2 (offset range csr_range) no vertex's entries reach a padding element.
 * The kinds' element totals join the capacity check: a batch whose padded elements of a kind exceed its capacity is
 * over capacity (status 2) and planned empty like any invalid fill.  Requires, besides the above: 0 <= n_kinds <=
 * DN_SLOT_MAX_ELEMENT_KINDS, every capacity a positive multiple of 128 with k capacity < 2^31, k >= 1, n_meshes tail >=
 * capacity, and corner_range, every range and every csr_range distinct, in [4, n_ranges). */
#define DN_SLOT_MAX_ELEMENT_KINDS 2
typedef struct dn_slot_elements {
  int64_t capacity;          /* elements of the slot's element layout   */
  int64_t tail;              /* elements per tail piece                  */
  int32_t k;                 /* corners per element: 3 faces, 2 edges    */
  int32_t range;             /* table range of the elements (corners)    */
  int32_t csr_range;         /* table range of the vertex -> element CSR */
  int32_t* begin;            /* [n_meshes + 1]                           */
  int32_t* count;            /* [n_meshes]                               */
  int32_t* tile_seg;         /* [capacity / 128]                         */
} dn_slot_elements;
int dn_mesh_batch_plan_device_elements(const int64_t* ids, int n_meshes, const int64_t* dataset_sizes, int size_cols,
                                       int64_t n_dataset, int sm_count, int64_t V_cap, int64_t entry_cap,
                                       int n_tb_ctas, int64_t tail_rows, int n_ranges, const dn_slot_plan* out_host,
                                       const dn_slot_elements* elements_host, int n_kinds, int corner_range,
                                       dn_stream_t stream);

/* Per-mesh rotations of the (V, 3) rows of a batch laid out as above (the reference's random_rotate_points on every
 * mesh of a batch or slot): out[v] = x[v] @ R[tile_mesh[v / 128]], R device (n_meshes, 3, 3) row-major, each output
 * one fp32 FMA chain x0 R[0][j], + x1 R[1][j], + x2 R[2][j].  tile_mesh is the batch's (device, V / 128 entries), so
 * a host-planned batch and a device-planned slot are served alike; padding rows, 0 in x, stay 0.  A row whose tile
 * names no mesh in [0, n_meshes) is written as NaN.  x and out may be the same array.  V a positive multiple of 128.
 * 1 launch; nothing is read back. */
int dn_rotate_rows(const float* x, int64_t V, const float* R, int n_meshes, const int32_t* tile_mesh, float* out,
                   dn_stream_t stream);

/* dn_block_fwd over a batch laid out as above (V = padded total, a multiple of 128).  Tensor-core engines only
 * (DN_ERR_UNSUPPORTED otherwise and for shapes outside the fused kernels' envelope: the caller loops over meshes). */
int dn_block_fwd_batched(const float* x_in, const float* mass, const float* evals, const float* evecs,
                         const dn_csr* grad, const dn_block_params* params, const dn_mesh_batch* batch, int64_t V,
                         int K, int C, float* out, void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream);

/* dn_learned_time_diffusion_fwd / _bwd over a batch laid out as above, for training over many small meshes in one
 * launch sequence (3 launches forward, 4 backward, whatever the mesh count; C = 256 adds one to_basis launch to each).
 * evals is (n_meshes, K); x_spec (n_meshes, K, C) holds each mesh's unscaled coefficients Phi_b^T M_b x_b.
 *   fwd: time (C) is clamped in place (layers.py:48-49); x_diffuse is 0 on padding rows; x_spec_out optional.
 *   bwd: grad_x = M * Phi_b (exp(-lambda_b t) * Phi_b^T g_b) on the rows of mesh b and exactly 0 on padding rows;
 *        grad_time[c] += sum_b sum_k G_b[k][c] * (-lambda_bk) * exp(-lambda_bk t_c) * x_spec_b[k][c], G_b = Phi_b^T g_b,
 *        in a fixed summation order (deterministic).  `time` is the clamped time the forward left; it is only read.
 * Same envelope as dn_block_fwd_batched: tensor-core engines only, V % 128 == 0, and a from_basis layer the fused chain
 * takes; anything else (the SIMT engine included: batches have no SIMT route) is DN_ERR_UNSUPPORTED before any work is
 * enqueued.  Workspace: dn_workspace_bytes(V, K, C) plus, per mesh, one packed K x C matrix and one fp32 K x C sum:
 * n_meshes * (8 * C * (K rounded up to 16) + 4 * K * C + 512) bytes. */
int dn_learned_time_diffusion_fwd_batched(const float* x, const float* mass, const float* evals, const float* evecs,
                                          float* time, const dn_mesh_batch* batch, int64_t V, int K, int C,
                                          float* x_diffuse, float* x_spec_out, void* workspace, int64_t ws_bytes,
                                          int engine, dn_stream_t stream);
int dn_learned_time_diffusion_bwd_batched(const float* grad_out, const float* mass, const float* evals,
                                          const float* evecs, const float* time, const float* x_spec,
                                          const dn_mesh_batch* batch, int64_t V, int K, int C, float* grad_x,
                                          float* grad_time, void* workspace, int64_t ws_bytes, int engine,
                                          dn_stream_t stream);

/* The spectral projection over a batch laid out as above (the functional-map head of many shapes at once):
 *   dn_to_basis_batched:   out (n_meshes, K, C), out[b] = Phi_b^T M_b F_b: the grouped to_basis partials (tb_rows), then
 *                          each mesh's CTA partials summed in CTA order.  mass may be NULL (no weighting).  2 launches
 *                          (3 for C = 256).
 *   dn_from_basis_batched: out (V, C), the rows of mesh b = row_scale (.) Phi_b G_b with G = values (n_meshes, K, C),
 *                          exactly 0 on padding rows (the basis is 0 there).  Every G_b is packed in one launch and the
 *                          from_basis chain picks G_b per 128-row tile.  row_scale may be NULL.  2 launches.
 * The launch counts do not depend on n_meshes.  Envelope and workspace as dn_learned_time_diffusion_fwd_batched's
 * (tensor-core engines only; the SIMT engine is DN_ERR_UNSUPPORTED before any work is enqueued). */
int dn_to_basis_batched(const float* values, const float* basis, const float* mass, const dn_mesh_batch* batch,
                        int64_t V, int K, int C, float* out, void* workspace, int64_t ws_bytes, int engine,
                        dn_stream_t stream);
int dn_from_basis_batched(const float* values, const float* basis, const float* row_scale, const dn_mesh_batch* batch,
                          int64_t V, int K, int C, float* out, void* workspace, int64_t ws_bytes, int engine,
                          dn_stream_t stream);

/* dn_implicit_diffusion_fwd / _bwd (implicit diffusion, above) over a batch laid out as above, in one cooperative
 * launch whatever the mesh count: for every mesh b and channel c (a "pair"), the rows of mesh b in column c of
 * x_diffuse are (M_b + t_c L_b)^-1 M_b x_bc.  `L` is the batch's block-diagonal Laplacian (dn_csr with batch-global
 * column indices, L at even positions of vals as above); `mass` (V) and x (V, C) are in the batch layout, V the padded
 * total (a positive multiple of 128).  From `batch` only n_meshes and tile_mesh are read; `mesh_rows` (device,
 * 2 n_meshes int32) holds the rows [begin, end) of mesh b, begin a multiple of 128 and the tiles of [begin, end) marked
 * b in tile_mesh.  Every pair has its own step lengths, convergence test, freezing and NaN state, exactly as a column
 * of the single-mesh call, so one mesh's iterations do not change another's.  Every sum over a mesh's rows is a sum of
 * 32-row partials in a fixed order: results are bitwise reproducible and do not depend on the device's size.
 * Padding rows (not in any [begin, end)) are written as exact zeros (x_diffuse, grad_x).
 * `status` (device, 2 + 2 P doubles, P = n_meshes C, pair p = b C + c): [0] the number of pairs that did not converge
 * within max_iter iterations, [1] the largest iteration count, [2 + p] the iterations of pair p, [2 + P + p] its final
 * ||r|| / ||b|| (0 when b = 0, NaN for a non-finite pair).  When [0] > 0 no output is written and grad_time is not
 * accumulated.  time is clamped in place by the forward as above.
 *   bwd: grad_x = M_b w_bc on the rows of mesh b; grad_time[c] += -sum_b sum_v w_bc[v] (L_b x_diffuse_bc)[v], the meshes
 *        added in mesh order (NaN when any pair of channel c is non-finite).
 * Workspace: dn_implicit_diffusion_workspace_bytes_batched(V, C, n_meshes) (about 32 V C bytes). */
int64_t dn_implicit_diffusion_workspace_bytes_batched(int64_t V, int C, int n_meshes);
int dn_implicit_diffusion_fwd_batched(const dn_csr* L, const float* x, const float* mass, float* time,
                                      const dn_mesh_batch* batch, const int32_t* mesh_rows, int64_t V, int C,
                                      double rtol, int max_iter, float* x_diffuse, double* status, void* workspace,
                                      int64_t ws_bytes, dn_stream_t stream);
int dn_implicit_diffusion_bwd_batched(const dn_csr* L, const float* grad_out, const float* mass, const float* time,
                                      const float* x_diffuse, const dn_mesh_batch* batch,
                                      const int32_t* mesh_rows, int64_t V, int C, double rtol, int max_iter,
                                      float* grad_x, float* grad_time, double* status, void* workspace,
                                      int64_t ws_bytes, dn_stream_t stream);

/* ---- functional maps over a pair batch ------------------------------------------------------------------------------
 * S shapes and P ordered pairs (x_p, y_p) of shape indices (self-pairs, repeats and unused shapes allowed).  The spectral
 * features are one stack F: shape s at F + s * ld_shape, n x d with row stride d (ld_shape >= n d, so a padded (S, K, d)
 * projection is read in place); evals (S, ld_evals), the first n of each row used.  pair_x, pair_y are device int32 [P]
 * with every index in [0, S) (the caller checks).  C is (P, n, n).  Pair p computes exactly what dn_fmap_solve_fwd /
 * _bwd compute for A = F_{x_p}, B = F_{y_p}, evals_x = evals[x_p], evals_y = evals[y_p]: bitwise the same C, NaN rows
 * where S_i is singular.  1 <= n <= 128, P < 65536, S < 65536 (DN_ERR_UNSUPPORTED above); no host read, so both calls
 * capture in a CUDA graph.
 *   fwd: 1 launch, one CTA per (row, pair).
 *   bwd: 3 launches whatever P is: the per-(row, pair) re-solve, the per-pair dA_p, dB_p (fp32, as dn_fmap_solve_bwd
 *        writes them), then grad_F[s] = sum over the entries of shape s in the role list of dA_p (role x) or dB_p
 *        (role y), summed in fp32 from 0 in list order, with no atomics.  role_begin (device int32 [S + 1]) and role_list
 *        (device int32 [2 P], entry 2 p + role, role 0 = x, 1 = y) form a CSR from shape to entries; each shape's entries
 *        are in increasing order (increasing p, the x role before the y role of a self-pair).  The n x d block of every
 *        shape in grad_F (same layout as F) is OVERWRITTEN, exactly 0 for a shape in no pair; the rest of each ld_shape
 *        stride is not written.  Workspace: dn_fmap_solve_batched_workspace_bytes(P, n, d), 16 n^2 P + 8 n d P bytes
 *        (each part rounded up to 256). */
int64_t dn_fmap_solve_batched_workspace_bytes(int n_pairs, int n, int d);
int dn_fmap_solve_fwd_batched(const float* F, int64_t ld_shape, const float* evals, int64_t ld_evals, int n_shapes,
                              const int32_t* pair_x, const int32_t* pair_y, int n_pairs, int n, int d, double lambda,
                              float* C, dn_stream_t stream);
int dn_fmap_solve_bwd_batched(const float* F, int64_t ld_shape, const float* evals, int64_t ld_evals, int n_shapes,
                              const int32_t* pair_x, const int32_t* pair_y, int n_pairs, const int32_t* role_begin,
                              const int32_t* role_list, int n, int d, double lambda, const float* grad_C,
                              float* grad_F, void* workspace, int64_t ws_bytes, dn_stream_t stream);

/* The pointwise maps of a pair batch: for every pair, out_index[o_p + v] (o_p = sum_{q<p} V_{y_q}) is the index of the
 * nearest row of T_p = Phi_{x_p}[:, :n] C_p^T to row v of Phi_{y_p}[:, :n], bitwise what dn_from_basis on the SIMT engine
 * followed by dn_nearest_neighbor give for that pair (ties to the lowest index).  Phi is `evecs` in a batch layout
 * (shape s at rows row_begin_host[s] .. + n_rows_host[s], row stride ld_evecs >= n); C is (P, n, n) dense; the pair and
 * row arrays are HOST int32 arrays (indices checked here).  T_p goes to the workspace, entries formed as one fmaf chain in
 * increasing k from 0 (the SIMT kernel's order).  Pairs run in chunks of at most 64 pairs whose T rows total at most
 * 2^24 floats (a chunk holds at least one pair); per chunk 2 launches, or 3 when the chunk's source rows are too few to
 * fill the GPU and the targets are split into ranges.  Workspace (dn_fmap_pointwise_map_batched_workspace_bytes): the
 * largest chunk's T (4 NP sum V_x bytes, NP = n rounded up to a power of two >= 4; at most 64 MiB unless one pair is
 * larger) plus its split partials (8 splits sum V_y bytes, splits <= 16). */
int64_t dn_fmap_pointwise_map_batched_workspace_bytes(int n, int n_pairs, const int32_t* pair_x_host,
                                                      const int32_t* pair_y_host, const int32_t* row_begin_host,
                                                      const int32_t* n_rows_host, int n_shapes);
int dn_fmap_pointwise_map_batched(const float* C, int n, const float* evecs, int64_t ld_evecs,
                                  const int32_t* row_begin_host, const int32_t* n_rows_host, int n_shapes,
                                  const int32_t* pair_x_host, const int32_t* pair_y_host, int n_pairs,
                                  int64_t* out_index, void* workspace, int64_t ws_bytes, dn_stream_t stream);

/* Ground-truth functional maps of shape pairs (faust_scape_dataset.py:186-190, the functional-map model's training
 * target): for pair p with table entry (x, y) = pair_table[pair_ids[p]], A = Phi_x[vts_x, :n] and B = Phi_y[vts_y, :n]
 * (m rows each), C_gt[p] = X^T with X = argmin ||A X - B||, solved from the normal equations A^T A X = A^T B.
 *   evecs (dataset rows, row stride ld_evecs >= n): the eigenvectors of every shape, back to back;
 *   vts_rows (device int64): the correspondences of every shape as evecs rows (already rebased to the dataset), shape s
 *     owning vts_rows[vts_begin[s] .. vts_begin[s + 1]) (vts_begin device int64 [n_shapes + 1]);
 *   pair_table (device int64 [n_table][2]) the allowed ordered pairs, pair_ids (device int64 [n_pairs]) the drawn ones.
 * The caller checks that every table pair's shapes have equal correspondence counts m <= max_m and that every row is in
 * evecs.  A and B are gathered straight from evecs in shared memory (never materialised); A^T A and A^T B are summed in
 * fp64 over fixed 512-row chunks, each chunk's partial one FMA chain in row order, the partials added in chunk order;
 * A^T A is factored by the fp64 Cholesky of the functional-map solve and the n columns solved; C_gt is written in fp32.
 * A pair's result depends on its own rows only: bitwise the same alone or among other pairs, at any position.
 * 2 launches; the grid is sized from max_m and n_pairs, not from the drawn pairs, and nothing is read back, so the
 * call captures in a CUDA graph and replays for any draw.
 * Where the reference's least squares returns a solution, a pair whose A^T A has a pivot at or below 1e-10 of its
 * diagonal entry gets NaN in all of C_gt[p]: a rank-deficient system (fewer than n distinct rows, for instance), and
 * also a full-rank but near-singular one (a column of A within about 1e-5 radians of the span of the others, so
 * roughly kappa(A) >= 1e5), whose fp64 normal equations would lose every digit of fp32 accuracy.  So does a pair
 * index outside [0, n_table).  Either sets the sticky status (device int64 [3]) when status[0] is 0: (1 = bad pair
 * index / 2 = singular, position p, pair_ids[p]).  The caller reads and clears it.
 * 1 <= n <= 128 (DN_ERR_UNSUPPORTED above), n_pairs <= 65535, max_m < 2^31.
 * Workspace: dn_fmap_ground_truth_workspace_bytes(n_pairs, n, max_m), each part rounded up to 256 bytes:
 *   16 n^2 n_pairs max(1, ceil(max_m / 512)) + 8 n^2 n_pairs bytes. */
int64_t dn_fmap_ground_truth_workspace_bytes(int n_pairs, int n, int64_t max_m);
int dn_fmap_ground_truth(const float* evecs, int64_t ld_evecs, int n, const int64_t* vts_rows,
                         const int64_t* vts_begin, int64_t n_shapes, const int64_t* pair_table, int64_t n_table,
                         const int64_t* pair_ids, int n_pairs, int64_t max_m, float* C_gt, int64_t* status,
                         void* workspace, int64_t ws_bytes, dn_stream_t stream);

/* Linear head fused behind a block (SURVEY.md 8f-1): `DiffusionNet.last_lin` (layers.py:366-370 -- the nn.Linear applied
 * to the last block's output) computed in the epilogue of that block's MiniMLP chain, in exact fp32, so that the
 * C_width-wide block output is never written: out_head[v][o] = bias[o] + sum_c weight[o][c] * block_out[v][c]. */
typedef struct dn_head {
  const float* weight;  /* (n_out, C) nn.Linear layout */
  const float* bias;    /* (n_out) or NULL             */
  int32_t n_out;        /* 1..8                        */
  float* out;           /* (V, n_out), row stride ld_out floats */
  int64_t ld_out;
} dn_head;

/* dn_block_fwd / dn_block_fwd_batched with options: `batch` may be NULL (one mesh), `head` may be NULL.  With a head, `out`
 * (the block output) may be NULL; DN_ERR_UNSUPPORTED when the MiniMLP does not run on the fused tensor-core chain (the
 * caller then applies the head as a separate layer). */
int dn_block_fwd_ex(const float* x_in, const float* mass, const float* evals, const float* evecs, const dn_csr* grad,
                    const dn_block_params* params, const dn_mesh_batch* batch, const dn_head* head, int64_t V, int K,
                    int C, float* out, void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream);

/* ---- fused classification head: last_lin -> log_softmax -> nll_loss (SURVEY.md 8f-1, training) -------------------
 * The head of the segmentation and per-vertex classification experiments (last_lin, last_activation = log_softmax,
 * F.nll_loss) as one op on R rows: z = x weight^T + bias (x (R, C), weight (n_class, C) nn.Linear layout, bias (n_class)
 * or NULL, labels int64 (R)), and per row
 *   nll[r] = lse[r] - z[r][labels[r]],  lse[r] = log sum_n exp z[r][n],  argmax[r] = argmax_n z[r][n]
 * with ties to the lowest class.  The (R, n_class) logits and log-probabilities are never written to memory: every CTA
 * owns 128 rows and streams the weights in 128-class tiles through wgmma, keeping a running (max, sum-exp), the label's
 * logit and the running argmax per row.  Any n_class >= 1; C a multiple of 16 up to 256; x and weight 16-byte aligned
 * (DN_ERR_UNSUPPORTED otherwise).  Tensor-core engines only (the arithmetic of the logits is the engine's: 3xTF32,
 * TF32 or bf16; the softmax is fp32): DN_ENGINE_SIMT is DN_ERR_UNSUPPORTED, and so is every refusal, before any work is
 * enqueued.  Rows with labels[r] == ignore_index get nll = 0 and no gradient.  A label outside [0, n_class) that is not
 * ignore_index gives nll = NaN on that row and a NaN gradient, and the call goes on (torch's nll_loss asserts on the
 * device instead); a row with a non-finite logit gets lse = nll = NaN.  Nothing is read back on the host, so both
 * calls capture in a CUDA graph.
 *   fwd: 1 launch.  nll, lse (R floats) and argmax (R int64) are OVERWRITTEN; lse is what the backward needs.
 *   bwd: 3 launches whatever R and n_class are.  With dZ = grad_nll[r] (softmax(z[r]) - onehot(labels[r])), the logits
 *        recomputed from the saved lse: grad_x = dZ weight (R, C), grad_weight = dZ^T x (n_class, C) and
 *        grad_bias = sum_r dZ (n_class; may be NULL when bias is NULL), all OVERWRITTEN.  The weight and bias gradients
 *        are per-row-range partials in the workspace (dn_linear_nll_workspace_bytes(R, C, n_class)), summed in a fixed
 *        order without atomics: two calls give bitwise-equal results. */
int64_t dn_linear_nll_workspace_bytes(int64_t R, int C, int n_class);
int dn_linear_nll_fwd(const float* x, const float* weight, const float* bias, const int64_t* labels, int64_t R, int C,
                      int n_class, int64_t ignore_index, float* nll, int64_t* argmax, float* lse, int engine,
                      dn_stream_t stream);
int dn_linear_nll_bwd(const float* x, const float* weight, const float* bias, const int64_t* labels, const float* lse,
                      const float* grad_nll, int64_t R, int C, int n_class, int64_t ignore_index, float* grad_x,
                      float* grad_weight, float* grad_bias, void* workspace, int64_t ws_bytes, int engine,
                      dn_stream_t stream);

/* The head with label smoothing: dn_linear_nll_fwd / _bwd with the smoothed target of the reference's
 * utils.label_smoothing_log_loss (the classification experiment's loss).  With s = label_smoothing and
 * s' = s / (n_class - 1), the target is t_j = 1 - s on the label and s' on every other class, and per row
 *   nll[r] = -sum_j t_j log_softmax(z[r])_j,   dZ = grad_nll[r] (softmax(z[r]) - t)
 * (torch's cross_entropy(label_smoothing = e) is this target with s = e (n_class - 1) / n_class).  The forward keeps one
 * more running quantity per row, sum_j (max - z_j), so the smoothed sum of log-probabilities needs no cancellation.
 * Everything else (shapes, engines, ignore_index and out-of-range labels, workspace, launch counts, determinism) is as
 * for dn_linear_nll_fwd / _bwd; at s = 0 the results are theirs bit for bit.  s outside [0, 1] (or NaN), or s > 0 with
 * n_class < 2, is DN_ERR_INVALID_ARGUMENT before anything is enqueued. */
int dn_linear_nll_ls_fwd(const float* x, const float* weight, const float* bias, const int64_t* labels, int64_t R,
                         int C, int n_class, int64_t ignore_index, float* nll, int64_t* argmax, float* lse, int engine,
                         dn_stream_t stream, float label_smoothing);
int dn_linear_nll_ls_bwd(const float* x, const float* weight, const float* bias, const int64_t* labels,
                         const float* lse, const float* grad_nll, int64_t R, int C, int n_class, int64_t ignore_index,
                         float* grad_x, float* grad_weight, float* grad_bias, void* workspace, int64_t ws_bytes,
                         int engine, dn_stream_t stream, float label_smoothing);

/* Element rows of the head for outputs_at = 'faces' / 'edges' (layers.py:394-398 takes the mean of the corner logits;
 * the mean commutes with last_lin, so the head runs on the mean of the corner features instead).
 *   fwd: out[e][c] = (sum_j x[elems[e][j]][c]) / k over the k corners in order, x (V, C), elems int64 (E, k) with every
 *        index in [0, V) (the caller checks); out (E, C) OVERWRITTEN.  1 launch (none when E = 0).
 *   bwd: grad_x[v][c] = sum over the entries of vertex v of grad_out[e][c] / k, through a vertex -> element CSR
 *        (rowptr int32 (V + 1), entries int32: the element of each corner slot, each vertex's entries in increasing
 *        element order) built once per element array; grad_x (V, C) OVERWRITTEN, in a fixed order without atomics.
 *        1 launch. */
int dn_element_mean_fwd(const float* x, int64_t V, int C, const int64_t* elems, int64_t E, int k, float* out,
                        dn_stream_t stream);
int dn_element_mean_bwd(const float* grad_out, int64_t E, int C, const int32_t* rowptr, const int32_t* entries,
                        int64_t V, int k, float* grad_x, dn_stream_t stream);

/* Rows of the head for outputs_at = 'global_mean': the mass-weighted mean of each mesh's features (layers.py:393-397
 * weights the per-vertex logits by mass / sum(mass); the weights sum to 1, so the mean commutes with last_lin and the
 * head runs on the pooled features).  x (V, C) fp32, C a multiple of 4 up to 256, x 16-byte aligned; mass (V).  Segment b
 * is rows [seg_begin[b], seg_begin[b] + seg_rows[b]) (int32 device arrays of n_seg entries); every segment begins on a
 * 128-row tile and every tile lies in at most one segment, named by tile_seg[t] (int32, ceil(V / 128) entries, -1 for
 * a tile of no segment): a dn_mesh_batch layout with one segment per mesh, or one segment [0, V) for one mesh.  Rows
 * outside every segment (a batch's padding rows) are never read.  The tables live on the device and nothing is read
 * back, so both calls capture in a CUDA graph.
 *   fwd: pooled[b][c] = sum_{v in b} mass[v] x[v][c] / M_b, M_b = sum_{v in b} mass[v]; pooled (n_seg, C) and mass_sum
 *        (n_seg: M_b, what the backward needs) OVERWRITTEN.  2 launches whatever V, C and n_seg are: per-tile-run
 *        partials in the workspace (dn_global_mean_workspace_bytes(V, C), 16-byte aligned), then one CTA per segment
 *        sums its partials in tile order.  No atomics: two calls give bitwise-equal results.
 *   bwd: grad_x[v][c] = mass[v] / M_b grad_pooled[b][c] for v in segment b and exactly 0 on every other row; grad_x
 *        (V, C) OVERWRITTEN.  1 launch.
 * C outside the envelope, V >= 2^31 or a misaligned x, pooled, grad_pooled, grad_x or workspace is DN_ERR_UNSUPPORTED,
 * a short workspace DN_ERR_WORKSPACE, before anything is enqueued. */
int64_t dn_global_mean_workspace_bytes(int64_t V, int C);
int dn_global_mean_fwd(const float* x, const float* mass, int64_t V, int C, const int32_t* seg_begin,
                       const int32_t* seg_rows, const int32_t* tile_seg, int n_seg, float* pooled, float* mass_sum,
                       void* workspace, int64_t ws_bytes, dn_stream_t stream);
int dn_global_mean_bwd(const float* grad_pooled, const float* mass, const float* mass_sum, int64_t V, int C,
                       const int32_t* seg_begin, const int32_t* seg_rows, const int32_t* tile_seg, int n_seg,
                       float* grad_x, dn_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DIFFUSION_NET_B200_H */
