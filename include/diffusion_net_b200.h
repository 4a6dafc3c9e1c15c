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

#ifdef __cplusplus
}
#endif
#endif /* DIFFUSION_NET_B200_H */
