// Internal (non-ABI) declarations shared by the SIMT kernels, the wgmma kernels and the
// C-ABI glue.  Everything here is device-pointer based; no torch types anywhere in csrc/.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include "../../include/diffusion_net_b200.h"

#define DN_MAX_SRC 3
#define DN_MAX_LAYERS 8

#define DN_CUDA_TRY(expr)                          \
  do {                                             \
    cudaError_t _e = (expr);                       \
    if (_e != cudaSuccess) return (int)_e;         \
  } while (0)

extern long long g_dn_launches;   // kernels launched by this library (reported by bench.py)

#define DN_LAUNCH_CHECK()                          \
  do {                                             \
    cudaError_t _e = cudaGetLastError();           \
    if (_e != cudaSuccess) return (int)_e;         \
    ++g_dn_launches;                               \
  } while (0)

// One affine layer applied to 128-row tiles of vertices:  out = epi(A @ W^T + bias)
//   A = concat_s src[s] (layer 0) -- or the previous layer's output inside a fused chain.
struct DnLayer {
  const float* W;        // nn.Linear layout [N][K] (ldw = K) when !w_trans; [K][N] (ldw = N) when w_trans
  int64_t ldw;
  int w_trans;
  const float* W2;       // optional second block: !w_trans: output rows n >= n_split come from W2[n - n_split]
  int n_split;           //   (stacks [A_re; A_im] without a copy);  w_trans: input rows k >= n_split come from W2[k - n_split]
  const float* prepacked;  // optional: weights already in the tensor-core layout (tc_pack_layers)
  int pack_fmt;            // layout of `prepacked` (set by tc_chain_plan): 0 = 16-wide K stages of [tf32 hi | tf32 lo]
                           //   (TF32 engines); 2 = 16-wide K stages of bf16 (DN_ENGINE_BF16)
  const float* bias;     // [N] or null
  int relu;
  const float* emul;     // optional elementwise multiplier [V][N] applied after the activation
  const float* relu_mask_src;  // optional [V][N]: multiply by (src > 0)   (backward of ReLU)
  const float* row_scale;      // optional [V]: multiply rows (mass, backward of to_basis)
  const float* residual; // optional [V][N] added last (times res_scale)
  int64_t ld_res;
  float res_scale;
  float* out;            // optional [V][N] (ld_out); null => stays on chip (fused chain only)
  int64_t ld_out;
  int K, N;
  // mesh batches (layer 0 of a chain only): `prepacked` holds one packed matrix per mesh, group_stride floats apart,
  // and 128-row tile t uses matrix tile_group[t] (device array)
  const int32_t* tile_group;
  int64_t group_stride;
  // inside a fused chain (layer 2 or later): this layer reads the input of the layer before it instead of that layer's
  // output (P and Q of the gradient features both read x_diffuse)
  int sibling;
  // linear head fused behind the last layer's epilogue (DiffusionNet.last_lin, layers.py:366-370): after bias / residual the
  // N-wide row y is NOT stored (out may be null); head_out[v][o] = head_b[o] + sum_n head_w[o][n] * y[n], o < head_n <= 8,
  // exact fp32 FMAs in the output warps
  const float* head_w;
  const float* head_b;
  float* head_out;
  int64_t ld_head_out;
  int head_n;
};

// ---- the spectral multiplier exp(-lambda max(t, 1e-8)) (layers.py:48-49, 62-64) ----
// torch.clamp(t, min=1e-8): the diffusion time every spectral, implicit and write-back path uses
__device__ __forceinline__ float dn_clamp_time(float t) { return fmaxf(t, 1e-8f); }
// exp(-lambda t), the heat factor of eigenvalue lambda (also the HKS kernels' factor at scale t)
__device__ __forceinline__ float dn_heat(float lam, float t) { return expf(-(lam * t)); }
// one eigenpair's term of dL/dt: g * (-lambda) * e * x_spec with e = dn_heat(lambda, t), multiplied left to right
__device__ __forceinline__ float dn_time_grad_term(float g, float lam, float e, float x_spec) {
  return g * (-lam) * e * x_spec;
}
// x[0] + ... + x[(N - 1) * stride] as a pairwise tree: ((x0 + x1) + (x2 + x3)) + ... for N a power of two
template <int N> __device__ __forceinline__ float pairwise_sum(const float* x, int stride) {
  if constexpr (N == 1) return x[0];
  else return pairwise_sum<N / 2>(x, stride) + pairwise_sum<N / 2>(x + (N / 2) * stride, stride);
}

struct DnRowsSrc {
  const float* ptr[DN_MAX_SRC];
  int width[DN_MAX_SRC];
  int64_t ld[DN_MAX_SRC];
  int nsrc;
};

// ---- SIMT engine (dn_simt.cu) ----
int simt_rows_gemm(const DnRowsSrc& src, const DnLayer& layer, int64_t V, cudaStream_t st);
// out[i][j] (ld_out) (+)= sum_v A[v][i] * scale[v] * B[v][j];  partial sums staged in ws.
int simt_atb(const float* A, int64_t lda, int I, const float* B, int64_t ldb, int J, const float* scale,
             int64_t V, float* out, int64_t ld_out, int accumulate, float* ws, int64_t ws_floats,
             cudaStream_t st);
int simt_atb_partial_st(const float* A, int64_t lda, int I, const float* B, int64_t ldb, int J, const float* scale,
                        int64_t V, float* ws, int64_t ws_floats, int* P_out, cudaStream_t st);
// out[n] (+)= sum_v A[v][n] in a fixed order (bias gradients): one partial row per row slice in ws, then the slices
// summed in slice order.  Deterministic: no atomics.
int simt_colsum(const float* A, int64_t lda, int N, int64_t V, float* out, int accumulate, float* ws,
                int64_t ws_floats, cudaStream_t st);

// ---- shared small kernels (dn_simt.cu) ----
// S[k][c] = exp(-evals[k]*max(t[c],1e-8)) * sum_p partial[p][k][c]; optionally writes the raw sum
// (x_spec) and the clamped time back.  s_trans: write S as [c][k].
int launch_spectral_scale(const float* partial, int P, const float* evals, float* time, int K, int C,
                          float* x_spec_out, float* S_out, int clamp_writeback, cudaStream_t st);
// Sums split-V partials, each a [rows][cols] matrix, in partial order from 0 into out (row stride ld_out; accumulate:
// added to what out holds).  Without mesh_cta_begin the sum runs over partials [0, P); with it (a mesh batch, n_meshes
// meshes, P unused) mesh b sums its to_basis CTAs [mesh_cta_begin[b], mesh_cta_begin[b + 1]) into rows
// [b * rows, (b + 1) * rows) of out.
int launch_reduce_partials(const float* partial, int P, const int32_t* mesh_cta_begin, int n_meshes, int64_t rows,
                           int cols, float* out, int64_t ld_out, int accumulate, cudaStream_t st);
int launch_csr_from_coo(const int64_t* rows, const int64_t* cols, const float* vx, const float* vy,
                        int64_t nnz, int64_t V, int32_t* rowptr, int32_t* colidx, float* vals, cudaStream_t st);
int launch_compute_hks(const float* evals, const float* evecs, const float* scales, int64_t V, int K, int S,
                       float* out, cudaStream_t st);
int launch_build_grad(const float* verts, const float* frames, const float* edge_tangent, const int64_t* edges, int64_t E,
                      int64_t V, int32_t* rowptr, int32_t* colidx, float* vals, int32_t* cursor, cudaStream_t st);
int launch_csr_transpose(const dn_csr* in, int64_t V, int32_t* rowptr_t, int32_t* colidx_t, float* vals_t,
                         int32_t* cursor, cudaStream_t st);
// mesh operators (dn_geom.cu) and the eigensolver's kernels (dn_eig.cu); fp64
int64_t mesh_laplacian_ws_bytes(int64_t F, int64_t V);
int64_t vertex_frames_ws_bytes(int64_t F, int64_t V);
int launch_mesh_laplacian(const double* verts, const int64_t* faces, int64_t F, int64_t V, double eps, int32_t* rowptr,
                          int32_t* colidx, double* lvals, double* mass, double* avals, double* adiag, double* bound,
                          int32_t* nan_out, void* ws, cudaStream_t st);
int launch_vertex_frames(const double* verts, const int64_t* faces, int64_t F, int64_t V, const double* normals_in,
                         double* normals_out, double* frames, int32_t* n_bad, void* ws, cudaStream_t st);
int64_t eig_gram_ws_bytes(int64_t V, int m, int n);
int64_t eig_resid_ws_bytes(int64_t V, int n);
int launch_eig_filter(const int32_t* rowptr, const int32_t* colidx, const double* avals, const double* adiag, int64_t V,
                      int n, const double* Y, const double* Yp, int64_t ld, double alpha, double beta, double gamma,
                      double* out, cudaStream_t st);
int launch_eig_gram(const double* X, int64_t ldx, const double* Y, int64_t ldy, int64_t V, int m, int n, double* out,
                    double* ws, cudaStream_t st);
int launch_eig_rotate(const double* X, int64_t ldx, const double* Cm, int64_t ldc, int64_t V, int kd, int n, double beta,
                      double* Z, int64_t ldz, cudaStream_t st);
int launch_eig_residual_norms(const double* W, int64_t ldw, const double* Q, int64_t ldq, const double* theta, int64_t V,
                              int n, double* out, double* ws, cudaStream_t st);
int launch_eig_finalize(const double* Y, int64_t ldy, const int32_t* cols, int k, const double* mass, int64_t V,
                        double* out, double* sign_ws, cudaStream_t st);
// the same over a batch of meshes laid out by dn_eig_batch (a mesh with active[b] == 0 is skipped; active may be null)
int launch_mesh_laplacian_batched(const double* verts, const int64_t* faces, int64_t F, int64_t V, int n_meshes,
                                  const int32_t* row_begin, double eps, int32_t* rowptr, int32_t* colidx, double* lvals,
                                  double* mass, double* avals, double* adiag, double* bound, int32_t* nan_out, void* ws,
                                  cudaStream_t st);
int64_t eig_gram_batched_ws_bytes(int n_slices, int m, int n);
int64_t eig_resid_batched_ws_bytes(int n_slices, int n);
int launch_eig_filter_batched(const int32_t* rowptr, const int32_t* colidx, const double* avals, const double* adiag,
                              const dn_eig_batch* bt, int n, const double* Y, const double* Yp, int64_t ld,
                              const double* alpha, const double* beta, const double* gamma, const int32_t* active,
                              double* out, cudaStream_t st);
int launch_eig_gram_batched(const double* X, int64_t ldx, const double* Y, int64_t ldy, const dn_eig_batch* bt, int m, int n,
                            const int32_t* active, double* out, double* ws, cudaStream_t st);
int launch_eig_rotate_batched(const double* X, int64_t ldx, const double* Cm, const dn_eig_batch* bt, int kd, int n,
                              double beta, const int32_t* active, double* Z, int64_t ldz, cudaStream_t st);
int launch_eig_residual_norms_batched(const double* W, int64_t ldw, const double* Q, int64_t ldq, const double* theta,
                                      const dn_eig_batch* bt, int n, const int32_t* active, double* out, double* ws,
                                      cudaStream_t st);
int launch_eig_finalize_batched(const double* Y, int64_t ldy, const int32_t* cols, int k, const double* mass,
                                const dn_eig_batch* bt, double* out, double* sign_ws, cudaStream_t st);
// implicit diffusion (dn_implicit.cu): one cooperative block-PCG solve of (M + diag(t) (x) L) Y = b, fp64 state
int64_t implicit_ws_bytes(int64_t V, int C);
int launch_implicit_diffusion(const dn_csr* L, const float* mass, float* time, const float* rhs, const float* y,
                              int64_t V, int C, double rtol, int max_iter, int backward, float* out, float* grad_time,
                              double* status, void* ws, cudaStream_t st);
// the same over a mesh batch (dn_implicit_batch.cu): one solve per (mesh, channel) pair; mesh_rows (device,
// 2 n_meshes) holds each mesh's rows [begin, end)
int64_t implicit_batched_ws_bytes(int64_t V, int C, int n_meshes);
int launch_implicit_diffusion_batched(const dn_csr* L, const float* mass, float* time, const float* rhs, const float* y,
                                      const dn_mesh_batch* batch, const int32_t* mesh_rows, int64_t V, int C,
                                      double rtol, int max_iter, int backward, float* out, float* grad_time,
                                      double* status, void* ws, cudaStream_t st);
int launch_grad_spmm_pair(const dn_csr* g, const float* x, int64_t V, int C, float* out_vc2, cudaStream_t st);
// R-order fused features: feat = tanh(gX*Bre + gY*Bim) from gathers of xd, P, Q (pq = [P|Q], ld 2C or C).
int launch_spmm_features(const dn_csr* g, const float* xd, const float* pq, int rotations, int64_t V, int C,
                         float* feat, cudaStream_t st);
int launch_features_bwd_local(const dn_csr* g, const float* xd, const float* pq, const float* feat,
                              const float* dfeat, int rotations, int64_t V, int C, float* U /*V x 4C*/,
                              cudaStream_t st);
int launch_features_bwd_transpose(const dn_csr* gt, const float* U, int rotations, int64_t V, int C,
                                  float* dxd /*V x C*/, float* dP, float* dQ /*V x C each, leading dim ld_pq*/,
                                  int64_t ld_pq, cudaStream_t st);
int launch_deinterleave_vc2(const float* vc2, int64_t V, int C, float* g01 /*V x 2C*/, cudaStream_t st);
int launch_complex_dots_tanh(const float* g01, const float* b01, int64_t V, int C, float* out, cudaStream_t st);
int launch_spectral_bwd(const float* gs_partial, int P, const float* evals, const float* time,
                        const float* x_spec, int K, int C, float* dS /*K x C*/, float* grad_time /*+=*/,
                        cudaStream_t st);
// Time gradient of a mesh batch: grad_time[c] += sum_b sum_k G[b][k][c] * (-evals[b][k]) * E * x_spec[b][k][c] with
// E = exp(-evals[b][k] * max(time[c], 1e-8)).  Fixed summation order, no atomics: deterministic.
int launch_spectral_time_grad_batched(const float* G, const float* x_spec, const float* evals, const float* time,
                                      int n_meshes, int K, int C, float* grad_time, cudaStream_t st);

// a mesh batch gathered from a dataset (dn_batch_gather.cu); parts were checked by dn_batch_gather
int launch_batch_gather(const dn_gather_part* parts, int n_parts, const int64_t* table, int n_ranges, int n_meshes,
                        cudaStream_t st);
// a batch slot's layout planned on the device (dn_batch_plan.cu); arguments checked by dn_mesh_batch_plan_device
int launch_mesh_batch_plan_device(const int64_t* ids, int n_meshes, const int64_t* sizes, int size_cols,
                                  int64_t n_dataset, int sm_count, int64_t V_cap, int64_t entry_cap, int n_tb_ctas,
                                  int64_t tail_rows, int n_ranges, const dn_slot_plan& out,
                                  const dn_slot_elements* kinds, int n_kinds, int corner_range, cudaStream_t st);

// ---- wgmma engine (dn_tc.cu) ----
// Per-device table, filled on first use of a device: whether it runs the tensor-core kernels (sm_90, with their
// >48 KB dynamic shared memory attributes set on it) and its SM count (1 if it cannot be queried), which sizes grids
// and split-V partials.
bool tc_supported_device();
int dn_sm_count();
// `passes`: 3 = 3xTF32-grade (fp32 parity), 1 = single-pass TF32, DN_PASSES_BF16 = single-pass bf16 (DN_ENGINE_BF16)
#define DN_PASSES_BF16 16
// Whether rows_chain_kernel takes this chain: the packed-weight format it runs it with (also stored in every
// layers[i].pack_fmt), or DN_ERR_UNSUPPORTED.  Layer 0's sources are copied with 2-D TMA: each must be 16-byte
// aligned with a row stride that is a multiple of 4 floats.
int tc_chain_plan(const DnRowsSrc& src, DnLayer* layers, int n_layers, int passes);
// Fused chain of up to DN_MAX_LAYERS layers over 128- or 192-row tiles; layer 0 reads `src`.  The chain was planned
// (tc_chain_plan) on a device that runs the tensor-core kernels; layers that are not prepacked are packed into ws.
int tc_rows_chain(const DnRowsSrc& src, const DnLayer* layers, int n_layers, int64_t V, int passes, void* ws,
                  int64_t ws_bytes, cudaStream_t st);
// partial[p][k][c] for p < *P_out
// `values` may be a column slice (row stride ld_values >= C) and a partial a slice of a wider one (row stride ldp):
// C_width = 256 runs as two 128-column launches into the same [P][K][256] partials.  0 = contiguous (== C).
int tc_to_basis_partial(const float* values, const float* basis, const float* massvec, int64_t V, int K, int C,
                        float* partial, int* P_out, int passes, cudaStream_t st, int64_t ld_values = 0, int64_t ldp = 0,
                        const int32_t* cta_rows = nullptr, int n_ctas = 0);
int tc_to_basis_supported(int K, int C);
// The spectral multiplier, packed in place of layers[0]'s weight (w_trans, K = eigen count, N = channels):
//   S_b[k][n] = exp(-evals[b][k] * max(time[n], 1e-8)) * sum_{p in [p0_b, p1_b)} partial[p][k][n]
// for every mesh b < n_meshes, with [p0_b, p1_b) = [mesh_cta_begin[b], mesh_cta_begin[b + 1]) for a mesh batch (row
// tile t of layer 0 then streams matrix tile_mesh[t]) and [0, P) without one.  The clamped time is written back unless
// no_clamp_writeback is set (the backward pass reads a saved copy of the clamped time).
struct TcSpectral {
  const float* partial;
  int P;
  const float* evals;              // [n_meshes][K]
  float* time;
  int n_meshes;
  const int32_t* mesh_cta_begin;   // device [n_meshes + 1], null without a batch
  const int32_t* tile_mesh;        // device, null without a batch
  float* sum_out;                  // optional [n_meshes][K][N]: the reduced partial sums before the exp(-lambda t) scale
  int no_clamp_writeback;
  // plain: `partial` is (n_meshes, K, N) and mesh b's matrix is partial[b] as it is (no sum, no scale; evals, time,
  // mesh_cta_begin and sum_out are not read)
  int plain;
};
// bytes tc_pack_layers needs (layer 0 n_meshes times)
int64_t tc_chain_ws_bytes(const DnLayer* layers, int n_layers, int n_meshes = 1);
// one launch: pack the weights of n layers (layer 0 the spectral multiplier when sp is given) into ws and set
// layers[i].prepacked
int tc_pack_layers(DnLayer* layers, int n_layers, void* ws, int64_t ws_bytes, const TcSpectral* sp, cudaStream_t st);

// 2-D tensor map of fp32 [rows][width] with a row stride of ld floats, boxes of box_cols x box_rows and the 128-byte
// swizzle or none; false where the driver has no encoder or rejects the map.  Elements outside the tensor are
// zero-filled on loads and not written by stores.
bool encode_tensor_map_f32(CUtensorMap* m, const float* base, int64_t rows, int width, int64_t ld, int box_cols,
                           int box_rows, bool swizzle128);

// ---- fused classification head (dn_head.cu) ----
// row splits of the weight-gradient kernel and the workspace its partials need
int head_splits(int64_t R, int C, int n_class);
int64_t head_ws_bytes(int64_t R, int C, int n_class);
// label_smoothing: the reference's target (label 1 - s, every other class s / (n_class - 1)); 0 = plain NLL
int launch_linear_nll_fwd(const float* X, const float* W, const float* b, const int64_t* labels, int64_t R, int C,
                          int n_class, int64_t ignore_index, float label_smoothing, float* nll, int64_t* argmax,
                          float* lse, int passes, cudaStream_t st);
int launch_linear_nll_bwd(const float* X, const float* W, const float* b, const int64_t* labels, const float* lse,
                          const float* g, int64_t R, int C, int n_class, int64_t ignore_index, float label_smoothing,
                          float* dX, float* dW, float* db, void* ws, int passes, cudaStream_t st);
int launch_element_mean_fwd(const float* x, int C, const int64_t* elems, int64_t E, int k, float* out, cudaStream_t st);
int launch_element_mean_bwd(const float* g, int C, const int32_t* rowptr, const int32_t* ent, int64_t V, int k,
                            float* gx, cudaStream_t st);
// mass-weighted mean over segments of 128-row tiles (dn_global_mean_fwd / _bwd)
int64_t pool_ws_bytes(int64_t V, int C);
int launch_global_mean_fwd(const float* x, const float* mass, int64_t V, int C, const int32_t* begin,
                           const int32_t* rows, const int32_t* tile_seg, int n_seg, float* pooled, float* msum,
                           void* ws, cudaStream_t st);
int launch_global_mean_bwd(const float* g, const float* mass, const float* msum, int64_t V, int C,
                           const int32_t* begin, const int32_t* rows, const int32_t* tile_seg, int n_seg, float* gx,
                           cudaStream_t st);
