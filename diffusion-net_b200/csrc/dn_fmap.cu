// Functional-map head of the correspondence model (reference experiments/functional_correspondence/fmaps_model.py:11-40)
// and the exact 1-nearest-neighbour search that turns a functional map into a pointwise map
// (functional_correspondence.py:194-196).
//
// Solve.  A = F_hat, B = G_hat (n x d, fp32), D[i][j] = (evals_x[j] - evals_y[i])^2.  Row i of C solves
//   S_i c_i = A b_i,   S_i = A A^T + lambda diag(D[i, :]),   b_i = B[i, :]^T.
// One CTA per row: A A^T (lower triangle) and A b_i are formed in fp64 from the exactly promoted fp32 inputs, each entry a
// sequential sum over d in increasing order; then an in-place fp64 Cholesky of S_i in shared memory and two triangular
// solves.  A non-positive (or NaN) pivot marks the row singular: it is written as NaN, nothing is read on the host.
// Backward: launch 1 re-factors S_i and solves for c_i and w_i = S_i^-1 g_i (fp64, to the workspace); launch 2, one CTA
// per row j, forms M[j][:] = sum_i (w_i[j] c_i + c_i[j] w_i), dA[j] = sum_i w_i[j] b_i - sum_k M[j][k] a_k and
// dB[j] = sum_k w_j[k] a_k, every sum in a fixed order with no atomics.
//
// Nearest neighbour.  Each thread owns one source row, kept in registers (n padded with zeros to a power of two NP; a
// zero pad adds exactly 0), and scans target rows in increasing index through shared-memory tiles, computing
// sum_k (q_k - t_k)^2 as one fp32 fmaf chain in increasing k and keeping the first strict minimum.  The V_s x V_t
// distance matrix never exists.  When there are too few source blocks to fill the GPU the targets are split into
// contiguous ranges (grid y); the per-range (distance, index) partials are combined in range order by a second launch,
// so ties still go to the lowest target index and the result does not depend on the split.
#include "dn_fmap_common.cuh"

namespace {

using dnfm::kNnThreads;
using dnfm::kNnTileFloats;
using dnfm::kNnTargetCtas;
using dnfm::kNnMaxSplit;
using dnfm::kSolveThreads;
using dnfm::nn_np;
using dnfm::solve_smem_bytes;

// Factor S_i and solve for row i = blockIdx.x (dnfm::row_solve).
__global__ void __launch_bounds__(kSolveThreads) fmap_row_solve_kernel(
    const float* __restrict__ A, const float* __restrict__ B, const float* __restrict__ ex, const float* __restrict__ ey,
    double lambda, int n, int d, const float* __restrict__ G, float* __restrict__ C_out, double* __restrict__ Cd,
    double* __restrict__ Wd) {
  extern __shared__ double smem[];
  dnfm::row_solve(A, B, ex, ey, lambda, n, d, blockIdx.x, G, C_out, Cd, Wd, smem);
}

// Row j = blockIdx.x of dA and dB from c_i, w_i (dnfm::grad_row).
__global__ void __launch_bounds__(kSolveThreads) fmap_grad_kernel(const float* __restrict__ A,
                                                                  const float* __restrict__ B,
                                                                  const double* __restrict__ Cd,
                                                                  const double* __restrict__ Wd, int n, int d,
                                                                  float* __restrict__ dA, float* __restrict__ dB) {
  extern __shared__ double smem[];
  dnfm::grad_row(A, B, Cd, Wd, n, d, blockIdx.x, dA, dB, smem);
}

// ---- nearest neighbour --------------------------------------------------------------------------------------------
struct NnPlan {
  int np, tile, splits;
  int64_t qblocks, tiles, tiles_per_split;
};

NnPlan nn_plan(int64_t Vs, int64_t Vt, int n) {
  NnPlan p;
  p.np = nn_np(n);
  p.tile = kNnTileFloats / p.np;
  p.qblocks = (Vs + kNnThreads - 1) / kNnThreads;
  p.tiles = (Vt + p.tile - 1) / p.tile;
  int64_t s = p.qblocks > 0 ? (kNnTargetCtas + p.qblocks - 1) / p.qblocks : 1;
  s = s < 1 ? 1 : (s > kNnMaxSplit ? kNnMaxSplit : s);
  if (s > p.tiles) s = p.tiles > 0 ? p.tiles : 1;
  p.tiles_per_split = p.tiles > 0 ? (p.tiles + s - 1) / s : 1;
  p.splits = p.tiles > 0 ? (int)((p.tiles + p.tiles_per_split - 1) / p.tiles_per_split) : 1;
  return p;
}

template <int NP>
__global__ void __launch_bounds__(kNnThreads) nn_kernel(const float* __restrict__ src, int64_t Vs,
                                                        const float* __restrict__ tgt, int64_t Vt, int n,
                                                        int64_t tiles_per_split, int64_t* __restrict__ out,
                                                        float* __restrict__ part_d, int32_t* __restrict__ part_i) {
  constexpr int TT = kNnTileFloats / NP;
  __shared__ __align__(16) float ts[kNnTileFloats];
  const int tid = threadIdx.x;
  const int64_t row = (int64_t)blockIdx.x * kNnThreads + tid;
  float q[NP];
#pragma unroll
  for (int k = 0; k < NP; ++k) q[k] = (row < Vs && k < n) ? src[row * n + k] : 0.f;
  float best = INFINITY;
  int64_t bi = -1;
  const int64_t t_begin = (int64_t)blockIdx.y * tiles_per_split * TT;
  const int64_t t_end = min(Vt, t_begin + tiles_per_split * TT);
  dnfm::nn_scan<NP>(q, tgt, n, n, t_begin, t_end, ts, best, bi);
  if (row >= Vs) return;
  if (part_d) {
    part_d[(int64_t)blockIdx.y * Vs + row] = best;
    part_i[(int64_t)blockIdx.y * Vs + row] = (int32_t)bi;
  } else {
    out[row] = bi < 0 ? 0 : bi;
  }
}

__global__ void nn_combine_kernel(const float* __restrict__ part_d, const int32_t* __restrict__ part_i, int64_t Vs,
                                  int splits, int64_t* __restrict__ out) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= Vs) return;
  out[row] = dnfm::nn_combine_row(part_d, part_i, Vs, splits, row);
}

template <int NP>
int launch_nn(const float* src, int64_t Vs, const float* tgt, int64_t Vt, int n, const NnPlan& p, int64_t* out,
              void* ws, cudaStream_t st) {
  float* part_d = nullptr;
  int32_t* part_i = nullptr;
  if (p.splits > 1) {
    part_d = (float*)ws;
    part_i = (int32_t*)(part_d + (int64_t)p.splits * Vs);
  }
  nn_kernel<NP><<<dim3((unsigned)p.qblocks, (unsigned)p.splits), kNnThreads, 0, st>>>(src, Vs, tgt, Vt, n,
                                                                                     p.tiles_per_split, out, part_d,
                                                                                     part_i);
  DN_LAUNCH_CHECK();
  if (p.splits > 1) {
    nn_combine_kernel<<<(unsigned)((Vs + 255) / 256), 256, 0, st>>>(part_d, part_i, Vs, p.splits, out);
    DN_LAUNCH_CHECK();
  }
  return DN_OK;
}

int fmap_check(const float* A, const float* B, const float* ex, const float* ey, int n, int d, double lambda) {
  if (n <= 0 || d <= 0 || !A || !B || !ex || !ey || !(lambda >= 0.0)) return DN_ERR_INVALID_ARGUMENT;
  if (n > 128) return DN_ERR_UNSUPPORTED;
  return DN_OK;
}

}  // namespace

extern "C" {

int dn_fmap_solve_fwd(const float* A, const float* B, const float* evals_x, const float* evals_y, int n, int d,
                      double lambda, float* C, dn_stream_t stream) {
  int rc = fmap_check(A, B, evals_x, evals_y, n, d, lambda);
  if (rc != DN_OK) return rc;
  if (!C) return DN_ERR_INVALID_ARGUMENT;
  const int64_t smem = solve_smem_bytes(n);
  DN_CUDA_TRY(cudaFuncSetAttribute(fmap_row_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  fmap_row_solve_kernel<<<n, kSolveThreads, smem, (cudaStream_t)stream>>>(A, B, evals_x, evals_y, lambda, n, d, nullptr,
                                                                          C, nullptr, nullptr);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int dn_fmap_solve_bwd(const float* A, const float* B, const float* evals_x, const float* evals_y, int n, int d,
                      double lambda, const float* grad_C, float* grad_A, float* grad_B, void* workspace,
                      int64_t ws_bytes, dn_stream_t stream) {
  int rc = fmap_check(A, B, evals_x, evals_y, n, d, lambda);
  if (rc != DN_OK) return rc;
  if (!grad_C || !grad_A || !grad_B) return DN_ERR_INVALID_ARGUMENT;
  if (!workspace || ws_bytes < 16ll * n * n) return DN_ERR_WORKSPACE;
  double* Cd = (double*)workspace;
  double* Wd = Cd + (int64_t)n * n;
  const int64_t smem = solve_smem_bytes(n);
  DN_CUDA_TRY(cudaFuncSetAttribute(fmap_row_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaStream_t st = (cudaStream_t)stream;
  fmap_row_solve_kernel<<<n, kSolveThreads, smem, st>>>(A, B, evals_x, evals_y, lambda, n, d, grad_C, nullptr, Cd, Wd);
  DN_LAUNCH_CHECK();
  fmap_grad_kernel<<<n, kSolveThreads, 3 * n * sizeof(double), st>>>(A, B, Cd, Wd, n, d, grad_A, grad_B);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int64_t dn_nearest_neighbor_workspace_bytes(int64_t Vs, int64_t Vt, int n) {
  if (Vs < 0 || Vt < 0 || n <= 0) return -1;
  const NnPlan p = nn_plan(Vs, Vt, n);
  return p.splits > 1 ? 8ll * p.splits * Vs : 0;
}

int dn_nearest_neighbor(const float* source, int64_t Vs, const float* target, int64_t Vt, int n, int64_t* out_index,
                        void* workspace, int64_t ws_bytes, dn_stream_t stream) {
  if (Vs < 0 || Vt <= 0 || n <= 0 || (Vs > 0 && (!source || !target || !out_index))) return DN_ERR_INVALID_ARGUMENT;
  if (n > 128 || Vt >= (1ll << 31)) return DN_ERR_UNSUPPORTED;
  if (Vs == 0) return DN_OK;
  const NnPlan p = nn_plan(Vs, Vt, n);
  if (p.splits > 1 && (!workspace || ws_bytes < 8ll * p.splits * Vs)) return DN_ERR_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  switch (p.np) {
    case 4: return launch_nn<4>(source, Vs, target, Vt, n, p, out_index, workspace, st);
    case 8: return launch_nn<8>(source, Vs, target, Vt, n, p, out_index, workspace, st);
    case 16: return launch_nn<16>(source, Vs, target, Vt, n, p, out_index, workspace, st);
    case 32: return launch_nn<32>(source, Vs, target, Vt, n, p, out_index, workspace, st);
    case 64: return launch_nn<64>(source, Vs, target, Vt, n, p, out_index, workspace, st);
    default: return launch_nn<128>(source, Vs, target, Vt, n, p, out_index, workspace, st);
  }
}

}  // extern "C"
