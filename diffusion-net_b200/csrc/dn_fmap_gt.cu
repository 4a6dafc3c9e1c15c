// Ground-truth functional maps of shape pairs (dn_fmap_ground_truth, fmaps.PairDataset.ground_truth): the training
// target of the functional-map model (faust_scape_dataset.py:186-190), C_gt = X^T with
// X = argmin || Phi_x[vts_x, :n] X - Phi_y[vts_y, :n] ||, solved through the normal equations A^T A X = A^T B in fp64.
//
// Two launches whatever the pairs are.  (1) gt_partial_kernel: one CTA per (row chunk, entry group, pair) gathers its
// kGtRows correspondence rows of A = Phi_x[vts_x, :n] and B = Phi_y[vts_y, :n] straight from the dataset's eigenvectors
// through the rebased row indices (kGtTile rows at a time in shared memory; the (m, n) gathers never exist in global
// memory) and writes its partial sums of A^T A and A^T B in fp64, each entry one fma chain over the chunk's rows in
// increasing order.  (2) gt_solve_kernel: one CTA per pair sums its chunks' partials in chunk order from 0, factors
// A^T A by dnfm::cholesky_lower (the functional-map solve's factorisation) and solves the n right-hand sides, one thread
// per column.  A pair's arithmetic depends on its own rows only, so its C_gt is bitwise the same alone or among any
// pairs, at any position.  The grid is sized from max_m, not from the drawn pairs: a CUDA graph replays it for any draw.
#include "dn_fmap_common.cuh"

namespace {

using dnfm::kSolveThreads;

constexpr int kGtMaxN = 128;                      // n cap (MAX_FMAP)
constexpr int kGtRows = 512;                       // correspondence rows per chunk
constexpr int kGtTile = 32;                        // rows staged in shared memory at a time
constexpr int kGtPer = 8;                          // entries per thread
constexpr int kGtGroup = kGtPer * kSolveThreads;   // entries per CTA
constexpr double kGtPivotTol = 1e-10;              // a pivot at or below this fraction of its diagonal: singular
                                                   // (rank deficient, or near-singular: kappa(A) >~ 1e5)
constexpr int64_t kGtBadPair = 1, kGtSingular = 2;

struct GtPair {
  int64_t a0, b0, m;   // first correspondence of x and of y in vts_rows, and their count; m < 0: invalid pair index
};

__device__ __forceinline__ GtPair gt_pair(const int64_t* __restrict__ vts_begin, int64_t n_shapes,
                                          const int64_t* __restrict__ table, int64_t n_table, int64_t id,
                                          int64_t max_m) {
  GtPair g{0, 0, -1};
  if (id < 0 || id >= n_table) return g;
  const int64_t x = table[2 * id], y = table[2 * id + 1];
  if (x < 0 || x >= n_shapes || y < 0 || y >= n_shapes) return g;
  g.a0 = vts_begin[x];
  g.b0 = vts_begin[y];
  const int64_t mx = vts_begin[x + 1] - g.a0, my = vts_begin[y + 1] - g.b0;
  g.m = min(min(mx, my), max_m);
  return g;
}

__global__ void __launch_bounds__(kSolveThreads) gt_partial_kernel(
    const float* __restrict__ evecs, int64_t ld_evecs, int n, const int64_t* __restrict__ vts_rows,
    const int64_t* __restrict__ vts_begin, int64_t n_shapes, const int64_t* __restrict__ table, int64_t n_table,
    const int64_t* __restrict__ pair_ids, int64_t max_m, int64_t n_chunks, double* __restrict__ part) {
  __shared__ float As[kGtTile * kGtMaxN];
  __shared__ float Bs[kGtTile * kGtMaxN];
  const int p = blockIdx.z;
  const GtPair g = gt_pair(vts_begin, n_shapes, table, n_table, pair_ids[p], max_m);
  const int64_t r0 = (int64_t)blockIdx.x * kGtRows;
  if (g.m < 0 || r0 >= g.m) return;   // no partial: the solve reads only the pair's own chunks
  const int64_t r1 = min(g.m, r0 + kGtRows);
  const int tid = threadIdx.x;
  const int nn = n * n;
  const int e0 = blockIdx.y * kGtGroup + tid;
  int j[kGtPer], k[kGtPer];
  bool ab[kGtPer];
#pragma unroll
  for (int u = 0; u < kGtPer; ++u) {
    const int e = e0 + u * kSolveThreads;
    const int f = e < nn ? e : e - nn;
    j[u] = f / n;
    k[u] = f % n;
    ab[u] = e >= nn;   // an entry of A^T B (else of A^T A)
  }
  double acc[kGtPer];
#pragma unroll
  for (int u = 0; u < kGtPer; ++u) acc[u] = 0.0;
  for (int64_t t0 = r0; t0 < r1; t0 += kGtTile) {
    const int rows = (int)min((int64_t)kGtTile, r1 - t0);
    __syncthreads();
    for (int e = tid; e < rows * n; e += kSolveThreads) {
      const int r = e / n, c = e % n;
      As[e] = evecs[vts_rows[g.a0 + t0 + r] * ld_evecs + c];
      Bs[e] = evecs[vts_rows[g.b0 + t0 + r] * ld_evecs + c];
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < kGtPer; ++u) {
      if (e0 + u * kSolveThreads >= 2 * nn) break;
      const float* src = ab[u] ? Bs : As;
      double a = acc[u];
      for (int r = 0; r < rows; ++r) a = fma((double)As[r * n + j[u]], (double)src[r * n + k[u]], a);
      acc[u] = a;
    }
  }
  double* out = part + ((int64_t)p * n_chunks + blockIdx.x) * 2 * nn;
#pragma unroll
  for (int u = 0; u < kGtPer; ++u) {
    const int e = e0 + u * kSolveThreads;
    if (e < 2 * nn) out[e] = acc[u];
  }
}

__device__ __forceinline__ void gt_flag(int64_t* status, int64_t kind, int64_t pos, int64_t id) {
  if (atomicCAS(reinterpret_cast<unsigned long long*>(status), 0ull, (unsigned long long)kind) == 0ull) {
    status[1] = pos;
    status[2] = id;
  }
}

__global__ void __launch_bounds__(kSolveThreads) gt_solve_kernel(
    const int64_t* __restrict__ vts_begin, int64_t n_shapes, const int64_t* __restrict__ table, int64_t n_table,
    const int64_t* __restrict__ pair_ids, int64_t max_m, int64_t n_chunks, int n, const double* __restrict__ part,
    double* __restrict__ rhs, float* __restrict__ C_gt, int64_t* __restrict__ status) {
  extern __shared__ double smem[];
  const int ld = n + 1;
  double* S = smem;                       // n x ld: A^T A, then its Cholesky factor
  double* floor_ = S + (int64_t)n * ld;   // pivot floors
  const int p = blockIdx.x;
  const int tid = threadIdx.x;
  const int nn = n * n;
  const int64_t id = pair_ids[p];
  const GtPair g = gt_pair(vts_begin, n_shapes, table, n_table, id, max_m);
  float* C = C_gt + (int64_t)p * nn;
  if (g.m < 0) {
    for (int e = tid; e < nn; e += kSolveThreads) C[e] = NAN;
    if (tid == 0) gt_flag(status, kGtBadPair, p, id);
    return;
  }
  const int64_t own = (g.m + kGtRows - 1) / kGtRows;
  const double* P0 = part + (int64_t)p * n_chunks * 2 * nn;
  double* X = rhs + (int64_t)p * nn;      // column c of the right-hand side (A^T B)[:, c] at X + c n
  for (int e = tid; e < 2 * nn; e += kSolveThreads) {
    double s = 0.0;
    for (int64_t c = 0; c < own; ++c) s += P0[c * 2 * nn + e];
    const int f = e < nn ? e : e - nn;
    const int j = f / n, k = f % n;
    if (e < nn) S[j * ld + k] = s;
    else X[k * n + j] = s;
  }
  __syncthreads();
  for (int j = tid; j < n; j += kSolveThreads) floor_[j] = kGtPivotTol * S[j * ld + j];
  const bool singular = dnfm::cholesky_lower(S, ld, n, floor_);
  __syncthreads();
  if (singular) {
    for (int e = tid; e < nn; e += kSolveThreads) C[e] = NAN;
    if (tid == 0) gt_flag(status, kGtSingular, p, id);
    return;
  }
  // L y = b, then L^T x = y, for column c of the right-hand side; C_gt[c][i] = X[i][c]
  for (int c = tid; c < n; c += kSolveThreads) {
    double* x = X + (int64_t)c * n;
    for (int i = 0; i < n; ++i) {
      double v = x[i];
      for (int l = 0; l < i; ++l) v -= S[i * ld + l] * x[l];
      x[i] = v / S[i * ld + i];
    }
    for (int i = n - 1; i >= 0; --i) {
      double v = x[i];
      for (int l = i + 1; l < n; ++l) v -= S[l * ld + i] * x[l];
      x[i] = v / S[i * ld + i];
    }
    for (int i = 0; i < n; ++i) C[(int64_t)c * n + i] = (float)x[i];
  }
}

int64_t align256(int64_t b) { return (b + 255) / 256 * 256; }

}  // namespace

extern "C" {

int64_t dn_fmap_ground_truth_workspace_bytes(int n_pairs, int n, int64_t max_m) {
  if (n_pairs <= 0 || n <= 0 || max_m < 0) return DN_ERR_INVALID_ARGUMENT;
  const int64_t n_chunks = max_m > 0 ? (max_m + kGtRows - 1) / kGtRows : 1;
  const int64_t nn = (int64_t)n * n;
  return align256(8 * n_pairs * n_chunks * 2 * nn) + align256(8 * n_pairs * nn);
}

int dn_fmap_ground_truth(const float* evecs, int64_t ld_evecs, int n, const int64_t* vts_rows,
                         const int64_t* vts_begin, int64_t n_shapes, const int64_t* pair_table, int64_t n_table,
                         const int64_t* pair_ids, int n_pairs, int64_t max_m, float* C_gt, int64_t* status,
                         void* workspace, int64_t ws_bytes, dn_stream_t stream) {
  if (!evecs || !vts_rows || !vts_begin || !pair_table || !pair_ids || !C_gt || !status || n <= 0 || ld_evecs < n ||
      n_shapes <= 0 || n_table <= 0 || n_pairs <= 0 || max_m < 0)
    return DN_ERR_INVALID_ARGUMENT;
  if (n > kGtMaxN || n_pairs > 65535 || max_m >= (1ll << 31)) return DN_ERR_UNSUPPORTED;
  if (!workspace || ws_bytes < dn_fmap_ground_truth_workspace_bytes(n_pairs, n, max_m)) return DN_ERR_WORKSPACE;
  const int64_t n_chunks = max_m > 0 ? (max_m + kGtRows - 1) / kGtRows : 1;
  const int64_t nn = (int64_t)n * n;
  double* part = static_cast<double*>(workspace);
  double* rhs = reinterpret_cast<double*>(static_cast<char*>(workspace) + align256(8 * n_pairs * n_chunks * 2 * nn));
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned groups = (unsigned)((2 * nn + kGtGroup - 1) / kGtGroup);
  gt_partial_kernel<<<dim3((unsigned)n_chunks, groups, (unsigned)n_pairs), kSolveThreads, 0, st>>>(
      evecs, ld_evecs, n, vts_rows, vts_begin, n_shapes, pair_table, n_table, pair_ids, max_m, n_chunks, part);
  DN_LAUNCH_CHECK();
  const int smem = (int)(sizeof(double) * (nn + 2 * n));
  DN_CUDA_TRY(cudaFuncSetAttribute(gt_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  gt_solve_kernel<<<(unsigned)n_pairs, kSolveThreads, smem, st>>>(vts_begin, n_shapes, pair_table, n_table, pair_ids,
                                                                  max_m, n_chunks, n, part, rhs, C_gt, status);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

}  // extern "C"
