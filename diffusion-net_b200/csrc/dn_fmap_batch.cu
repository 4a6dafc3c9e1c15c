// The functional-map head over a batch of shape pairs (include/diffusion_net_b200.h, "functional maps over a pair
// batch"): the solve of dn_fmap_solve_fwd / _bwd for P pairs of S shapes in one launch forward and three backward, and
// the pointwise map of many pairs in a launch count that does not depend on P (up to the documented chunking).
//
// Solve.  The spectral features of the shapes are one stack F (shape s at F + s * ld_shape, n x d, row stride d); pair p
// reads A = F_{x_p}, B = F_{y_p} through its indices, so no (P, n, d) gathered copy exists (the gather's backward would
// scatter-add, and the order of those adds would vary between runs).  Forward: one CTA per (row, pair) runs
// dnfm::row_solve, the single-pair kernel's body.  Backward: (1) the same per (row, pair) with the upstream gradient,
// c_i and w_i to the workspace in fp64; (2) dnfm::grad_row per (row, pair): dA_p, dB_p in fp32 to the workspace, as
// fmap_grad_kernel forms them; (3) per shape s and entry e: grad_F[s][e] = sum over the shape's (pair, role) list of
// dA_p[e] (role x) or dB_p[e] (role y), in fp32 from 0, in list order (increasing p, role x before role y).
//
// Pointwise map.  Pairs go in chunks (at most kPmChunkPairs pairs and, unless a single pair is larger, kPmChunkFloats
// floats of targets).  Per chunk: one launch forms T_p = Phi_{x_p}[:, :n] C_p^T for every pair of the chunk (each entry
// one fmaf chain over k in increasing order from 0, the order of the SIMT rows_gemm_kernel), rows padded with zeros to
// NP columns; one launch runs dnfm::nn_scan for the source rows Phi_{y_p}[:, :n] of every pair, with the targets split
// into ranges when the chunk has few source blocks; a third combines the ranges in order.  Every distance is the
// single-pair kernel's fmaf chain and the first strict minimum is kept, so each pair's map is bitwise
// dn_nearest_neighbor's on the same T_p.
#include "dn_fmap_common.cuh"

#include <string.h>

#include <algorithm>
#include <vector>

namespace {

using dnfm::kNnThreads;
using dnfm::kNnTileFloats;
using dnfm::kSolveThreads;

// ---- solve --------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kSolveThreads) fmap_row_solve_batched_kernel(
    const float* __restrict__ F, int64_t ld_shape, const float* __restrict__ evals, int64_t ld_evals,
    const int32_t* __restrict__ pair_x, const int32_t* __restrict__ pair_y, double lambda, int n, int d,
    const float* __restrict__ G, float* __restrict__ C_out, double* __restrict__ Cd, double* __restrict__ Wd) {
  extern __shared__ double smem[];
  const int p = blockIdx.y;
  const int x = pair_x[p], y = pair_y[p];
  const int64_t nn = (int64_t)n * n;
  dnfm::row_solve(F + x * ld_shape, F + y * ld_shape, evals + x * ld_evals, evals + y * ld_evals, lambda, n, d,
                  blockIdx.x, G ? G + p * nn : nullptr, C_out ? C_out + p * nn : nullptr, Cd ? Cd + p * nn : nullptr,
                  Wd ? Wd + p * nn : nullptr, smem);
}

__global__ void __launch_bounds__(kSolveThreads) fmap_grad_batched_kernel(
    const float* __restrict__ F, int64_t ld_shape, const int32_t* __restrict__ pair_x,
    const int32_t* __restrict__ pair_y, const double* __restrict__ Cd, const double* __restrict__ Wd, int n, int d,
    float* __restrict__ dA, float* __restrict__ dB) {
  extern __shared__ double smem[];
  const int p = blockIdx.y;
  const int64_t nn = (int64_t)n * n, nd = (int64_t)n * d;
  dnfm::grad_row(F + pair_x[p] * ld_shape, F + pair_y[p] * ld_shape, Cd + p * nn, Wd + p * nn, n, d, blockIdx.x,
                 dA + p * nd, dB + p * nd, smem);
}

// grad_F[s][e] (e < n d) = sum over the (pair, role) entries of shape s, in list order, of dA_p[e] or dB_p[e]
__global__ void fmap_shape_grad_kernel(const float* __restrict__ dA, const float* __restrict__ dB, int64_t nd,
                                       const int32_t* __restrict__ role_begin, const int32_t* __restrict__ role_list,
                                       float* __restrict__ grad_F, int64_t ld_shape) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int s = blockIdx.y;
  if (e >= nd) return;
  float acc = 0.f;
  for (int r = role_begin[s]; r < role_begin[s + 1]; ++r) {
    const int q = role_list[r];
    acc += ((q & 1) ? dB : dA)[(int64_t)(q >> 1) * nd + e];
  }
  grad_F[(int64_t)s * ld_shape + e] = acc;
}

int solve_batched_check(const float* F, int64_t ld_shape, const float* evals, int64_t ld_evals, int n_shapes,
                        const int32_t* pair_x, const int32_t* pair_y, int n_pairs, int n, int d, double lambda) {
  if (n <= 0 || d <= 0 || n_shapes <= 0 || n_pairs <= 0 || !F || !evals || !pair_x || !pair_y || !(lambda >= 0.0) ||
      ld_shape < (int64_t)n * d || ld_evals < n)
    return DN_ERR_INVALID_ARGUMENT;
  if (n > 128 || n_pairs >= 65536 || n_shapes >= 65536) return DN_ERR_UNSUPPORTED;
  return DN_OK;
}

int64_t align256(int64_t b) { return (b + 255) / 256 * 256; }

// ---- pointwise map ------------------------------------------------------------------------------------------------
constexpr int kPmChunkPairs = 64;
constexpr int64_t kPmChunkFloats = 16ll << 20;   // 64 MiB of T per chunk unless one pair alone needs more
constexpr int kPmBuildRows = 32;                 // rows of T one CTA of the build forms

struct PmPair {
  int32_t tgt_row0, vt;   // rows of Phi_x in the basis, and their count
  int32_t src_row0, vs;   // rows of Phi_y
  int32_t t_row0;         // first row of T_p in the chunk's T (NP floats per row)
  int32_t out_row0;       // first output / partial row of the pair inside the chunk
  int32_t qblk0;          // first search CTA of the pair
  int32_t tblk0;          // first build CTA of the pair
  int32_t pair;           // pair index (its C)
};
struct PmChunk {
  PmPair p[kPmChunkPairs];
  int n_pairs;
  int splits;
};

__device__ __forceinline__ int pm_find(const PmChunk& c, int blk, bool build) {
  int pi = 0;
  for (int i = 1; i < c.n_pairs; ++i)
    if (blk >= (build ? c.p[i].tblk0 : c.p[i].qblk0)) pi = i;
  return pi;
}

// T_p[v][j] = sum_k Phi_x[v][k] C_p[j][k] (j < n; zero for n <= j < NP): one fmaf chain in increasing k from 0
template <int NP>
__global__ void __launch_bounds__(256) pm_build_kernel(const __grid_constant__ PmChunk c, const float* __restrict__ Cm,
                                                       int n, const float* __restrict__ evecs, int64_t ld_evecs,
                                                       float* __restrict__ T) {
  const PmPair& P = c.p[pm_find(c, blockIdx.x, true)];
  const float* Cp = Cm + (int64_t)P.pair * n * n;
  const int64_t v0 = (int64_t)(blockIdx.x - P.tblk0) * kPmBuildRows;
  for (int e = threadIdx.x; e < kPmBuildRows * NP; e += blockDim.x) {
    const int64_t v = v0 + e / NP;
    const int j = e % NP;
    if (v >= P.vt) break;
    float acc = 0.f;
    if (j < n) {
      const float* phi = evecs + (P.tgt_row0 + v) * ld_evecs;
      const float* cj = Cp + (int64_t)j * n;
      for (int k = 0; k < n; ++k) acc = fmaf(phi[k], cj[k], acc);
    }
    T[(P.t_row0 + v) * NP + j] = acc;
  }
}

template <int NP>
__global__ void __launch_bounds__(kNnThreads) pm_nn_kernel(const __grid_constant__ PmChunk c, int n,
                                                           const float* __restrict__ evecs, int64_t ld_evecs,
                                                           const float* __restrict__ T, int64_t* __restrict__ out,
                                                           float* __restrict__ part_d, int32_t* __restrict__ part_i,
                                                           int64_t rows) {
  constexpr int TT = kNnTileFloats / NP;
  __shared__ __align__(16) float ts[kNnTileFloats];
  const PmPair& P = c.p[pm_find(c, blockIdx.x, false)];
  const int tid = threadIdx.x;
  const int64_t row = (int64_t)(blockIdx.x - P.qblk0) * kNnThreads + tid;
  float q[NP];
#pragma unroll
  for (int k = 0; k < NP; ++k) q[k] = (row < P.vs && k < n) ? evecs[(P.src_row0 + row) * ld_evecs + k] : 0.f;
  float best = INFINITY;
  int64_t bi = -1;
  const int64_t tiles = (P.vt + TT - 1) / TT;
  const int64_t tps = (tiles + c.splits - 1) / c.splits;
  const int64_t t_begin = (int64_t)blockIdx.y * tps * TT;
  const int64_t t_end = min((int64_t)P.vt, t_begin + tps * TT);
  dnfm::nn_scan<NP>(q, T + (int64_t)P.t_row0 * NP, NP, n, t_begin, t_end, ts, best, bi);
  if (row >= P.vs) return;
  const int64_t r = P.out_row0 + row;
  if (part_d) {
    part_d[(int64_t)blockIdx.y * rows + r] = best;
    part_i[(int64_t)blockIdx.y * rows + r] = (int32_t)bi;
  } else {
    out[r] = bi < 0 ? 0 : bi;
  }
}

__global__ void pm_combine_kernel(const float* __restrict__ part_d, const int32_t* __restrict__ part_i, int64_t rows,
                                  int splits, int64_t* __restrict__ out) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= rows) return;
  out[row] = dnfm::nn_combine_row(part_d, part_i, rows, splits, row);
}

// The chunks of a pair batch, with each chunk's T rows and source rows (the workspace it needs).
struct PmPlan {
  std::vector<PmChunk> chunks;
  std::vector<int64_t> t_rows, src_rows, out_base;
  int64_t ws_bytes = 0;
};

int pm_plan(int n, int n_pairs, const int32_t* pair_x, const int32_t* pair_y, const int32_t* row_begin,
            const int32_t* n_rows, int n_shapes, PmPlan* plan) {
  const int np = dnfm::nn_np(n);
  const int tt = kNnTileFloats / np;
  int64_t out_base = 0;
  for (int p = 0; p < n_pairs;) {
    PmChunk c;
    memset(&c, 0, sizeof(c));
    int64_t t_rows = 0, src_rows = 0, qblk = 0, tblk = 0;
    while (p < n_pairs && c.n_pairs < kPmChunkPairs) {
      const int x = pair_x[p], y = pair_y[p];
      if (x < 0 || x >= n_shapes || y < 0 || y >= n_shapes) return DN_ERR_INVALID_ARGUMENT;
      const int64_t vt = n_rows[x], vs = n_rows[y];
      if (vt <= 0 || vs < 0) return DN_ERR_INVALID_ARGUMENT;
      if (c.n_pairs > 0 && (t_rows + vt) * np > kPmChunkFloats) break;
      if ((t_rows + vt) >= (1ll << 31) / np || src_rows + vs >= (1ll << 31)) {
        if (c.n_pairs == 0) return DN_ERR_UNSUPPORTED;
        break;
      }
      PmPair& P = c.p[c.n_pairs++];
      P.tgt_row0 = row_begin[x]; P.vt = (int32_t)vt;
      P.src_row0 = row_begin[y]; P.vs = (int32_t)vs;
      P.t_row0 = (int32_t)t_rows; P.out_row0 = (int32_t)src_rows;
      P.qblk0 = (int32_t)qblk; P.tblk0 = (int32_t)tblk; P.pair = p;
      t_rows += vt;
      src_rows += vs;
      qblk += (vs + kNnThreads - 1) / kNnThreads;
      tblk += (vt + kPmBuildRows - 1) / kPmBuildRows;
      ++p;
    }
    // splits as dn_nearest_neighbor plans them, over the chunk's source blocks and its largest target count
    int64_t max_tiles = 1;
    for (int i = 0; i < c.n_pairs; ++i) max_tiles = std::max<int64_t>(max_tiles, (c.p[i].vt + tt - 1) / tt);
    int64_t s = qblk > 0 ? (dnfm::kNnTargetCtas + qblk - 1) / qblk : 1;
    s = s < 1 ? 1 : (s > dnfm::kNnMaxSplit ? dnfm::kNnMaxSplit : s);
    if (s > max_tiles) s = max_tiles;
    c.splits = (int)s;
    plan->chunks.push_back(c);
    plan->t_rows.push_back(t_rows);
    plan->src_rows.push_back(src_rows);
    plan->out_base.push_back(out_base);
    out_base += src_rows;
    const int64_t b = align256(t_rows * np * 4) + (c.splits > 1 ? align256(8 * c.splits * src_rows) : 0);
    plan->ws_bytes = std::max(plan->ws_bytes, b);
  }
  return DN_OK;
}

template <int NP>
int launch_pm_chunk(const PmChunk& c, int64_t t_rows, int64_t src_rows, const float* Cm, int n, const float* evecs,
                    int64_t ld_evecs, int64_t* out, char* ws, cudaStream_t st) {
  float* T = reinterpret_cast<float*>(ws);
  float* part_d = nullptr;
  int32_t* part_i = nullptr;
  if (c.splits > 1) {
    part_d = reinterpret_cast<float*>(ws + align256(t_rows * NP * 4));
    part_i = reinterpret_cast<int32_t*>(part_d + (int64_t)c.splits * src_rows);
  }
  const PmPair& last = c.p[c.n_pairs - 1];
  const int tblocks = last.tblk0 + (last.vt + kPmBuildRows - 1) / kPmBuildRows;
  const int qblocks = last.qblk0 + (last.vs + kNnThreads - 1) / kNnThreads;
  pm_build_kernel<NP><<<tblocks, 256, 0, st>>>(c, Cm, n, evecs, ld_evecs, T);
  DN_LAUNCH_CHECK();
  if (qblocks == 0) return DN_OK;
  pm_nn_kernel<NP><<<dim3((unsigned)qblocks, (unsigned)c.splits), kNnThreads, 0, st>>>(c, n, evecs, ld_evecs, T, out,
                                                                                      part_d, part_i, src_rows);
  DN_LAUNCH_CHECK();
  if (c.splits > 1) {
    pm_combine_kernel<<<(unsigned)((src_rows + 255) / 256), 256, 0, st>>>(part_d, part_i, src_rows, c.splits, out);
    DN_LAUNCH_CHECK();
  }
  return DN_OK;
}

int pm_check(int n, int n_pairs, const int32_t* pair_x, const int32_t* pair_y, const int32_t* row_begin,
             const int32_t* n_rows, int n_shapes) {
  if (n <= 0 || n_pairs <= 0 || n_shapes <= 0 || !pair_x || !pair_y || !row_begin || !n_rows)
    return DN_ERR_INVALID_ARGUMENT;
  if (n > 128) return DN_ERR_UNSUPPORTED;
  return DN_OK;
}

}  // namespace

extern "C" {

int64_t dn_fmap_solve_batched_workspace_bytes(int n_pairs, int n, int d) {
  if (n_pairs <= 0 || n <= 0 || d <= 0) return -1;
  return align256(16ll * n * n * n_pairs) + align256(4ll * n_pairs * n * d) * 2;
}

int dn_fmap_solve_fwd_batched(const float* F, int64_t ld_shape, const float* evals, int64_t ld_evals, int n_shapes,
                              const int32_t* pair_x, const int32_t* pair_y, int n_pairs, int n, int d, double lambda,
                              float* C, dn_stream_t stream) {
  int rc = solve_batched_check(F, ld_shape, evals, ld_evals, n_shapes, pair_x, pair_y, n_pairs, n, d, lambda);
  if (rc != DN_OK) return rc;
  if (!C) return DN_ERR_INVALID_ARGUMENT;
  const int64_t smem = dnfm::solve_smem_bytes(n);
  DN_CUDA_TRY(cudaFuncSetAttribute(fmap_row_solve_batched_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)smem));
  fmap_row_solve_batched_kernel<<<dim3(n, n_pairs), kSolveThreads, smem, (cudaStream_t)stream>>>(
      F, ld_shape, evals, ld_evals, pair_x, pair_y, lambda, n, d, nullptr, C, nullptr, nullptr);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int dn_fmap_solve_bwd_batched(const float* F, int64_t ld_shape, const float* evals, int64_t ld_evals, int n_shapes,
                              const int32_t* pair_x, const int32_t* pair_y, int n_pairs, const int32_t* role_begin,
                              const int32_t* role_list, int n, int d, double lambda, const float* grad_C,
                              float* grad_F, void* workspace, int64_t ws_bytes, dn_stream_t stream) {
  int rc = solve_batched_check(F, ld_shape, evals, ld_evals, n_shapes, pair_x, pair_y, n_pairs, n, d, lambda);
  if (rc != DN_OK) return rc;
  if (!grad_C || !grad_F || !role_begin || !role_list) return DN_ERR_INVALID_ARGUMENT;
  if (!workspace || ws_bytes < dn_fmap_solve_batched_workspace_bytes(n_pairs, n, d)) return DN_ERR_WORKSPACE;
  char* w = static_cast<char*>(workspace);
  const int64_t nn = (int64_t)n * n * n_pairs, nd = (int64_t)n * d;
  double* Cd = reinterpret_cast<double*>(w);
  double* Wd = Cd + nn;
  float* dA = reinterpret_cast<float*>(w + align256(16 * nn));
  float* dB = reinterpret_cast<float*>(w + align256(16 * nn) + align256(4 * nd * n_pairs));
  const int64_t smem = dnfm::solve_smem_bytes(n);
  DN_CUDA_TRY(cudaFuncSetAttribute(fmap_row_solve_batched_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)smem));
  cudaStream_t st = (cudaStream_t)stream;
  fmap_row_solve_batched_kernel<<<dim3(n, n_pairs), kSolveThreads, smem, st>>>(
      F, ld_shape, evals, ld_evals, pair_x, pair_y, lambda, n, d, grad_C, nullptr, Cd, Wd);
  DN_LAUNCH_CHECK();
  fmap_grad_batched_kernel<<<dim3(n, n_pairs), kSolveThreads, 3 * n * sizeof(double), st>>>(F, ld_shape, pair_x, pair_y,
                                                                                            Cd, Wd, n, d, dA, dB);
  DN_LAUNCH_CHECK();
  fmap_shape_grad_kernel<<<dim3((unsigned)((nd + 255) / 256), n_shapes), 256, 0, st>>>(dA, dB, nd, role_begin, role_list,
                                                                                      grad_F, ld_shape);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int64_t dn_fmap_pointwise_map_batched_workspace_bytes(int n, int n_pairs, const int32_t* pair_x_host,
                                                      const int32_t* pair_y_host, const int32_t* row_begin_host,
                                                      const int32_t* n_rows_host, int n_shapes) {
  int rc = pm_check(n, n_pairs, pair_x_host, pair_y_host, row_begin_host, n_rows_host, n_shapes);
  if (rc != DN_OK) return rc;
  PmPlan plan;
  if ((rc = pm_plan(n, n_pairs, pair_x_host, pair_y_host, row_begin_host, n_rows_host, n_shapes, &plan))) return rc;
  return plan.ws_bytes;
}

int dn_fmap_pointwise_map_batched(const float* C, int n, const float* evecs, int64_t ld_evecs,
                                  const int32_t* row_begin_host, const int32_t* n_rows_host, int n_shapes,
                                  const int32_t* pair_x_host, const int32_t* pair_y_host, int n_pairs,
                                  int64_t* out_index, void* workspace, int64_t ws_bytes, dn_stream_t stream) {
  int rc = pm_check(n, n_pairs, pair_x_host, pair_y_host, row_begin_host, n_rows_host, n_shapes);
  if (rc != DN_OK) return rc;
  if (!C || !evecs || !out_index || ld_evecs < n) return DN_ERR_INVALID_ARGUMENT;
  PmPlan plan;
  if ((rc = pm_plan(n, n_pairs, pair_x_host, pair_y_host, row_begin_host, n_rows_host, n_shapes, &plan))) return rc;
  if (!workspace || ws_bytes < plan.ws_bytes) return DN_ERR_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = static_cast<char*>(workspace);
  for (size_t i = 0; i < plan.chunks.size(); ++i) {
    const PmChunk& c = plan.chunks[i];
    int64_t* out = out_index + plan.out_base[i];
    const int64_t tr = plan.t_rows[i], sr = plan.src_rows[i];
    switch (dnfm::nn_np(n)) {
      case 4: rc = launch_pm_chunk<4>(c, tr, sr, C, n, evecs, ld_evecs, out, ws, st); break;
      case 8: rc = launch_pm_chunk<8>(c, tr, sr, C, n, evecs, ld_evecs, out, ws, st); break;
      case 16: rc = launch_pm_chunk<16>(c, tr, sr, C, n, evecs, ld_evecs, out, ws, st); break;
      case 32: rc = launch_pm_chunk<32>(c, tr, sr, C, n, evecs, ld_evecs, out, ws, st); break;
      case 64: rc = launch_pm_chunk<64>(c, tr, sr, C, n, evecs, ld_evecs, out, ws, st); break;
      default: rc = launch_pm_chunk<128>(c, tr, sr, C, n, evecs, ld_evecs, out, ws, st); break;
    }
    if (rc) return rc;
  }
  return DN_OK;
}

}  // extern "C"
