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
#include <math.h>

#include "dn_internal.h"

namespace {

constexpr int kSolveThreads = 256;
constexpr int kChunk = 32;          // columns of A / B staged per pass over d
constexpr int kChunkLd = kChunk + 1;  // padded row of the staged chunk (no bank conflicts between rows)

int64_t solve_smem_bytes(int n) {
  return (int64_t)sizeof(double) * ((int64_t)n * (n + 1) + 2 * n) + (int64_t)sizeof(float) * (n * kChunkLd + kChunk);
}

// Factor S_i and solve for row i.  Forward (G == null): C_out[i] = c_i in fp32 (NaN when singular).  Backward: Cd[i] = c_i
// and Wd[i] = w_i = S_i^-1 g_i in fp64.
__global__ void __launch_bounds__(kSolveThreads) fmap_row_solve_kernel(
    const float* __restrict__ A, const float* __restrict__ B, const float* __restrict__ ex, const float* __restrict__ ey,
    double lambda, int n, int d, const float* __restrict__ G, float* __restrict__ C_out, double* __restrict__ Cd,
    double* __restrict__ Wd) {
  extern __shared__ double smem[];
  const int ld = n + 1;
  double* S = smem;
  double* r = S + (int64_t)n * ld;  // A b_i, then c_i
  double* w = r + n;                // g_i, then w_i
  float* As = reinterpret_cast<float*>(w + n);
  float* bs = As + n * kChunkLd;
  const int i = blockIdx.x, tid = threadIdx.x;
  const bool bwd = G != nullptr;

  for (int e = tid; e < n * n; e += kSolveThreads) S[(e / n) * ld + e % n] = 0.0;
  for (int j = tid; j < n; j += kSolveThreads) {
    r[j] = 0.0;
    w[j] = bwd ? (double)G[(int64_t)i * n + j] : 0.0;
  }
  // S = A A^T (lower triangle) and r = A b_i: each entry owned by one thread, summed over t = 0 .. d-1 in order
  for (int t0 = 0; t0 < d; t0 += kChunk) {
    const int tc = min(kChunk, d - t0);
    __syncthreads();
    for (int e = tid; e < n * kChunk; e += kSolveThreads) {
      const int j = e / kChunk, t = e % kChunk;
      As[j * kChunkLd + t] = t < tc ? A[(int64_t)j * d + t0 + t] : 0.f;
    }
    for (int t = tid; t < kChunk; t += kSolveThreads) bs[t] = t < tc ? B[(int64_t)i * d + t0 + t] : 0.f;
    __syncthreads();
    for (int e = tid; e < n * n + n; e += kSolveThreads) {
      if (e < n * n) {
        const int j = e / n, k = e % n;
        if (k > j) continue;
        double acc = S[j * ld + k];
        for (int t = 0; t < tc; ++t) acc = fma((double)As[j * kChunkLd + t], (double)As[k * kChunkLd + t], acc);
        S[j * ld + k] = acc;
      } else {
        const int j = e - n * n;
        double acc = r[j];
        for (int t = 0; t < tc; ++t) acc = fma((double)As[j * kChunkLd + t], (double)bs[t], acc);
        r[j] = acc;
      }
    }
  }
  __syncthreads();
  for (int j = tid; j < n; j += kSolveThreads) {
    const double dl = (double)ex[j] - (double)ey[i];
    S[j * ld + j] += lambda * (dl * dl);
  }
  // right-looking Cholesky, lower triangle in place; the diagonal ends as L_kk
  bool singular = false;
  for (int k = 0; k < n; ++k) {
    __syncthreads();
    const double piv = S[k * ld + k];
    if (!(piv > 0.0)) {  // every thread reads the same pivot: a uniform exit
      singular = true;
      break;
    }
    const double lkk = sqrt(piv);
    for (int j = k + 1 + tid; j < n; j += kSolveThreads) S[j * ld + k] /= lkk;
    __syncthreads();
    if (tid == 0) S[k * ld + k] = lkk;
    const int m = n - k - 1;
    for (int e = tid; e < m * m; e += kSolveThreads) {
      const int j = k + 1 + e / m, l = k + 1 + e % m;
      if (l <= j) S[j * ld + l] -= S[j * ld + k] * S[l * ld + k];
    }
  }
  __syncthreads();
  if (!singular && tid < 32) {  // L y = r, then L^T x = y (both right-hand sides in the backward), one warp
    const int lane = tid;
    for (int k = 0; k < n; ++k) {
      if (lane == 0) {
        r[k] /= S[k * ld + k];
        if (bwd) w[k] /= S[k * ld + k];
      }
      __syncwarp();
      for (int j = k + 1 + lane; j < n; j += 32) {
        r[j] -= S[j * ld + k] * r[k];
        if (bwd) w[j] -= S[j * ld + k] * w[k];
      }
      __syncwarp();
    }
    for (int k = n - 1; k >= 0; --k) {
      if (lane == 0) {
        r[k] /= S[k * ld + k];
        if (bwd) w[k] /= S[k * ld + k];
      }
      __syncwarp();
      for (int j = lane; j < k; j += 32) {
        r[j] -= S[k * ld + j] * r[k];
        if (bwd) w[j] -= S[k * ld + j] * w[k];
      }
      __syncwarp();
    }
  }
  __syncthreads();
  for (int j = tid; j < n; j += kSolveThreads) {
    if (bwd) {
      Cd[(int64_t)i * n + j] = singular ? (double)NAN : r[j];
      Wd[(int64_t)i * n + j] = singular ? (double)NAN : w[j];
    } else {
      C_out[(int64_t)i * n + j] = singular ? NAN : (float)r[j];
    }
  }
}

// Row j of dA and dB from c_i, w_i (fp64, rows of Cd / Wd).
__global__ void __launch_bounds__(kSolveThreads) fmap_grad_kernel(const float* __restrict__ A,
                                                                  const float* __restrict__ B,
                                                                  const double* __restrict__ Cd,
                                                                  const double* __restrict__ Wd, int n, int d,
                                                                  float* __restrict__ dA, float* __restrict__ dB) {
  extern __shared__ double smem[];
  double* M = smem;          // M[j][:]
  double* wcol = M + n;      // w_i[j], i < n
  double* wrow = wcol + n;   // w_j[k], k < n
  const int j = blockIdx.x, tid = threadIdx.x;
  for (int i = tid; i < n; i += kSolveThreads) {
    wcol[i] = Wd[(int64_t)i * n + j];
    wrow[i] = Wd[(int64_t)j * n + i];
  }
  for (int k = tid; k < n; k += kSolveThreads) {
    double acc = 0.0;
    for (int i = 0; i < n; ++i)
      acc = fma(Wd[(int64_t)i * n + j], Cd[(int64_t)i * n + k], fma(Cd[(int64_t)i * n + j], Wd[(int64_t)i * n + k], acc));
    M[k] = acc;
  }
  __syncthreads();
  for (int t = tid; t < d; t += kSolveThreads) {
    double wb = 0.0, ma = 0.0, wa = 0.0;
    for (int i = 0; i < n; ++i) wb = fma(wcol[i], (double)B[(int64_t)i * d + t], wb);
    for (int k = 0; k < n; ++k) {
      const double a = (double)A[(int64_t)k * d + t];
      ma = fma(M[k], a, ma);
      wa = fma(wrow[k], a, wa);
    }
    dA[(int64_t)j * d + t] = (float)(wb - ma);
    dB[(int64_t)j * d + t] = (float)wa;
  }
}

// ---- nearest neighbour --------------------------------------------------------------------------------------------
constexpr int kNnThreads = 128;
constexpr int kNnTileFloats = 8192;   // 32 KB of targets per tile
constexpr int kNnTargetCtas = 264;    // split the targets until the grid has about this many CTAs (two waves of 132 SMs)
constexpr int kNnMaxSplit = 16;

int nn_np(int n) {
  int np = 4;
  while (np < n) np *= 2;
  return np;
}

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
  for (int64_t base = t_begin; base < t_end; base += TT) {
    const int cnt = (int)min((int64_t)TT, t_end - base);
    __syncthreads();
    for (int e = tid; e < cnt * NP; e += kNnThreads) {
      const int rr = e / NP, k = e % NP;
      ts[e] = k < n ? tgt[(base + rr) * n + k] : 0.f;
    }
    __syncthreads();
    int rr = 0;
    for (; rr + 1 < cnt; rr += 2) {  // two independent chains; each distance is still one chain in increasing k
      const float4* t0 = reinterpret_cast<const float4*>(ts + rr * NP);
      const float4* t1 = reinterpret_cast<const float4*>(ts + (rr + 1) * NP);
      float d0 = 0.f, d1 = 0.f;
#pragma unroll
      for (int kk = 0; kk < NP / 4; ++kk) {
        const float4 a = t0[kk], b = t1[kk];
        float e;
        e = q[4 * kk + 0] - a.x; d0 = fmaf(e, e, d0);
        e = q[4 * kk + 0] - b.x; d1 = fmaf(e, e, d1);
        e = q[4 * kk + 1] - a.y; d0 = fmaf(e, e, d0);
        e = q[4 * kk + 1] - b.y; d1 = fmaf(e, e, d1);
        e = q[4 * kk + 2] - a.z; d0 = fmaf(e, e, d0);
        e = q[4 * kk + 2] - b.z; d1 = fmaf(e, e, d1);
        e = q[4 * kk + 3] - a.w; d0 = fmaf(e, e, d0);
        e = q[4 * kk + 3] - b.w; d1 = fmaf(e, e, d1);
      }
      if (d0 < best) { best = d0; bi = base + rr; }
      if (d1 < best) { best = d1; bi = base + rr + 1; }
    }
    if (rr < cnt) {
      const float4* t0 = reinterpret_cast<const float4*>(ts + rr * NP);
      float d0 = 0.f;
#pragma unroll
      for (int kk = 0; kk < NP / 4; ++kk) {
        const float4 a = t0[kk];
        float e;
        e = q[4 * kk + 0] - a.x; d0 = fmaf(e, e, d0);
        e = q[4 * kk + 1] - a.y; d0 = fmaf(e, e, d0);
        e = q[4 * kk + 2] - a.z; d0 = fmaf(e, e, d0);
        e = q[4 * kk + 3] - a.w; d0 = fmaf(e, e, d0);
      }
      if (d0 < best) { best = d0; bi = base + rr; }
    }
  }
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
  float best = INFINITY;
  int64_t bi = -1;
  for (int s = 0; s < splits; ++s) {  // ranges in increasing target order, strict <: the lowest index wins a tie
    const float dd = part_d[(int64_t)s * Vs + row];
    if (dd < best) { best = dd; bi = part_i[(int64_t)s * Vs + row]; }
  }
  out[row] = bi < 0 ? 0 : bi;
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
