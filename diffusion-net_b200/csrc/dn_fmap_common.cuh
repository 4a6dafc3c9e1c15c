// Device bodies of the functional-map kernels, shared by the single-pair kernels (dn_fmap.cu) and their pair-batch
// forms (dn_fmap_batch.cu), so that both run the same arithmetic in the same order.  See dn_fmap.cu for the method.
#pragma once
#include <math.h>

#include "dn_internal.h"

namespace dnfm {

constexpr int kSolveThreads = 256;
constexpr int kChunk = 32;            // columns of A / B staged per pass over d
constexpr int kChunkLd = kChunk + 1;  // padded row of the staged chunk (no bank conflicts between rows)

inline int64_t solve_smem_bytes(int n) {
  return (int64_t)sizeof(double) * ((int64_t)n * (n + 1) + 2 * n) + (int64_t)sizeof(float) * (n * kChunkLd + kChunk);
}

// Right-looking Cholesky of the symmetric n x n matrix S (lower triangle, row stride ld) in place; the diagonal ends as
// L_kk.  Returns true (the same on every thread) at the first pivot k that is not above piv_floor[k] (not above 0 when
// piv_floor is null; a NaN pivot always stops), leaving S partly factored.  Run by all kSolveThreads threads of a CTA.
__device__ __forceinline__ bool cholesky_lower(double* S, int ld, int n, const double* piv_floor) {
  const int tid = threadIdx.x;
  for (int k = 0; k < n; ++k) {
    __syncthreads();
    const double piv = S[k * ld + k];
    if (!(piv > (piv_floor ? piv_floor[k] : 0.0))) return true;  // every thread reads the same pivot: a uniform exit
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
  return false;
}

// Factor S_i and solve for row i of one pair (A, B: n x d, row stride d).  Forward (G == null): C_out[i] = c_i in fp32
// (NaN when singular).  Backward: Cd[i] = c_i and Wd[i] = w_i = S_i^-1 g_i in fp64.  Run by all kSolveThreads threads of
// a CTA with the dynamic shared memory of solve_smem_bytes(n).
__device__ __forceinline__ void row_solve(const float* __restrict__ A, const float* __restrict__ B,
                                          const float* __restrict__ ex, const float* __restrict__ ey, double lambda,
                                          int n, int d, int i, const float* __restrict__ G, float* __restrict__ C_out,
                                          double* __restrict__ Cd, double* __restrict__ Wd, double* smem) {
  const int ld = n + 1;
  double* S = smem;
  double* r = S + (int64_t)n * ld;  // A b_i, then c_i
  double* w = r + n;                // g_i, then w_i
  float* As = reinterpret_cast<float*>(w + n);
  float* bs = As + n * kChunkLd;
  const int tid = threadIdx.x;
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
  const bool singular = cholesky_lower(S, ld, n, nullptr);
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

// Row j of dA and dB of one pair from c_i, w_i (fp64, rows of Cd / Wd).  Shared memory: 3 n doubles.
__device__ __forceinline__ void grad_row(const float* __restrict__ A, const float* __restrict__ B,
                                         const double* __restrict__ Cd, const double* __restrict__ Wd, int n, int d,
                                         int j, float* __restrict__ dA, float* __restrict__ dB, double* smem) {
  double* M = smem;          // M[j][:]
  double* wcol = M + n;      // w_i[j], i < n
  double* wrow = wcol + n;   // w_j[k], k < n
  const int tid = threadIdx.x;
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

inline int nn_np(int n) {
  int np = 4;
  while (np < n) np *= 2;
  return np;
}

// Scan target rows [t_begin, t_end) (row stride ld_tgt, the first n columns) in increasing index through shared-memory
// tiles `ts` (kNnTileFloats floats), keeping in (best, bi) the first strict minimum of sum_k (q_k - t_k)^2, one fp32
// fmaf chain in increasing k over NP columns (zero pads add exactly 0).  Run by all kNnThreads threads of a CTA.
template <int NP>
__device__ __forceinline__ void nn_scan(const float (&q)[NP], const float* __restrict__ tgt, int64_t ld_tgt, int n,
                                        int64_t t_begin, int64_t t_end, float* ts, float& best, int64_t& bi) {
  constexpr int TT = kNnTileFloats / NP;
  const int tid = threadIdx.x;
  for (int64_t base = t_begin; base < t_end; base += TT) {
    const int cnt = (int)min((int64_t)TT, t_end - base);
    __syncthreads();
    for (int e = tid; e < cnt * NP; e += kNnThreads) {
      const int rr = e / NP, k = e % NP;
      ts[e] = k < n ? tgt[(base + rr) * ld_tgt + k] : 0.f;
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
}

// Index of row `row` from the per-range partials (ranges in increasing target order, strict <: the lowest index wins a
// tie; a row no range found anything for gets 0).
__device__ __forceinline__ int64_t nn_combine_row(const float* __restrict__ part_d, const int32_t* __restrict__ part_i,
                                                  int64_t Vs, int splits, int64_t row) {
  float best = INFINITY;
  int64_t bi = -1;
  for (int s = 0; s < splits; ++s) {
    const float dd = part_d[(int64_t)s * Vs + row];
    if (dd < best) { best = dd; bi = part_i[(int64_t)s * Vs + row]; }
  }
  return bi < 0 ? 0 : bi;
}

}  // namespace dnfm
