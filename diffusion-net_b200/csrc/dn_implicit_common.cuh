// Device bodies of the implicit heat solve, shared by the single-mesh kernel (dn_implicit.cu) and its mesh-batch form
// (dn_implicit_batch.cu), so that both run the same arithmetic in the same order: the row sweeps of the block
// Jacobi-preconditioned conjugate gradient, the per-column (per-pair) scalar updates, the CTA partial sums and the
// status entries.  See dn_implicit.cu for the method.
#pragma once
#include <cooperative_groups.h>

#include "dn_internal.h"

namespace dnim {

constexpr int kThreads = 256, kWarps = kThreads / 32, kMaxCtas = 1024, kMaxC = 256;

// CTAs per SM each column-group width (NC = ceil(C / 32)) is compiled for: 3 at NC = 1, 1 at NC = 8, 2 in between.
// The occupancy sizes the cooperative grid, and the single-mesh kernel's partial sums are grouped by CTA, so this
// also fixes its summation order.
constexpr int min_ctas_per_sm(int nc) { return nc == 1 ? 3 : nc == 8 ? 1 : 2; }

struct ImplicitArgs {
  const int32_t* rowptr;
  const int32_t* colidx;
  const float* lvals;       // dn_csr vals: L at even positions, the gy half ignored
  const float* mass;        // (V)
  float* time;              // (C): forward clamps in place at the end; backward only reads
  const float* rhs;         // forward: x (b = M x); backward: grad_out (b = g)
  const float* y;           // backward: the forward output, for the time gradient
  int64_t V;
  int C;
  int backward;
  double rtol;
  int max_iter;
  float* out;               // forward: y; backward: grad_x = M w
  float* grad_time;         // backward: += -sum_v w (L y)
  double* status;           // 2 + 2 n, n = C (one mesh) or n_meshes C (a batch), see the header
  double *X, *R, *P, *Q;    // V x C each
  double* ldiag;            // V
  double* part;             // 2 x (partial slots) x C
  double* col;              // 6 x n: rz, |b|, alpha, beta, r.r, and the iteration count
  int* active;              // n: 1 iterating, 0 converged, -1 non-finite (NaN result)
  int* n_active;            // one mesh: 1; a batch: the per-CTA counts, kMaxCtas
  // a mesh batch (dn_implicit_batch.cu) only
  int n_meshes;
  const int32_t* tile_mesh;  // [V / 128]
  const int32_t* mesh_rows;  // [2 n_meshes]: rows [begin, end) of mesh b, begin a multiple of 128
};

__device__ __forceinline__ double ldg_cg(const double* p) { return __ldcg(p); }
__device__ __forceinline__ int ldg_cg(const int* p) { return __ldcg(p); }

// the Jacobi preconditioner of row v, column c: m_v + t_c L_vv
__device__ __forceinline__ double jacobi(double m, double t, double dg) { return m + t * dg; }

// Sum the per-warp partials of this CTA in warp order and store them in the partial slot `slot` (columns < C).
template <int NC>
__device__ void cta_partial(double (*red)[kMaxC], const double* acc, int C, double* slot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < NC; ++q) {
    const int c = lane + 32 * q;
    if (c < C) red[warp][c] = acc[q];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kThreads) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += red[w][c];
    slot[c] = s;
  }
  __syncthreads();
}

// sum of column c over the partial slots [g0, g1), in slot order
__device__ __forceinline__ double slot_sum(const double* part, int g0, int g1, int C, int c) {
  double s = 0.0;
  for (int g = g0; g < g1; ++g) s += ldg_cg(part + (int64_t)g * C + c);
  return s;
}

// This CTA's total of `act` over its threads, valid in thread 0.
__device__ __forceinline__ int cta_total(int act, int* s_act) {
  const int lane = threadIdx.x & 31;
  for (int o = 16; o > 0; o >>= 1) act += __shfl_xor_sync(0xffffffffu, act, o);
  if (lane == 0) s_act[threadIdx.x >> 5] = act;
  __syncthreads();
  int n = 0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kWarps; ++w) n += s_act[w];
  return n;
}

// ---- row sweeps: one warp per row v, lane l owning columns l, l + 32, ...; t: the lane's clamped times

// init: L_vv (stored), b, x = 0, r = b, p = z = b / d; acc0 += b.b, acc1 += b.z
template <int NC>
__device__ __forceinline__ void row_init(const ImplicitArgs& a, int64_t v, int lane, const double (&t)[NC],
                                         const bool (&cok)[NC], double (&acc0)[NC], double (&acc1)[NC]) {
  const int C = a.C;
  const int s = a.rowptr[v], e = a.rowptr[v + 1];
  double dg = 0.0;
  for (int p = s + lane; p < e; p += 32)
    if (a.colidx[p] == v) dg += (double)a.lvals[2 * (int64_t)p];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dg += __shfl_xor_sync(0xffffffffu, dg, o);
  if (lane == 0) a.ldiag[v] = dg;
  const double m = (double)a.mass[v];
#pragma unroll
  for (int q = 0; q < NC; ++q) {
    if (!cok[q]) continue;
    const int64_t i = v * C + lane + 32 * q;
    const double b = a.backward ? (double)a.rhs[i] : m * (double)a.rhs[i];
    const double z = b / jacobi(m, t[q], dg);
    a.X[i] = 0.0;
    a.R[i] = b;
    a.P[i] = z;
    acc0[q] = fma(b, b, acc0[q]);
    acc1[q] = fma(b, z, acc1[q]);
  }
}

// q = M p + t (L p); acc0 += p.q
template <int NC>
__device__ __forceinline__ void row_apply(const ImplicitArgs& a, int64_t v, int lane, const double (&t)[NC],
                                          const bool (&on)[NC], double (&acc0)[NC]) {
  const int C = a.C;
  double lp[NC];
#pragma unroll
  for (int q = 0; q < NC; ++q) lp[q] = 0.0;
  const int s = a.rowptr[v], e = a.rowptr[v + 1];
  for (int p = s; p < e; ++p) {
    const double l = (double)a.lvals[2 * (int64_t)p];
    const double* pc = a.P + (int64_t)a.colidx[p] * C;
#pragma unroll
    for (int q = 0; q < NC; ++q)
      if (on[q]) lp[q] = fma(l, ldg_cg(pc + lane + 32 * q), lp[q]);
  }
  const double m = (double)a.mass[v];
#pragma unroll
  for (int q = 0; q < NC; ++q) {
    if (!on[q]) continue;
    const int64_t i = v * C + lane + 32 * q;
    const double pv = ldg_cg(a.P + i);
    const double qv = fma(t[q], lp[q], m * pv);
    a.Q[i] = qv;
    acc0[q] = fma(pv, qv, acc0[q]);
  }
}

// x += alpha p, r -= alpha q; acc0 += r.r, acc1 += r.z
template <int NC>
__device__ __forceinline__ void row_update(const ImplicitArgs& a, int64_t v, int lane, const double (&t)[NC],
                                           const bool (&on)[NC], const double (&al)[NC], double (&acc0)[NC],
                                           double (&acc1)[NC]) {
  const int C = a.C;
  const double m = (double)a.mass[v], dg = ldg_cg(a.ldiag + v);
#pragma unroll
  for (int q = 0; q < NC; ++q) {
    if (!on[q]) continue;
    const int64_t i = v * C + lane + 32 * q;
    a.X[i] = fma(al[q], a.P[i], a.X[i]);
    const double r = fma(-al[q], a.Q[i], a.R[i]);
    a.R[i] = r;
    acc0[q] = fma(r, r, acc0[q]);
    acc1[q] = fma(r, r / jacobi(m, t[q], dg), acc1[q]);
  }
}

// p = r / d + beta p
template <int NC>
__device__ __forceinline__ void row_direction(const ImplicitArgs& a, int64_t v, int lane, const double (&t)[NC],
                                              const bool (&on)[NC], const double (&be)[NC]) {
  const int C = a.C;
  const double m = (double)a.mass[v], dg = ldg_cg(a.ldiag + v);
#pragma unroll
  for (int q = 0; q < NC; ++q) {
    if (!on[q]) continue;
    const int64_t i = v * C + lane + 32 * q;
    a.P[i] = fma(be[q], a.P[i], a.R[i] / jacobi(m, t[q], dg));
  }
}

// forward output of row v: x where the column converged (on), NaN where it went non-finite
template <int NC>
__device__ __forceinline__ void row_write_fwd(const ImplicitArgs& a, int64_t v, int lane, const bool (&cok)[NC],
                                              const bool (&on)[NC]) {
  const float fnan = __int_as_float(0x7fc00000);
  const int C = a.C;
#pragma unroll
  for (int q = 0; q < NC; ++q)
    if (cok[q]) a.out[v * C + lane + 32 * q] = on[q] ? (float)a.X[v * C + lane + 32 * q] : fnan;
}

// backward output of row v: grad_x = M w (NaN where the column went non-finite); acc0 += w (L y)
template <int NC>
__device__ __forceinline__ void row_write_bwd(const ImplicitArgs& a, int64_t v, int lane, const bool (&cok)[NC],
                                              const bool (&on)[NC], double (&acc0)[NC]) {
  const float fnan = __int_as_float(0x7fc00000);
  const int C = a.C;
  double ly[NC];
#pragma unroll
  for (int q = 0; q < NC; ++q) ly[q] = 0.0;
  const int s = a.rowptr[v], e = a.rowptr[v + 1];
  for (int p = s; p < e; ++p) {
    const double l = (double)a.lvals[2 * (int64_t)p];
    const float* yc = a.y + (int64_t)a.colidx[p] * C;
#pragma unroll
    for (int q = 0; q < NC; ++q)
      if (cok[q]) ly[q] = fma(l, (double)yc[lane + 32 * q], ly[q]);
  }
  const double m = (double)a.mass[v];
#pragma unroll
  for (int q = 0; q < NC; ++q) {
    if (!cok[q]) continue;
    const int64_t i = v * C + lane + 32 * q;
    const double w = a.X[i];
    a.out[i] = on[q] ? (float)(m * w) : fnan;
    acc0[q] = fma(w, ly[q], acc0[q]);
  }
}

// ---- the scalars of column (pair) j, one thread each: col is 6 x n

struct PairCols {
  double *rz, *bnorm, *alpha, *beta, *rr, *iters;
};

__device__ __forceinline__ PairCols pair_cols(double* col, int64_t n) {
  return {col, col + n, col + 2 * n, col + 3 * n, col + 4 * n, col + 5 * n};
}

// start from b.b and r.z; 1 when the column iterates (b = 0: x = 0 is exact; a non-finite b: NaN result)
__device__ __forceinline__ int pair_start(const PairCols& k, int* active, int64_t j, double bb, double rzv) {
  k.bnorm[j] = sqrt(bb);
  k.rz[j] = rzv;
  k.rr[j] = bb;
  k.iters[j] = 0.0;
  const int live = bb > 0.0;
  active[j] = isfinite(bb) ? live : -1;
  return live && isfinite(bb);
}

// the step length from p.q
__device__ __forceinline__ void pair_alpha(const PairCols& k, int64_t j, double pq) { k.alpha[j] = k.rz[j] / pq; }

// after an update with r.r = r2 and r.z = rzn: 1 when the column iterates again
__device__ __forceinline__ int pair_step(const PairCols& k, int* active, int64_t j, double r2, double rzn,
                                         double rtol) {
  k.rr[j] = r2;
  k.iters[j] += 1.0;
  if (!(isfinite(k.alpha[j]) && isfinite(r2) && isfinite(rzn))) {   // p.q or the data went non-finite
    active[j] = -1;
  } else if (sqrt(r2) <= rtol * k.bnorm[j]) {
    active[j] = 0;              // frozen: x_j is final
  } else {
    k.beta[j] = rzn / k.rz[j];
    k.rz[j] = rzn;
    return 1;
  }
  return 0;
}

// status[2 + j] (iterations) and status[2 + n + j] (relative residual, NaN for a non-finite column); returns the
// iterations
__device__ __forceinline__ double pair_status(const PairCols& k, const int* active, double* status, int64_t n,
                                              int64_t j) {
  const double itc = ldg_cg(k.iters + j);
  status[2 + j] = itc;
  const double bn = ldg_cg(k.bnorm + j);
  status[2 + n + j] = ldg_cg(active + j) < 0 ? __longlong_as_double(0x7ff8000000000000ll)
                      : bn > 0.0              ? sqrt(ldg_cg(k.rr + j)) / bn
                                              : 0.0;
  return itc;
}

// One cooperative launch of `kernel` over as many CTAs as fit on the device at once, at most max_ctas (>= 1) and
// kMaxCtas.
template <typename Kernel>
int launch_cooperative(Kernel kernel, const ImplicitArgs& a, int64_t max_ctas, cudaStream_t st) {
  int nb = 0;
  DN_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernel, kThreads, 0));
  if (nb < 1) return DN_ERR_UNSUPPORTED;
  int64_t g = (int64_t)nb * dn_sm_count();
  if (g > max_ctas) g = max_ctas < 1 ? 1 : max_ctas;
  if (g > kMaxCtas) g = kMaxCtas;
  ImplicitArgs args = a;
  void* params[] = {&args};
  DN_CUDA_TRY(cudaLaunchCooperativeKernel((const void*)kernel, dim3((unsigned)g), dim3(kThreads), params, 0, st));
  DN_LAUNCH_CHECK();
  return DN_OK;
}

}  // namespace dnim
