// Implicit heat diffusion (reference layers.py:69-84, method='implicit_dense'): per channel c,
//   y_c = (M + t_c L)^-1 M x_c,
// solved for all C columns at once by a block Jacobi-preconditioned conjugate gradient on the Laplacian's CSR, with
// per-column shifts t_c, step lengths alpha_c / beta_c and preconditioner d[v][c] = m_v + t_c L_vv.  The solver state
// (x, r, p, q) and every reduction are fp64; L's and the mass's fp32 values are promoted exactly and used as given.
//
// One persistent cooperative kernel per solve: the CTAs sweep the rows (one warp per row, lane l owning columns
// l, l + 32, ...) between grid-wide barriers, and the per-column scalars are reduced by the first CTA between two
// barriers.  Convergence is decided on the device per column: a column with ||r_c|| <= rtol ||b_c|| is frozen (its x is
// never touched again), so the result does not depend on the other columns or on anything the host does.  Every
// reduction over V is a per-CTA partial (warps added in a fixed order) followed by a sum over the CTAs in index order,
// with no atomics: two calls on the same device give bitwise-equal results.
//
// A column whose b_c is not finite (a NaN or inf in x or grad_out, a NaN mass entry), or whose p.q, alpha, r.r or r.z
// turns non-finite during the iteration (an inf in the data, a NaN in L), is frozen at once with a NaN result, as the
// reference's dense solve returns NaN: active[c] = -1, where 1 is iterating and 0 converged.  It does not count as
// unconverged, so the other columns are still written.
//
// Data written by other CTAs inside the kernel is read with ld.global.cg (L2), never through the non-coherent L1 or
// read-only paths.
#include <cooperative_groups.h>

#include "dn_internal.h"

namespace cg = cooperative_groups;

namespace {

constexpr int kThreads = 256, kWarps = kThreads / 32, kMaxCtas = 1024, kMaxC = 256;

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
  double* status;           // 2 + 2C, see the header
  double *X, *R, *P, *Q;    // V x C each
  double* ldiag;            // V
  double* part;             // 2 x kMaxCtas x C
  double* col;              // 6 x C: rz, |b|, alpha, beta, r.r, and the iteration count
  int* active;              // C: 1 iterating, 0 converged, -1 non-finite (NaN result)
  int* n_active;            // 1
};

__device__ __forceinline__ double ldg_cg(const double* p) { return __ldcg(p); }
__device__ __forceinline__ int ldg_cg(const int* p) { return __ldcg(p); }

// Sum the per-warp partials of this CTA in warp order and store them as this CTA's partial (columns < C).
template <int NC>
__device__ void cta_partial(double (*red)[kMaxC], const double* acc, int C, double* part_out) {
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
    part_out[(int64_t)blockIdx.x * C + c] = s;
  }
  __syncthreads();
}

// sum over CTAs in index order of partial column c
__device__ __forceinline__ double cta_sum(const double* part, int G, int C, int c) {
  double s = 0.0;
  for (int g = 0; g < G; ++g) s += ldg_cg(part + (int64_t)g * C + c);
  return s;
}

template <int NC>
__global__ void __launch_bounds__(kThreads) implicit_cg_kernel(ImplicitArgs a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ double red[2][kWarps][kMaxC];
  __shared__ int s_act[kWarps];
  const int lane = threadIdx.x & 31;
  const int G = gridDim.x;
  const int64_t warp0 = ((int64_t)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const int64_t n_warps = (int64_t)G * kWarps;
  const int C = a.C;
  const int64_t V = a.V;
  double* const rz = a.col;
  double* const bnorm = a.col + C;
  double* const alpha = a.col + 2 * C;
  double* const beta = a.col + 3 * C;
  double* const rr = a.col + 4 * C;
  double* const iters = a.col + 5 * C;
  double* const part0 = a.part;
  double* const part1 = a.part + (int64_t)kMaxCtas * C;
  const bool first_cta = blockIdx.x == 0;

  // the clamped time of this lane's columns (torch.clamp(t, min=1e-8), layers.py:48-49); `time` is only written back at
  // the very end, after every CTA has read it
  double t[NC];
  bool cok[NC];
#pragma unroll
  for (int q = 0; q < NC; ++q) {
    const int c = lane + 32 * q;
    cok[q] = c < C;
    t[q] = cok[q] ? (double)fmaxf(a.time[c], 1e-8f) : 0.0;
  }

  // ---- init: L_vv, b, x = 0, r = b, p = z = r / d; partials of b.b and r.z
  double acc0[NC], acc1[NC];
#pragma unroll
  for (int q = 0; q < NC; ++q) acc0[q] = acc1[q] = 0.0;
  for (int64_t v = warp0; v < V; v += n_warps) {
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
      const double z = b / (m + t[q] * dg);
      a.X[i] = 0.0;
      a.R[i] = b;
      a.P[i] = z;
      acc0[q] = fma(b, b, acc0[q]);
      acc1[q] = fma(b, z, acc1[q]);
    }
  }
  cta_partial<NC>(red[0], acc0, C, part0);
  cta_partial<NC>(red[1], acc1, C, part1);
  grid.sync();
  if (first_cta) {
    int act = 0;
    for (int c = threadIdx.x; c < C; c += kThreads) {
      const double bb = cta_sum(part0, G, C, c);
      bnorm[c] = sqrt(bb);
      rz[c] = cta_sum(part1, G, C, c);
      rr[c] = bb;
      iters[c] = 0.0;
      const int live = bb > 0.0;        // b_c = 0: x_c = 0 is exact
      a.active[c] = isfinite(bb) ? live : -1;
      act += live && isfinite(bb);
    }
    for (int o = 16; o > 0; o >>= 1) act += __shfl_xor_sync(0xffffffffu, act, o);
    if (lane == 0) s_act[threadIdx.x >> 5] = act;
    __syncthreads();
    if (threadIdx.x == 0) {
      int n = 0;
      for (int w = 0; w < kWarps; ++w) n += s_act[w];
      *a.n_active = n;
    }
  }
  grid.sync();

  for (int it = 0; it < a.max_iter && ldg_cg(a.n_active) > 0; ++it) {
    bool on[NC];
#pragma unroll
    for (int q = 0; q < NC; ++q) on[q] = cok[q] && ldg_cg(a.active + lane + 32 * q) > 0;

    // ---- q = M p + t (L p), partial p.q
#pragma unroll
    for (int q = 0; q < NC; ++q) acc0[q] = 0.0;
    for (int64_t v = warp0; v < V; v += n_warps) {
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
    cta_partial<NC>(red[0], acc0, C, part0);
    grid.sync();
    if (first_cta)
      for (int c = threadIdx.x; c < C; c += kThreads)
        if (a.active[c] > 0) alpha[c] = rz[c] / cta_sum(part0, G, C, c);
    grid.sync();

    // ---- x += alpha p, r -= alpha q; partials r.r and r.z
    double al[NC];
#pragma unroll
    for (int q = 0; q < NC; ++q) {
      al[q] = on[q] ? ldg_cg(alpha + lane + 32 * q) : 0.0;
      acc0[q] = acc1[q] = 0.0;
    }
    for (int64_t v = warp0; v < V; v += n_warps) {
      const double m = (double)a.mass[v], dg = ldg_cg(a.ldiag + v);
#pragma unroll
      for (int q = 0; q < NC; ++q) {
        if (!on[q]) continue;
        const int64_t i = v * C + lane + 32 * q;
        a.X[i] = fma(al[q], a.P[i], a.X[i]);
        const double r = fma(-al[q], a.Q[i], a.R[i]);
        a.R[i] = r;
        acc0[q] = fma(r, r, acc0[q]);
        acc1[q] = fma(r, r / (m + t[q] * dg), acc1[q]);
      }
    }
    cta_partial<NC>(red[0], acc0, C, part0);
    cta_partial<NC>(red[1], acc1, C, part1);
    grid.sync();
    if (first_cta) {
      int act = 0;
      for (int c = threadIdx.x; c < C; c += kThreads) {
        if (a.active[c] <= 0) continue;
        const double r2 = cta_sum(part0, G, C, c), rzn = cta_sum(part1, G, C, c);
        rr[c] = r2;
        iters[c] += 1.0;
        if (!(isfinite(alpha[c]) && isfinite(r2) && isfinite(rzn))) {   // p.q or the data went non-finite
          a.active[c] = -1;
        } else if (sqrt(r2) <= a.rtol * bnorm[c]) {
          a.active[c] = 0;              // frozen: x_c is final
        } else {
          beta[c] = rzn / rz[c];
          rz[c] = rzn;
          ++act;
        }
      }
      for (int o = 16; o > 0; o >>= 1) act += __shfl_xor_sync(0xffffffffu, act, o);
      if (lane == 0) s_act[threadIdx.x >> 5] = act;
      __syncthreads();
      if (threadIdx.x == 0) {
        int n = 0;
        for (int w = 0; w < kWarps; ++w) n += s_act[w];
        *a.n_active = n;
      }
    }
    grid.sync();
    if (ldg_cg(a.n_active) == 0) break;

    // ---- p = r / d + beta p
    double be[NC];
#pragma unroll
    for (int q = 0; q < NC; ++q) {
      on[q] = cok[q] && ldg_cg(a.active + lane + 32 * q) > 0;
      be[q] = on[q] ? ldg_cg(beta + lane + 32 * q) : 0.0;
    }
    for (int64_t v = warp0; v < V; v += n_warps) {
      const double m = (double)a.mass[v], dg = ldg_cg(a.ldiag + v);
#pragma unroll
      for (int q = 0; q < NC; ++q) {
        if (!on[q]) continue;
        const int64_t i = v * C + lane + 32 * q;
        a.P[i] = fma(be[q], a.P[i], a.R[i] / (m + t[q] * dg));
      }
    }
    grid.sync();
  }

  // ---- status, then the outputs only when every column converged
  const int unconverged = ldg_cg(a.n_active);
  if (first_cta) {
    double worst_it = 0.0;
    for (int c = threadIdx.x; c < C; c += kThreads) {
      const double itc = ldg_cg(iters + c);
      a.status[2 + c] = itc;
      const double bn = ldg_cg(bnorm + c);
      a.status[2 + C + c] = ldg_cg(a.active + c) < 0 ? __longlong_as_double(0x7ff8000000000000ll)
                            : bn > 0.0              ? sqrt(ldg_cg(rr + c)) / bn
                                                    : 0.0;
      worst_it = fmax(worst_it, itc);
    }
    for (int o = 16; o > 0; o >>= 1) worst_it = fmax(worst_it, __shfl_xor_sync(0xffffffffu, worst_it, o));
    __shared__ double s_it[kWarps];
    if (lane == 0) s_it[threadIdx.x >> 5] = worst_it;
    __syncthreads();
    if (threadIdx.x == 0) {
      double w = 0.0;
      for (int i = 0; i < kWarps; ++i) w = fmax(w, s_it[i]);
      a.status[0] = (double)unconverged;
      a.status[1] = w;
    }
    if (!a.backward)   // the clamp write-back (reference layers.py:48-49), every CTA has read `time` by now
      for (int c = threadIdx.x; c < C; c += kThreads) a.time[c] = fmaxf(a.time[c], 1e-8f);
  }
  if (unconverged) return;

  // on[q]: this lane's column q is written from x; a non-finite column is written as NaN
  const float fnan = __int_as_float(0x7fc00000);
  bool on[NC];
#pragma unroll
  for (int q = 0; q < NC; ++q) on[q] = cok[q] && ldg_cg(a.active + lane + 32 * q) == 0;
  if (!a.backward) {
    for (int64_t v = warp0; v < V; v += n_warps)
#pragma unroll
      for (int q = 0; q < NC; ++q)
        if (cok[q]) a.out[v * C + lane + 32 * q] = on[q] ? (float)a.X[v * C + lane + 32 * q] : fnan;
    return;
  }
  // backward: grad_x = M w; grad_time[c] += -sum_v w[v][c] (L y)[v][c]
#pragma unroll
  for (int q = 0; q < NC; ++q) acc0[q] = 0.0;
  for (int64_t v = warp0; v < V; v += n_warps) {
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
  cta_partial<NC>(red[0], acc0, C, part0);
  grid.sync();
  if (first_cta)
    for (int c = threadIdx.x; c < C; c += kThreads)
      a.grad_time[c] += ldg_cg(a.active + c) == 0 ? (float)(-cta_sum(part0, G, C, c)) : fnan;
}

template <int NC>
int launch_nc(const ImplicitArgs& a, cudaStream_t st) {
  int nb = 0;
  DN_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, implicit_cg_kernel<NC>, kThreads, 0));
  if (nb < 1) return DN_ERR_UNSUPPORTED;
  int64_t g = (int64_t)nb * dn_sm_count();
  const int64_t rows_needed = (a.V + kWarps - 1) / kWarps;   // no CTA without a row
  if (g > rows_needed) g = rows_needed < 1 ? 1 : rows_needed;
  if (g > kMaxCtas) g = kMaxCtas;
  ImplicitArgs args = a;
  void* params[] = {&args};
  DN_CUDA_TRY(cudaLaunchCooperativeKernel((const void*)implicit_cg_kernel<NC>, dim3((unsigned)g), dim3(kThreads), params,
                                          0, st));
  DN_LAUNCH_CHECK();
  return DN_OK;
}

}  // namespace

int64_t implicit_ws_bytes(int64_t V, int C) {
  return 8 * (4 * V * C + V + 2ll * kMaxCtas * C + 6ll * C) + 4ll * (C + 1) + 1024;
}

int launch_implicit_diffusion(const dn_csr* L, const float* mass, float* time, const float* rhs, const float* y,
                              int64_t V, int C, double rtol, int max_iter, int backward, float* out, float* grad_time,
                              double* status, void* ws, cudaStream_t st) {
  if (C > kMaxC) return DN_ERR_UNSUPPORTED;
  ImplicitArgs a;
  a.rowptr = L->rowptr;
  a.colidx = L->colidx;
  a.lvals = L->vals;
  a.mass = mass;
  a.time = time;
  a.rhs = rhs;
  a.y = y;
  a.V = V;
  a.C = C;
  a.backward = backward;
  a.rtol = rtol;
  a.max_iter = max_iter;
  a.out = out;
  a.grad_time = grad_time;
  a.status = status;
  double* w = (double*)(((uintptr_t)ws + 255) & ~(uintptr_t)255);
  const int64_t vc = V * C;
  a.X = w;
  a.R = w + vc;
  a.P = w + 2 * vc;
  a.Q = w + 3 * vc;
  a.ldiag = w + 4 * vc;
  a.part = a.ldiag + V;
  a.col = a.part + 2ll * kMaxCtas * C;
  a.active = (int*)(a.col + 6ll * C);
  a.n_active = a.active + C;
  switch ((C + 31) / 32) {
    case 1: return launch_nc<1>(a, st);
    case 2: return launch_nc<2>(a, st);
    case 3: return launch_nc<3>(a, st);
    case 4: return launch_nc<4>(a, st);
    case 5: return launch_nc<5>(a, st);
    case 6: return launch_nc<6>(a, st);
    case 7: return launch_nc<7>(a, st);
    default: return launch_nc<8>(a, st);
  }
}
