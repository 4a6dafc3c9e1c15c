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
#include "dn_implicit_common.cuh"

namespace cg = cooperative_groups;

namespace {

using namespace dnim;

template <int NC>
__global__ void __launch_bounds__(kThreads, min_ctas_per_sm(NC)) implicit_cg_kernel(ImplicitArgs a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ double red[2][kWarps][kMaxC];
  __shared__ int s_act[kWarps];
  const int lane = threadIdx.x & 31;
  const int G = gridDim.x;
  const int64_t warp0 = ((int64_t)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const int64_t n_warps = (int64_t)G * kWarps;
  const int C = a.C;
  const int64_t V = a.V;
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
    t[q] = cok[q] ? (double)dn_clamp_time(a.time[c]) : 0.0;
  }

  // ---- init: L_vv, b, x = 0, r = b, p = z = r / d; partials of b.b and r.z
  double acc0[NC], acc1[NC];
#pragma unroll
  for (int q = 0; q < NC; ++q) acc0[q] = acc1[q] = 0.0;
  for (int64_t v = warp0; v < V; v += n_warps) row_init<NC>(a, v, lane, t, cok, acc0, acc1);
  cta_partial<NC>(red[0], acc0, C, part0 + (int64_t)blockIdx.x * C);
  cta_partial<NC>(red[1], acc1, C, part1 + (int64_t)blockIdx.x * C);
  grid.sync();
  if (first_cta) {
    const PairCols k = pair_cols(a.col, C);
    int act = 0;
    for (int c = threadIdx.x; c < C; c += kThreads)
      act += pair_start(k, a.active, c, slot_sum(part0, 0, G, C, c), slot_sum(part1, 0, G, C, c));
    act = cta_total(act, s_act);
    if (threadIdx.x == 0) *a.n_active = act;
  }
  grid.sync();

  for (int it = 0; it < a.max_iter && ldg_cg(a.n_active) > 0; ++it) {
    bool on[NC];
#pragma unroll
    for (int q = 0; q < NC; ++q) on[q] = cok[q] && ldg_cg(a.active + lane + 32 * q) > 0;

    // ---- q = M p + t (L p), partial p.q
#pragma unroll
    for (int q = 0; q < NC; ++q) acc0[q] = 0.0;
    for (int64_t v = warp0; v < V; v += n_warps) row_apply<NC>(a, v, lane, t, on, acc0);
    cta_partial<NC>(red[0], acc0, C, part0 + (int64_t)blockIdx.x * C);
    grid.sync();
    if (first_cta)
      for (int c = threadIdx.x; c < C; c += kThreads)
        if (a.active[c] > 0) pair_alpha(pair_cols(a.col, C), c, slot_sum(part0, 0, G, C, c));
    grid.sync();

    // ---- x += alpha p, r -= alpha q; partials r.r and r.z
    double al[NC];
#pragma unroll
    for (int q = 0; q < NC; ++q) {
      al[q] = on[q] ? ldg_cg(a.col + 2 * C + lane + 32 * q) : 0.0;
      acc0[q] = acc1[q] = 0.0;
    }
    for (int64_t v = warp0; v < V; v += n_warps) row_update<NC>(a, v, lane, t, on, al, acc0, acc1);
    cta_partial<NC>(red[0], acc0, C, part0 + (int64_t)blockIdx.x * C);
    cta_partial<NC>(red[1], acc1, C, part1 + (int64_t)blockIdx.x * C);
    grid.sync();
    if (first_cta) {
      const PairCols k = pair_cols(a.col, C);
      int act = 0;
      for (int c = threadIdx.x; c < C; c += kThreads)
        if (a.active[c] > 0)
          act += pair_step(k, a.active, c, slot_sum(part0, 0, G, C, c), slot_sum(part1, 0, G, C, c), a.rtol);
      act = cta_total(act, s_act);
      if (threadIdx.x == 0) *a.n_active = act;
    }
    grid.sync();
    if (ldg_cg(a.n_active) == 0) break;

    // ---- p = r / d + beta p
    double be[NC];
#pragma unroll
    for (int q = 0; q < NC; ++q) {
      on[q] = cok[q] && ldg_cg(a.active + lane + 32 * q) > 0;
      be[q] = on[q] ? ldg_cg(a.col + 3 * C + lane + 32 * q) : 0.0;
    }
    for (int64_t v = warp0; v < V; v += n_warps) row_direction<NC>(a, v, lane, t, on, be);
    grid.sync();
  }

  // ---- status, then the outputs only when every column converged
  const int unconverged = ldg_cg(a.n_active);
  if (first_cta) {
    const PairCols k = pair_cols(a.col, C);
    double worst_it = 0.0;
    for (int c = threadIdx.x; c < C; c += kThreads) worst_it = fmax(worst_it, pair_status(k, a.active, a.status, C, c));
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
      for (int c = threadIdx.x; c < C; c += kThreads) a.time[c] = dn_clamp_time(a.time[c]);
  }
  if (unconverged) return;

  // on[q]: this lane's column q is written from x; a non-finite column is written as NaN
  bool on[NC];
#pragma unroll
  for (int q = 0; q < NC; ++q) on[q] = cok[q] && ldg_cg(a.active + lane + 32 * q) == 0;
  if (!a.backward) {
    for (int64_t v = warp0; v < V; v += n_warps) row_write_fwd<NC>(a, v, lane, cok, on);
    return;
  }
  // backward: grad_x = M w; grad_time[c] += -sum_v w[v][c] (L y)[v][c]
#pragma unroll
  for (int q = 0; q < NC; ++q) acc0[q] = 0.0;
  for (int64_t v = warp0; v < V; v += n_warps) row_write_bwd<NC>(a, v, lane, cok, on, acc0);
  cta_partial<NC>(red[0], acc0, C, part0 + (int64_t)blockIdx.x * C);
  grid.sync();
  if (first_cta)
    for (int c = threadIdx.x; c < C; c += kThreads)
      a.grad_time[c] += ldg_cg(a.active + c) == 0 ? (float)(-slot_sum(part0, 0, G, C, c))
                                                  : __int_as_float(0x7fc00000);
}

template <int NC>
int launch_nc(const ImplicitArgs& a, cudaStream_t st) {
  return launch_cooperative(implicit_cg_kernel<NC>, a, (a.V + kWarps - 1) / kWarps, st);   // no CTA without a row
}

}  // namespace

int64_t implicit_ws_bytes(int64_t V, int C) {
  return 8 * (4 * V * C + V + 2ll * kMaxCtas * C + 6ll * C) + 4ll * (C + 1) + 1024;
}

int launch_implicit_diffusion(const dn_csr* L, const float* mass, float* time, const float* rhs, const float* y,
                              int64_t V, int C, double rtol, int max_iter, int backward, float* out, float* grad_time,
                              double* status, void* ws, cudaStream_t st) {
  if (C > kMaxC) return DN_ERR_UNSUPPORTED;
  ImplicitArgs a{};
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
