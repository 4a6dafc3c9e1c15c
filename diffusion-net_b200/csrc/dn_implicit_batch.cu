// Implicit heat diffusion over a mesh batch (dn_implicit_diffusion_fwd_batched / _bwd_batched): for every mesh b and
// channel c (a "pair"), y_bc = (M_b + t_c L_b)^-1 M_b x_bc, by the single-mesh kernel's block Jacobi-PCG
// (dn_implicit_common.cuh, the same row sweeps and scalar updates) in one persistent cooperative launch.
//
// The batch is one row range (batch.MeshBatch): mesh b owns rows [begin_b, end_b), begin_b a multiple of 128, and L is
// block diagonal.  Every pair has its own scalars, freezing and NaN state, so a slow mesh does not change the iterates
// of a fast one.  The rows are cut into 32-row chunks, none of which crosses a mesh; a CTA sweeps its chunks one at a
// time (4 rows per warp) and writes one partial per chunk, so mesh b's sums are its chunks' partials added in a fixed
// order (mesh_sum).  The result therefore does not depend on the grid size, and a CTA can serve many small meshes while
// a large mesh spans many CTAs.  The per-pair scalar updates are spread over every warp of the grid, one pair each, the
// warp's lanes sharing the pair's sums.  Chunks
// whose mesh has no iterating pair are skipped.  Padding rows (past end_b) are never part of a solve: their outputs are
// written as exact zeros.  grad_time[c] adds the meshes' sums in mesh order.  No atomics: two calls give bitwise-equal
// results.
#include "dn_implicit_common.cuh"

namespace cg = cooperative_groups;

namespace {

using namespace dnim;

constexpr int kChunkRows = 32;

struct Chunk {
  int64_t v0, v1;   // its rows of mesh b: [v0, v1), empty for a chunk of padding rows only
  int b;
};

__device__ __forceinline__ Chunk chunk_rows(const ImplicitArgs& a, int64_t ch) {
  Chunk h;
  h.v0 = ch * kChunkRows;
  h.b = __ldg(a.tile_mesh + (h.v0 >> 7));
  const int64_t end = __ldg(a.mesh_rows + 2 * h.b + 1);
  h.v1 = h.v0 + kChunkRows < end ? h.v0 + kChunkRows : end;
  return h;
}

// the sum over mesh b's chunks of partial column c, by one warp: lane l adds chunks c0 + l, c0 + l + 32, ... in order,
// then the lanes are added by a fixed butterfly, which leaves the same total in every lane.  A mesh of n chunks costs
// n / 32 dependent loads per lane, so large meshes do not serialise the scalar updates.
__device__ __forceinline__ double mesh_sum(const ImplicitArgs& a, const double* part, int b, int c, int lane) {
  const int c0 = __ldg(a.mesh_rows + 2 * b) / kChunkRows;
  const int c1 = (__ldg(a.mesh_rows + 2 * b + 1) + kChunkRows - 1) / kChunkRows;
  double s = 0.0;
  for (int g = c0 + lane; g < c1; g += 32) s += ldg_cg(part + (int64_t)g * a.C + c);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

// on[q]: this lane's pair (b, lane + 32 q) is iterating (active > 0) or, with iterating false, converged (active == 0);
// returns whether any lane of the CTA has such a pair (a CTA-wide barrier)
template <int NC>
__device__ __forceinline__ bool lane_pairs(const ImplicitArgs& a, int b, int lane, const bool (&cok)[NC],
                                           bool (&on)[NC], bool iterating) {
  bool any = false;
#pragma unroll
  for (int q = 0; q < NC; ++q) {
    const int s = cok[q] ? ldg_cg(a.active + (int64_t)b * a.C + lane + 32 * q) : 0;
    on[q] = cok[q] && (iterating ? s > 0 : s == 0);
    any |= on[q];
  }
  return __syncthreads_or(any);
}

// the number of iterating pairs, from the per-CTA counts (every thread gets it)
__device__ __forceinline__ int grid_active(const ImplicitArgs& a, int G, int* s_total) {
  if (threadIdx.x < 32) {
    int n = 0;
    for (int g = threadIdx.x; g < G; g += 32) n += ldg_cg(a.n_active + g);
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
    if (threadIdx.x == 0) *s_total = n;
  }
  __syncthreads();
  const int n = *s_total;
  __syncthreads();
  return n;
}

template <int NC>
__global__ void __launch_bounds__(kThreads, min_ctas_per_sm(NC)) implicit_cg_batched_kernel(ImplicitArgs a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ double red[2][kWarps][kMaxC];
  __shared__ int s_act[kWarps];
  __shared__ int s_total;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int G = gridDim.x;
  const int C = a.C;
  const int64_t n_pairs = (int64_t)a.n_meshes * C;
  const int64_t n_chunks = a.V / kChunkRows;
  // the per-pair scalar updates: one warp per pair (its sums are warp-wide), every warp of the grid
  const int64_t pair0 = (int64_t)blockIdx.x * kWarps + warp, pair_stride = (int64_t)G * kWarps;
  double* const part0 = a.part;
  double* const part1 = a.part + n_chunks * C;

  // the clamped time of this lane's channels, as in the single-mesh kernel
  double t[NC];
  bool cok[NC];
#pragma unroll
  for (int q = 0; q < NC; ++q) {
    const int c = lane + 32 * q;
    cok[q] = c < C;
    t[q] = cok[q] ? (double)dn_clamp_time(a.time[c]) : 0.0;
  }

  // ---- init: L_vv, b, x = 0, r = b, p = z = r / d; chunk partials of b.b and r.z
  double acc0[NC], acc1[NC];
  for (int64_t ch = blockIdx.x; ch < n_chunks; ch += G) {
    const Chunk h = chunk_rows(a, ch);
    if (h.v1 <= h.v0) continue;
#pragma unroll
    for (int q = 0; q < NC; ++q) acc0[q] = acc1[q] = 0.0;
    for (int64_t v = h.v0 + warp; v < h.v1; v += kWarps) row_init<NC>(a, v, lane, t, cok, acc0, acc1);
    cta_partial<NC>(red[0], acc0, C, part0 + ch * C);
    cta_partial<NC>(red[1], acc1, C, part1 + ch * C);
  }
  grid.sync();
  {
    const PairCols k = pair_cols(a.col, n_pairs);
    int act = 0;
    for (int64_t p = pair0; p < n_pairs; p += pair_stride) {
      const int b = (int)(p / C), c = (int)(p % C);
      const double bb = mesh_sum(a, part0, b, c, lane), rzv = mesh_sum(a, part1, b, c, lane);
      if (lane == 0) act += pair_start(k, a.active, p, bb, rzv);
    }
    act = cta_total(act, s_act);
    if (threadIdx.x == 0) a.n_active[blockIdx.x] = act;
  }
  grid.sync();
  int n_act = grid_active(a, G, &s_total);

  int n_iter = 0;
  for (; n_iter < a.max_iter && n_act > 0;) {
    bool on[NC];
    // ---- q = M p + t (L p), partial p.q
    for (int64_t ch = blockIdx.x; ch < n_chunks; ch += G) {
      const Chunk h = chunk_rows(a, ch);
      if (h.v1 <= h.v0 || !lane_pairs<NC>(a, h.b, lane, cok, on, true)) continue;
#pragma unroll
      for (int q = 0; q < NC; ++q) acc0[q] = 0.0;
      for (int64_t v = h.v0 + warp; v < h.v1; v += kWarps) row_apply<NC>(a, v, lane, t, on, acc0);
      cta_partial<NC>(red[0], acc0, C, part0 + ch * C);
    }
    grid.sync();
    {
      const PairCols k = pair_cols(a.col, n_pairs);
      for (int64_t p = pair0; p < n_pairs; p += pair_stride)
        if (ldg_cg(a.active + p) > 0) {
          const double pq = mesh_sum(a, part0, (int)(p / C), (int)(p % C), lane);
          if (lane == 0) pair_alpha(k, p, pq);
        }
    }
    grid.sync();

    // ---- x += alpha p, r -= alpha q; partials r.r and r.z
    for (int64_t ch = blockIdx.x; ch < n_chunks; ch += G) {
      const Chunk h = chunk_rows(a, ch);
      if (h.v1 <= h.v0 || !lane_pairs<NC>(a, h.b, lane, cok, on, true)) continue;
      double al[NC];
#pragma unroll
      for (int q = 0; q < NC; ++q) {
        al[q] = on[q] ? ldg_cg(a.col + 2 * n_pairs + (int64_t)h.b * C + lane + 32 * q) : 0.0;
        acc0[q] = acc1[q] = 0.0;
      }
      for (int64_t v = h.v0 + warp; v < h.v1; v += kWarps) row_update<NC>(a, v, lane, t, on, al, acc0, acc1);
      cta_partial<NC>(red[0], acc0, C, part0 + ch * C);
      cta_partial<NC>(red[1], acc1, C, part1 + ch * C);
    }
    grid.sync();
    {
      const PairCols k = pair_cols(a.col, n_pairs);
      int act = 0;
      for (int64_t p = pair0; p < n_pairs; p += pair_stride)
        if (ldg_cg(a.active + p) > 0) {
          const int b = (int)(p / C), c = (int)(p % C);
          const double r2 = mesh_sum(a, part0, b, c, lane), rzn = mesh_sum(a, part1, b, c, lane);
          if (lane == 0) act += pair_step(k, a.active, p, r2, rzn, a.rtol);
        }
      act = cta_total(act, s_act);
      if (threadIdx.x == 0) a.n_active[blockIdx.x] = act;
    }
    grid.sync();
    ++n_iter;
    n_act = grid_active(a, G, &s_total);
    if (n_act == 0) break;

    // ---- p = r / d + beta p
    for (int64_t ch = blockIdx.x; ch < n_chunks; ch += G) {
      const Chunk h = chunk_rows(a, ch);
      if (h.v1 <= h.v0 || !lane_pairs<NC>(a, h.b, lane, cok, on, true)) continue;
      double be[NC];
#pragma unroll
      for (int q = 0; q < NC; ++q) be[q] = on[q] ? ldg_cg(a.col + 3 * n_pairs + (int64_t)h.b * C + lane + 32 * q) : 0.0;
      for (int64_t v = h.v0 + warp; v < h.v1; v += kWarps) row_direction<NC>(a, v, lane, t, on, be);
    }
    grid.sync();
  }

  // ---- status, then the outputs only when every pair converged.  Every iteration advanced the pairs that were still
  // iterating, and a pair never resumes, so the largest per-pair iteration count is the number of iterations run.
  {
    const PairCols k = pair_cols(a.col, n_pairs);
    for (int64_t p = pair0; p < n_pairs; p += pair_stride)
      if (lane == 0) pair_status(k, a.active, a.status, n_pairs, p);
  }
  if (blockIdx.x == 0) {
    if (threadIdx.x == 0) {
      a.status[0] = (double)n_act;
      a.status[1] = (double)n_iter;
    }
    if (!a.backward)   // the clamp write-back (reference layers.py:48-49), every CTA has read `time` by now
      for (int c = threadIdx.x; c < C; c += kThreads) a.time[c] = dn_clamp_time(a.time[c]);
  }
  if (n_act) return;

  // on[q]: this lane's pair is written from x; a non-finite pair is written as NaN; padding rows are 0
  bool on[NC];
  if (!a.backward) {
    for (int64_t ch = blockIdx.x; ch < n_chunks; ch += G) {
      const Chunk h = chunk_rows(a, ch);
      lane_pairs<NC>(a, h.b, lane, cok, on, false);
      for (int64_t v = h.v0 + warp; v < h.v0 + kChunkRows; v += kWarps) {
        if (v < h.v1) {
          row_write_fwd<NC>(a, v, lane, cok, on);
        } else {
#pragma unroll
          for (int q = 0; q < NC; ++q)
            if (cok[q]) a.out[v * C + lane + 32 * q] = 0.f;
        }
      }
    }
    return;
  }
  // backward: grad_x = M w; grad_time[c] += -sum_b sum_v w[v][bc] (L y)[v][bc]
  for (int64_t ch = blockIdx.x; ch < n_chunks; ch += G) {
    const Chunk h = chunk_rows(a, ch);
    lane_pairs<NC>(a, h.b, lane, cok, on, false);
#pragma unroll
    for (int q = 0; q < NC; ++q) acc0[q] = 0.0;
    for (int64_t v = h.v0 + warp; v < h.v0 + kChunkRows; v += kWarps) {
      if (v < h.v1) {
        row_write_bwd<NC>(a, v, lane, cok, on, acc0);
      } else {
#pragma unroll
        for (int q = 0; q < NC; ++q)
          if (cok[q]) a.out[v * C + lane + 32 * q] = 0.f;
      }
    }
    if (h.v1 > h.v0) cta_partial<NC>(red[0], acc0, C, part0 + ch * C);
  }
  grid.sync();
  // each pair's sum over its mesh, in the alpha slot
  for (int64_t p = pair0; p < n_pairs; p += pair_stride) {
    const double s = mesh_sum(a, part0, (int)(p / C), (int)(p % C), lane);
    if (lane == 0) a.col[2 * n_pairs + p] = s;
  }
  grid.sync();
  if (blockIdx.x == 0)
    for (int c = threadIdx.x; c < C; c += kThreads) {
      double s = 0.0;
      bool finite = true;
      for (int b = 0; b < a.n_meshes; ++b) {
        s += ldg_cg(a.col + 2 * n_pairs + (int64_t)b * C + c);
        finite &= ldg_cg(a.active + (int64_t)b * C + c) == 0;
      }
      a.grad_time[c] += finite ? (float)(-s) : __int_as_float(0x7fc00000);
    }
}

template <int NC>
int launch_nc(const ImplicitArgs& a, cudaStream_t st) {
  return launch_cooperative(implicit_cg_batched_kernel<NC>, a, a.V / kChunkRows, st);
}

}  // namespace

int64_t implicit_batched_ws_bytes(int64_t V, int C, int n_meshes) {
  const int64_t pairs = (int64_t)n_meshes * C;
  return 8 * (4 * V * C + V + 2 * (V / kChunkRows) * C + 6 * pairs) + 4 * (pairs + kMaxCtas) + 1024;
}

int launch_implicit_diffusion_batched(const dn_csr* L, const float* mass, float* time, const float* rhs, const float* y,
                                      const dn_mesh_batch* batch, const int32_t* mesh_rows, int64_t V, int C,
                                      double rtol, int max_iter, int backward, float* out, float* grad_time,
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
  a.n_meshes = batch->n_meshes;
  a.tile_mesh = batch->tile_mesh;
  a.mesh_rows = mesh_rows;
  const int64_t pairs = (int64_t)batch->n_meshes * C;
  double* w = (double*)(((uintptr_t)ws + 255) & ~(uintptr_t)255);
  const int64_t vc = V * C;
  a.X = w;
  a.R = w + vc;
  a.P = w + 2 * vc;
  a.Q = w + 3 * vc;
  a.ldiag = w + 4 * vc;
  a.part = a.ldiag + V;
  a.col = a.part + 2 * (V / kChunkRows) * C;
  a.active = (int*)(a.col + 6 * pairs);
  a.n_active = a.active + pairs;
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
