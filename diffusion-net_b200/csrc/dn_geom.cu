// Kernels for the two data-side neighbours of the block (SURVEY.md section 8f, items 2 and 3):
//   * heat-kernel-signature input features   (reference geometry.py:600-628, compute_hks)
//   * CSC (the reference's on-disk operator cache, geometry.py:548-568) -> device CSR, i.e. a sparse transpose
// Both are HBM-bound index/streaming work: plain coalesced SIMT, no tensor cores.
#include "dn_internal.h"

namespace {

// ---------------------------------------------------------------------------------------------
// HKS: out[v][s] = sum_k exp(-evals[k] * scales[s]) * evecs[v][k]^2
// Fast path (K = 32*KPL, S <= 16): one warp per vertex row, lane l owns k = l + 32 j.  The (k, s) coefficient
// table lives in registers (KPL*16 per lane), the row of evecs is read once, coalesced, and the 16 per-lane
// partial sums are reduced with a transposed butterfly (16 shuffles instead of 16 * 5).
// ---------------------------------------------------------------------------------------------
template <int KPL>
__global__ void __launch_bounds__(256) hks_warp_kernel(const float* __restrict__ evals, const float* __restrict__ evecs,
                                                        const float* __restrict__ scales, int64_t V, int S,
                                                        float* __restrict__ out) {
  constexpr int K = 32 * KPL;
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  float coef[KPL][16];
#pragma unroll
  for (int j = 0; j < KPL; ++j) {
    const float ev = evals[lane + 32 * j];
#pragma unroll
    for (int s = 0; s < 16; ++s) coef[j][s] = (s < S) ? expf(-(ev * scales[s < S ? s : 0])) : 0.f;
  }
  const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4, b1 = lane & 2;
  const int s_mine = (b4 ? 8 : 0) + (b3 ? 4 : 0) + (b2 ? 2 : 0) + (b1 ? 1 : 0);
  constexpr int RB = 4;                       // rows per warp iteration: 4 x K x 4 bytes of loads in flight per warp
  for (int64_t row0 = warp * RB; row0 < V; row0 += nwarps * RB) {
    float phi2[RB][KPL];
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      const bool ok = row0 + r < V;
      const float* p = evecs + (row0 + r) * K + lane;
#pragma unroll
      for (int j = 0; j < KPL; ++j) {
        const float f = ok ? __ldg(p + 32 * j) : 0.f;
        phi2[r][j] = f * f;
      }
    }
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      float a[16];
#pragma unroll
      for (int s = 0; s < 16; ++s) {
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < KPL; ++j) acc = fmaf(coef[j][s], phi2[r][j], acc);
        a[s] = acc;
      }
      float b[8], c[4], d[2];
#pragma unroll
      for (int i = 0; i < 8; ++i)
        b[i] = (b4 ? a[i + 8] : a[i]) + __shfl_xor_sync(0xffffffffu, b4 ? a[i] : a[i + 8], 16);
#pragma unroll
      for (int i = 0; i < 4; ++i)
        c[i] = (b3 ? b[i + 4] : b[i]) + __shfl_xor_sync(0xffffffffu, b3 ? b[i] : b[i + 4], 8);
#pragma unroll
      for (int i = 0; i < 2; ++i)
        d[i] = (b2 ? c[i + 2] : c[i]) + __shfl_xor_sync(0xffffffffu, b2 ? c[i] : c[i + 2], 4);
      float e = (b1 ? d[1] : d[0]) + __shfl_xor_sync(0xffffffffu, b1 ? d[0] : d[1], 2);
      e += __shfl_xor_sync(0xffffffffu, e, 1);
      if (!(lane & 1) && s_mine < S && row0 + r < V) out[(row0 + r) * S + s_mine] = e;
    }
  }
}

// any K, S: one warp per row, one scale at a time
__global__ void hks_generic_kernel(const float* __restrict__ evals, const float* __restrict__ evecs,
                                   const float* __restrict__ scales, int64_t V, int K, int S,
                                   float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= V) return;
  for (int s = 0; s < S; ++s) {
    const float t = scales[s];
    float acc = 0.f;
    for (int k = lane; k < K; k += 32) {
      const float f = __ldg(evecs + row * K + k);
      acc = fmaf(expf(-(evals[k] * t)), f * f, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) out[row * S + s] = acc;
  }
}

// ---------------------------------------------------------------------------------------------
// sparse transpose of the shared-pattern CSR (int32 indices, interleaved (x, y) values)
// ---------------------------------------------------------------------------------------------
__global__ void tr_count_kernel(const int32_t* __restrict__ colidx, int64_t nnz, int32_t* __restrict__ cnt) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < nnz) atomicAdd(cnt + colidx[p] + 1, 1);
}

// in-place exclusive scan of n ints by one block (n = V + 1; prep-time, ~tens of microseconds at V = 200k)
__global__ void __launch_bounds__(1024) tr_scan_kernel(int32_t* __restrict__ a, int64_t n) {
  __shared__ int32_t part[1024];
  const int t = threadIdx.x;
  const int64_t chunk = (n + 1023) / 1024;
  const int64_t lo = t * chunk, hi = (lo + chunk < n) ? lo + chunk : n;
  int32_t s = 0;
  for (int64_t i = lo; i < hi; ++i) s += a[i];
  part[t] = s;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const int32_t v = (t >= o) ? part[t - o] : 0;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  int32_t run = part[t] - s;   // exclusive prefix of this thread's chunk; a[] holds counts shifted by one, so an
  for (int64_t i = lo; i < hi; ++i) {   // INCLUSIVE scan of a[] is the exclusive scan of the counts
    run += a[i];
    a[i] = run;
  }
}

__global__ void tr_fill_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                               const float2* __restrict__ vals, int64_t V, const int32_t* __restrict__ rowptr_t,
                               int32_t* __restrict__ cursor, int32_t* __restrict__ colidx_t,
                               float2* __restrict__ vals_t) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= V) return;
  const int s = rowptr[row], e = rowptr[row + 1];
  for (int p = s; p < e; ++p) {
    const int c = colidx[p];
    const int dst = rowptr_t[c] + atomicAdd(cursor + c, 1);
    colidx_t[dst] = (int32_t)row;
    vals_t[dst] = vals[p];
  }
}

// the atomics above land entries of one output row in arbitrary order: sort each row by column (rows are short --
// vertex degree + 1 on meshes, 31 on point clouds -- so one thread per row with an insertion sort)
__global__ void tr_sort_rows_kernel(const int32_t* __restrict__ rowptr_t, int64_t V, int32_t* __restrict__ colidx_t,
                                    float2* __restrict__ vals_t) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= V) return;
  const int s = rowptr_t[row], e = rowptr_t[row + 1];
  for (int i = s + 1; i < e; ++i) {
    const int32_t ck = colidx_t[i];
    const float2 vk = vals_t[i];
    int j = i - 1;
    while (j >= s && colidx_t[j] > ck) {
      colidx_t[j + 1] = colidx_t[j];
      vals_t[j + 1] = vals_t[j];
      --j;
    }
    colidx_t[j + 1] = ck;
    vals_t[j + 1] = vk;
  }
}

// ---------------------------------------------------------------------------------------------
// build_grad (reference geometry.py:198-273): per-vertex least-squares tangent gradient operator, straight into the
// shared-pattern device CSR.  The reference's version is a pure-Python loop over vertices (44 % of its precompute
// time, SURVEY.md 8f-4); here: count / scan / scatter / per-row sort (deterministic column order), then one thread
// per vertex solves the regularised 2x2 normal equations in fp64 like numpy does.
// ---------------------------------------------------------------------------------------------
__global__ void bg_count_kernel(const int64_t* __restrict__ tail, const int64_t* __restrict__ tip, int64_t E, int64_t V,
                                int32_t* __restrict__ cnt /* V + 1, pre-set: cnt[0] = 0, cnt[v + 1] = 1 (self) */) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int64_t a = tail[e], b = tip[e];
  if (a != b && a >= 0 && a < V && b >= 0 && b < V) atomicAdd(cnt + a + 1, 1);
}
__global__ void bg_init_kernel(int32_t* __restrict__ cnt, int32_t* __restrict__ cursor, int64_t V) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v == 0) cnt[0] = 0;
  if (v < V) { cnt[v + 1] = 1; cursor[v] = 1; }
}
// scatter: slot 0 of every row is the vertex itself; the others take the edge's tangent vector as provisional value
__global__ void bg_fill_kernel(const int64_t* __restrict__ tail, const int64_t* __restrict__ tip, int64_t E, int64_t V,
                               const float* __restrict__ verts, const float* __restrict__ frames,
                               const float* __restrict__ edge_tangent, const int32_t* __restrict__ rowptr,
                               int32_t* __restrict__ cursor, int32_t* __restrict__ colidx, float2* __restrict__ vals) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < V) {                                                    // (the first V threads also write the self entries)
    colidx[rowptr[e]] = (int32_t)e;
    vals[rowptr[e]] = make_float2(0.f, 0.f);
  }
  if (e >= E) return;
  const int64_t a = tail[e], b = tip[e];
  if (a == b || a < 0 || a >= V || b < 0 || b >= V) return;
  float2 t;
  if (edge_tangent) {
    t = make_float2(edge_tangent[2 * e], edge_tangent[2 * e + 1]);
  } else {
    // edge_tangent_vectors (geometry.py:198-207) in fp32, products and sums rounded separately like the torch ops
    const float dx = __fsub_rn(verts[3 * b], verts[3 * a]), dy = __fsub_rn(verts[3 * b + 1], verts[3 * a + 1]),
                dz = __fsub_rn(verts[3 * b + 2], verts[3 * a + 2]);
    const float* f = frames + 9 * a;
    t.x = __fadd_rn(__fadd_rn(__fmul_rn(dx, f[0]), __fmul_rn(dy, f[1])), __fmul_rn(dz, f[2]));
    t.y = __fadd_rn(__fadd_rn(__fmul_rn(dx, f[3]), __fmul_rn(dy, f[4])), __fmul_rn(dz, f[5]));
  }
  const int dst = rowptr[a] + atomicAdd(cursor + a, 1);
  colidx[dst] = (int32_t)b;
  vals[dst] = t;
}
// rows are sorted by column now; entries with column == row are the vertex itself (exactly one, a self loop is never
// scattered).  (lhs^T lhs + 1e-5 I)^-1 lhs^T in fp64, self coefficient = -sum of the others (geometry.py:245-259)
__global__ void bg_solve_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, int64_t V,
                                float2* __restrict__ vals) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int s = rowptr[v], e = rowptr[v + 1];
  double a = 1e-5, b = 0.0, d = 1e-5;
  for (int p = s; p < e; ++p) {
    if (colidx[p] == (int32_t)v) continue;
    const double x = vals[p].x, y = vals[p].y;
    a += x * x; b += x * y; d += y * y;
  }
  const double det = a * d - b * b;
  const double i00 = d / det, i01 = -b / det, i11 = a / det;
  double sx = 0.0, sy = 0.0;
  int self = -1;
  for (int p = s; p < e; ++p) {
    if (colidx[p] == (int32_t)v) { self = p; continue; }
    const double x = vals[p].x, y = vals[p].y;
    const double cx = i00 * x + i01 * y, cy = i01 * x + i11 * y;
    sx += cx; sy += cy;
    vals[p] = make_float2((float)cx, (float)cy);
  }
  if (self >= 0) vals[self] = make_float2((float)(-sx), (float)(-sy));
}

}  // namespace

int launch_build_grad(const float* verts, const float* frames, const float* edge_tangent, const int64_t* edges, int64_t E,
                      int64_t V, int32_t* rowptr, int32_t* colidx, float* vals, int32_t* cursor /* V ints */,
                      cudaStream_t st) {
  if (V <= 0) return DN_OK;
  const unsigned vb = (unsigned)((V + 255) / 256);
  const int64_t n = E > V ? E : V;
  const unsigned eb = (unsigned)((n + 255) / 256);
  bg_init_kernel<<<vb, 256, 0, st>>>(rowptr, cursor, V);
  DN_LAUNCH_CHECK();
  if (E > 0) {
    bg_count_kernel<<<(unsigned)((E + 255) / 256), 256, 0, st>>>(edges, edges + E, E, V, rowptr);
    DN_LAUNCH_CHECK();
  }
  tr_scan_kernel<<<1, 1024, 0, st>>>(rowptr, V + 1);
  DN_LAUNCH_CHECK();
  bg_fill_kernel<<<eb, 256, 0, st>>>(edges, edges + E, E, V, verts, frames, edge_tangent, rowptr, cursor, colidx,
                                     reinterpret_cast<float2*>(vals));
  DN_LAUNCH_CHECK();
  tr_sort_rows_kernel<<<vb, 256, 0, st>>>(rowptr, V, colidx, reinterpret_cast<float2*>(vals));
  DN_LAUNCH_CHECK();
  bg_solve_kernel<<<vb, 256, 0, st>>>(rowptr, colidx, V, reinterpret_cast<float2*>(vals));
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_compute_hks(const float* evals, const float* evecs, const float* scales, int64_t V, int K, int S,
                       float* out, cudaStream_t st) {
  if (V <= 0 || S <= 0) return DN_OK;
  if (S <= 16 && K % 32 == 0 && K >= 32 && K <= 256 && (K / 32 <= 4 || K == 256)) {
    int64_t blocks = (V + 31) / 32;       // 8 warps x 4 rows per block iteration
    const int64_t cap = (int64_t)dn_sm_count() * 8;   // grid-stride: the coefficient table is built once per warp (4 rows/iteration)
    if (blocks > cap) blocks = cap;
    switch (K / 32) {
      case 1: hks_warp_kernel<1><<<(unsigned)blocks, 256, 0, st>>>(evals, evecs, scales, V, S, out); break;
      case 2: hks_warp_kernel<2><<<(unsigned)blocks, 256, 0, st>>>(evals, evecs, scales, V, S, out); break;
      case 3: hks_warp_kernel<3><<<(unsigned)blocks, 256, 0, st>>>(evals, evecs, scales, V, S, out); break;
      case 4: hks_warp_kernel<4><<<(unsigned)blocks, 256, 0, st>>>(evals, evecs, scales, V, S, out); break;
      default: hks_warp_kernel<8><<<(unsigned)blocks, 256, 0, st>>>(evals, evecs, scales, V, S, out); break;
    }
  } else {
    hks_generic_kernel<<<(unsigned)((V * 32 + 255) / 256), 256, 0, st>>>(evals, evecs, scales, V, K, S, out);
  }
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_csr_transpose(const dn_csr* in, int64_t V, int32_t* rowptr_t, int32_t* colidx_t, float* vals_t,
                         int32_t* cursor /* V ints */, cudaStream_t st) {
  DN_CUDA_TRY(cudaMemsetAsync(rowptr_t, 0, sizeof(int32_t) * (V + 1), st));
  if (V <= 0 || in->nnz <= 0) return DN_OK;
  DN_CUDA_TRY(cudaMemsetAsync(cursor, 0, sizeof(int32_t) * V, st));
  const unsigned vb = (unsigned)((V + 255) / 256);
  tr_count_kernel<<<(unsigned)((in->nnz + 255) / 256), 256, 0, st>>>(in->colidx, in->nnz, rowptr_t);
  DN_LAUNCH_CHECK();
  tr_scan_kernel<<<1, 1024, 0, st>>>(rowptr_t, V + 1);
  DN_LAUNCH_CHECK();
  tr_fill_kernel<<<vb, 256, 0, st>>>(in->rowptr, in->colidx, reinterpret_cast<const float2*>(in->vals), V, rowptr_t,
                                     cursor, colidx_t, reinterpret_cast<float2*>(vals_t));
  DN_LAUNCH_CHECK();
  tr_sort_rows_kernel<<<vb, 256, 0, st>>>(rowptr_t, V, colidx_t, reinterpret_cast<float2*>(vals_t));
  DN_LAUNCH_CHECK();
  return DN_OK;
}
