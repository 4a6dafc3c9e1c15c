// SIMT (FFMA, exact fp32) kernels of the DiffusionNetBlock hot path, and the sparse /
// elementwise kernels shared by every engine.  sm_90a.
//
// Reference functions restated here (file:line in /root/reference/src/diffusion_net):
//   to_basis geometry.py:572-583, from_basis geometry.py:586-598,
//   LearnedTimeDiffusion.forward layers.py:44-67, grad SpMM layers.py:216-223,
//   SpatialGradientFeatures.forward layers.py:117-130, MiniMLP layers.py:133-164.
#include "dn_internal.h"
#include "dn_tc_ptx.cuh"
#include <math.h>
#include <type_traits>

namespace {

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// ---------------------------------------------------------------------------------------------
// rows GEMM:  out[v][n] = epi( sum_k A[v][k] * W[n][k] + bias[n] ),  A = concat of up to 3 sources
// ---------------------------------------------------------------------------------------------
constexpr int RG_BM = 128, RG_BN = 64, RG_BK = 16;

__device__ __forceinline__ float load_src_scalar(const DnRowsSrc& s, int64_t row, int k) {
#pragma unroll
  for (int i = 0; i < DN_MAX_SRC; ++i) {
    if (i < s.nsrc) {
      if (k < s.width[i]) return __ldg(s.ptr[i] + row * s.ld[i] + k);
      k -= s.width[i];
    }
  }
  return 0.f;
}

__device__ __forceinline__ float4 load_src_vec4(const DnRowsSrc& s, int64_t row, int k) {
#pragma unroll
  for (int i = 0; i < DN_MAX_SRC; ++i) {
    if (i < s.nsrc) {
      if (k < s.width[i]) return ldg4(s.ptr[i] + row * s.ld[i] + k);
      k -= s.width[i];
    }
  }
  return make_float4(0.f, 0.f, 0.f, 0.f);
}

template <bool VEC>
__global__ void __launch_bounds__(256) rows_gemm_kernel(DnRowsSrc src, DnLayer L, int64_t V) {
  __shared__ __align__(16) float As[RG_BK][RG_BM + 4];
  __shared__ __align__(16) float Bs[RG_BK][RG_BN + 4];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int64_t row0 = (int64_t)blockIdx.x * RG_BM;
  const int n0 = blockIdx.y * RG_BN;
  const int K = L.K, N = L.N;
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += RG_BK) {
    // ---- A tile: 128 rows x 16 k, transposed into As[k][row]
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = (t >> 2) + 64 * i;
      const int kq = (t & 3) * 4;
      const int64_t gr = row0 + r;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (gr < V) {
        if (VEC && k0 + kq + 3 < K) {
          float4 q = load_src_vec4(src, gr, k0 + kq);
          v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (k0 + kq + j < K) v[j] = load_src_scalar(src, gr, k0 + kq + j);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) As[kq + j][r] = v[j];
    }
    // ---- B tile: 16 k x 64 n into Bs[k][n]
    if (!L.w_trans) {
      const int n = t >> 2, kq = (t & 3) * 4, gn = n0 + n;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (gn < N) {
        const float* wp = (L.W2 && gn >= L.n_split) ? L.W2 + (int64_t)(gn - L.n_split) * L.ldw + k0 + kq
                                                    : L.W + (int64_t)gn * L.ldw + k0 + kq;
        if (VEC && k0 + kq + 3 < K) {
          float4 q = ldg4(wp);
          v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (k0 + kq + j < K) v[j] = __ldg(wp + j);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) Bs[kq + j][n] = v[j];
    } else {
      const int k = t >> 4, nq = (t & 15) * 4;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (k0 + k < K) {
        const float* wp = L.W + (int64_t)(k0 + k) * L.ldw + n0 + nq;
        if (VEC && n0 + nq + 3 < N) {
          float4 q = ldg4(wp);
          v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (n0 + nq + j < N) v[j] = __ldg(wp + j);
        }
      }
      *reinterpret_cast<float4*>(&Bs[k][nq]) = make_float4(v[0], v[1], v[2], v[3]);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < RG_BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * 8]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[k][ty * 8 + 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
  // ---- epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t gr = row0 + ty * 8 + i;
    if (gr >= V) continue;
    const float rs = L.row_scale ? __ldg(L.row_scale + gr) : 1.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gn >= N) continue;
      float v = acc[i][j];
      if (L.bias) v += __ldg(L.bias + gn);
      if (L.relu) v = fmaxf(v, 0.f);
      if (L.emul) v *= __ldg(L.emul + gr * N + gn);
      if (L.relu_mask_src) v = (__ldg(L.relu_mask_src + gr * N + gn) > 0.f) ? v : 0.f;
      if (L.row_scale) v *= rs;
      if (L.residual) v = fmaf(L.res_scale, L.residual[gr * L.ld_res + gn], v);
      L.out[gr * L.ld_out + gn] = v;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// A^T B with a long reduction over vertices (to_basis, weight gradients):
//   partial[p][i][j] = sum_{v in split p} A[v][i] * scale[v] * B[v][j]
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) atb_partial_kernel(const float* __restrict__ A, int64_t lda, int I,
                                                          const float* __restrict__ B, int64_t ldb, int J,
                                                          const float* __restrict__ scale, int64_t V,
                                                          int64_t rows_per_split, float* __restrict__ partial) {
  __shared__ __align__(16) float As[16][64 + 4];
  __shared__ __align__(16) float Bs[16][64 + 4];
  const int tilesJ = (J + 63) / 64;
  const int i0 = (blockIdx.x / tilesJ) * 64, j0 = (blockIdx.x % tilesJ) * 64;
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int64_t vbeg = (int64_t)blockIdx.y * rows_per_split;
  const int64_t vend = min(V, vbeg + rows_per_split);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const bool veca = ((lda & 3) == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
  const bool vecb = ((ldb & 3) == 0) && ((reinterpret_cast<uintptr_t>(B) & 15) == 0);
  for (int64_t v0 = vbeg; v0 < vend; v0 += 16) {
    const int r = t >> 4, c4 = (t & 15) * 4;
    const int64_t gv = v0 + r;
    float a[4] = {0.f, 0.f, 0.f, 0.f}, b[4] = {0.f, 0.f, 0.f, 0.f};
    if (gv < vend) {
      const float s = scale ? __ldg(scale + gv) : 1.f;
      if (veca && i0 + c4 + 3 < I) {
        float4 q = ldg4(A + gv * lda + i0 + c4);
        a[0] = q.x; a[1] = q.y; a[2] = q.z; a[3] = q.w;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (i0 + c4 + j < I) a[j] = __ldg(A + gv * lda + i0 + c4 + j);
      }
      if (vecb && j0 + c4 + 3 < J) {
        float4 q = ldg4(B + gv * ldb + j0 + c4);
        b[0] = q.x; b[1] = q.y; b[2] = q.z; b[3] = q.w;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (j0 + c4 + j < J) b[j] = __ldg(B + gv * ldb + j0 + c4 + j);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] *= s;   // (values * massvec) as in geometry.py:583
    }
    *reinterpret_cast<float4*>(&As[r][c4]) = make_float4(a[0], a[1], a[2], a[3]);
    *reinterpret_cast<float4*>(&Bs[r][c4]) = make_float4(b[0], b[1], b[2], b[3]);
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float aa[4] = {av.x, av.y, av.z, av.w};
      const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(aa[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* pp = partial + (int64_t)blockIdx.y * I * J;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gi = i0 + ty * 4 + i;
    if (gi >= I) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gj = j0 + tx * 4 + j;
      if (gj < J) pp[(int64_t)gi * J + gj] = acc[i][j];
    }
  }
}

// out[b * rows + i][j] (+)= sum over the partials p of mesh b of partial[p][i][j], in partial order from 0: p in
// [mesh_cta_begin[b], mesh_cta_begin[b + 1]) with a per-mesh CTA table (grid y = meshes), [0, P) without one
__global__ void reduce_partials_kernel(const float* __restrict__ partial, int P, const int32_t* __restrict__ mesh_cta_begin,
                                       int64_t rows, int cols, float* __restrict__ out, int64_t ld_out, int accumulate) {
  const int64_t n = rows * cols, idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (idx >= n) return;
  const int p0 = mesh_cta_begin ? mesh_cta_begin[b] : 0, p1 = mesh_cta_begin ? mesh_cta_begin[b + 1] : P;
  const float* src = partial + (int64_t)p0 * n + idx;
  float s = 0.f;
  for (int q = 0; q < p1 - p0; ++q) s += src[(int64_t)q * n];
  float* o = out + ((int64_t)b * rows + idx / cols) * ld_out + idx % cols;
  *o = accumulate ? (*o + s) : s;
}

// partial[p][n] = sum over the rows of slice p of A[v][n].  Block (32, 8): 32 columns x 8 row lanes, combined in a
// fixed order, so the sum does not depend on scheduling.
__global__ void colsum_partial_kernel(const float* __restrict__ A, int64_t lda, int N, int64_t V,
                                      int64_t rows_per_split, float* __restrict__ partial) {
  __shared__ float red[8][33];
  const int n = blockIdx.y * 32 + threadIdx.x;
  const int64_t vbeg = (int64_t)blockIdx.x * rows_per_split;
  const int64_t vend = min(V, vbeg + rows_per_split);
  float s = 0.f;
  if (n < N)
    for (int64_t v = vbeg + threadIdx.y; v < vend; v += 8) s += __ldg(A + v * lda + n);
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && n < N) {
    float tot = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) tot += red[i][threadIdx.x];
    partial[(int64_t)blockIdx.x * N + n] = tot;
  }
}

// ---------------------------------------------------------------------------------------------
// spectral coefficient kernels (layers.py:48-49, 62-64)
// ---------------------------------------------------------------------------------------------
__global__ void spectral_scale_kernel(const float* __restrict__ partial, int P, const float* __restrict__ evals,
                                      float* __restrict__ time, int K, int C, float* __restrict__ x_spec_out,
                                      float* __restrict__ S_out, int clamp_writeback) {
  // block = 64 consecutive elements x 4 slices of the P partial sums (more loads in flight)
  __shared__ float red[4][64];
  const int e = threadIdx.x & 63, sl = threadIdx.x >> 6;
  const int idx = blockIdx.x * 64 + e;
  float acc = 0.f;
  if (idx < K * C)
    for (int p = sl; p < P; p += 4) acc += partial[(int64_t)p * K * C + idx];
  red[sl][e] = acc;
  __syncthreads();
  if (sl != 0 || idx >= K * C) return;
  const int k = idx / C, c = idx % C;
  const float s = pairwise_sum<4>(&red[0][e], 64);
  const float t = dn_clamp_time(time[c]);
  if (x_spec_out) x_spec_out[idx] = s;
  S_out[idx] = dn_heat(evals[k], t) * s;
  // every thread of row k == 0 re-writes the clamped time (same value from all writers is benign)
  if (clamp_writeback && k == K - 1) {
    // last row, after all reads of time[c] by this thread; other threads read the same c only
    // through fmaxf(...,1e-8) which is idempotent under this write.
    time[c] = t;
  }
}

// backward: Gs = sum_p partial (= Phi^T g), dS = E * Gs, dt[c] += sum_k Gs*( -lambda_k )*E*x_spec
__global__ void spectral_bwd_kernel(const float* __restrict__ partial, int P, const float* __restrict__ evals,
                                    const float* __restrict__ time, const float* __restrict__ x_spec, int K, int C,
                                    float* __restrict__ dS, float* __restrict__ grad_time) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float t = dn_clamp_time(time[c]);
  float dt = 0.f;
  for (int k = 0; k < K; ++k) {
    const int idx = k * C + c;
    float g = 0.f;
    for (int p = 0; p < P; ++p) g += partial[(int64_t)p * K * C + idx];
    const float lam = evals[k];
    const float e = dn_heat(lam, t);
    dS[idx] = e * g;
    dt += dn_time_grad_term(g, lam, e, x_spec[idx]);
  }
  grad_time[c] += dt;
}

// the same time gradient over a mesh batch: G, x_spec [n_meshes][K][C], evals [n_meshes][K].  Block (32, 16): 32
// consecutive channels (coalesced) x 16 slices of the n_meshes * K eigenpairs, combined in a fixed order.
__global__ void spectral_time_grad_batched_kernel(const float* __restrict__ G, const float* __restrict__ x_spec,
                                                  const float* __restrict__ evals, const float* __restrict__ time,
                                                  int rows, int C, float* __restrict__ grad_time) {
  __shared__ float red[16][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float dt = 0.f;
  if (c < C) {
    const float t = dn_clamp_time(time[c]);
    for (int r = threadIdx.y; r < rows; r += 16) {   // r = b * K + k
      const int64_t idx = (int64_t)r * C + c;
      const float lam = evals[r];
      dt += dn_time_grad_term(G[idx], lam, dn_heat(lam, t), x_spec[idx]);
    }
  }
  red[threadIdx.y][threadIdx.x] = dt;
  __syncthreads();
  if (threadIdx.y != 0 || c >= C) return;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) s += red[i][threadIdx.x];
  grad_time[c] += s;
}

// ---------------------------------------------------------------------------------------------
// sparse kernels
// ---------------------------------------------------------------------------------------------
__global__ void csr_from_coo_kernel(const int64_t* __restrict__ rows, const int64_t* __restrict__ cols,
                                    const float* __restrict__ vx, const float* __restrict__ vy, int64_t nnz,
                                    int64_t V, int32_t* __restrict__ rowptr, int32_t* __restrict__ colidx,
                                    float* __restrict__ vals) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= nnz) return;
  const int64_t r = rows[p];
  const int64_t rprev = (p == 0) ? -1 : rows[p - 1];
  for (int64_t rr = rprev + 1; rr <= r; ++rr) rowptr[rr] = (int32_t)p;
  if (p == nnz - 1)
    for (int64_t rr = r + 1; rr <= V; ++rr) rowptr[rr] = (int32_t)nnz;
  colidx[p] = (int32_t)cols[p];
  vals[2 * p] = vx[p];
  vals[2 * p + 1] = vy ? vy[p] : 0.f;
}

// out[v][c][0..1] = (gradX @ x, gradY @ x)  -- the reference's (V,C,2) layout, layers.py:216-223
__global__ void grad_spmm_pair_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                                      const float2* __restrict__ vals, const float* __restrict__ x, int64_t V,
                                      int C, float* __restrict__ out) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= V) return;
  const int s = rowptr[row], e = rowptr[row + 1];
  for (int c = lane; c < C; c += 32) {
    float gx = 0.f, gy = 0.f;
    for (int p = s; p < e; ++p) {
      const float2 g = __ldg(vals + p);
      const float xv = __ldg(x + (int64_t)__ldg(colidx + p) * C + c);
      gx = fmaf(g.x, xv, gx);
      gy = fmaf(g.y, xv, gy);
    }
    reinterpret_cast<float2*>(out)[row * C + c] = make_float2(gx, gy);
  }
}

// ---------------------------------------------------------------------------------------------
// gradient features (layers.py:121-130):  feat = tanh(gX*Bre + gY*Bim),  gX = GX x, gY = GY x,
// Bre = GX P - GY Q, Bim = GY P + GX Q, with P = xd A_re^T, Q = xd A_im^T ([P|Q], row stride ld_pq)
//
// Every kernel below that forms or differentiates the features accumulates a CSR row with feat_entry, in CSR order,
// and the forward kernels finish with feat_value, so they are bit-identical to each other.  Lane type T is float (one
// channel) or float4 (four consecutive channels, one 16-byte access per row and stream).
// ---------------------------------------------------------------------------------------------

// tanh(x) = 1 - 2 / (exp(2x) + 1) with the hardware exp2 and fast division: ~6 instructions instead of tanhf's ~30
// (the gather kernel issues instructions on 53 % of its cycles, profiles/r01: the four tanhf per lane were a fifth of
// them).  Absolute error below 11.5 * 2^-24 (6.9e-7) over the whole range, derived from the documented maximum errors
// of __expf (2 + floor(|1.173 y|) ulp) and __fdividef (2 ulp); measured worst 2.3e-7 over 2^27 arguments (H100 SXM,
// 700 W).  Saturates to +-1, NaN propagates.
__device__ __forceinline__ float dn_feat_tanh(float x) {
  const float e = __expf(2.f * x);
  return 1.f - __fdividef(2.f, e + 1.f);
}

// f applied channel by channel to lanes of type float or float4
template <class F, class... A>
__device__ __forceinline__ float per_ch(F f, float a, A... b) { return f(a, b...); }
template <class F, class... A>
__device__ __forceinline__ float4 per_ch(F f, float4 a, A... b) {
  return make_float4(f(a.x, b.x...), f(a.y, b.y...), f(a.z, b.z...), f(a.w, b.w...));
}

template <class T>
__device__ __forceinline__ T vfma(float w, T v, T acc) {
  return per_ch([w](float vi, float ai) { return fmaf(w, vi, ai); }, v, acc);
}

template <class T>
__device__ __forceinline__ T ldg_lane(const float* p) {
  if constexpr (sizeof(T) == sizeof(float4)) return ldg4(p);
  else return __ldg(p);
}

template <class T>
struct FeatAcc {
  T gX, gY, bre, bim;
};

// one CSR entry (col, g = (gx, gy)) of a row: x, P, Q are the lanes of row col of xd, P and Q.  The one place the
// per-channel FMA sequence is written.
template <bool ROT, class T>
__device__ __forceinline__ void feat_entry(FeatAcc<T>& a, float2 g, T x, T P, T Q) {
  a.gX = vfma(g.x, x, a.gX);
  a.gY = vfma(g.y, x, a.gY);
  a.bre = vfma(g.x, P, a.bre);
  a.bim = vfma(g.y, P, a.bim);
  if (ROT) {
    a.bre = vfma(-g.y, Q, a.bre);
    a.bim = vfma(g.x, Q, a.bim);
  }
}

template <class T>
__device__ __forceinline__ T feat_value(const FeatAcc<T>& a) {
  return per_ch([](float gX, float gY, float bre, float bim) { return dn_feat_tanh(fmaf(gX, bre, gY * bim)); },
                a.gX, a.gY, a.bre, a.bim);
}

// the accumulators of channels [c, c + |T|) over a row's CSR entries [s, e)
template <bool ROT, class T>
__device__ __forceinline__ FeatAcc<T> gather_row(const int32_t* __restrict__ colidx, const float2* __restrict__ vals,
                                                 const float* __restrict__ xd, const float* __restrict__ pq, int ld_pq,
                                                 int C, int s, int e, int c) {
  FeatAcc<T> a = {};
  for (int p = s; p < e; ++p) {
    const int64_t col = __ldg(colidx + p);
    const float2 g = __ldg(vals + p);
    const T x = ldg_lane<T>(xd + col * C + c);
    const T P = ldg_lane<T>(pq + col * ld_pq + c);
    feat_entry<ROT>(a, g, x, P, ROT ? ldg_lane<T>(pq + col * ld_pq + C + c) : T{});
  }
  return a;
}

// Runs body(row, s, e, c) for each lane of channels [c, c + |T|) the thread owns in a row-gather kernel, [s, e) being
// the row's CSR entries.  float4 lanes: G threads per row (a power of two, whole warps of 32 / G rows), each stepping
// over the row by 4 G channels.  float lanes (C % 4 != 0): one thread per (row, channel).
template <class T, class F>
__device__ __forceinline__ void feat_lanes(const int32_t* __restrict__ rowptr, int64_t V, int C, int G, F body) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if constexpr (sizeof(T) == sizeof(float4)) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (t >> 5) * (32 / G) + lane / G;
    if (row >= V) return;
    const int s = __ldg(rowptr + row), e = __ldg(rowptr + row + 1);
    for (int c = 4 * (lane % G); c < C; c += 4 * G) body(row, s, e, c);
  } else {
    if (t >= V * C) return;
    const int64_t row = t / C;
    const int c = (int)(t - row * C);
    body(row, __ldg(rowptr + row), __ldg(rowptr + row + 1), c);
  }
}

// feat = tanh(gX*Bre + gY*Bim) row by row, threads mapped by feat_lanes
template <bool ROT, class T>
__global__ void __launch_bounds__(256) spmm_features_kernel(const int32_t* __restrict__ rowptr,
                                                            const int32_t* __restrict__ colidx,
                                                            const float2* __restrict__ vals,
                                                            const float* __restrict__ xd, const float* __restrict__ pq,
                                                            int ld_pq, int64_t V, int C, int G,
                                                            float* __restrict__ feat) {
  feat_lanes<T>(rowptr, V, C, G, [&](int64_t row, int s, int e, int c) {
    *reinterpret_cast<T*>(feat + row * C + c) = feat_value(gather_row<ROT, T>(colidx, vals, xd, pq, ld_pq, C, s, e, c));
  });
}

// ---------------------------------------------------------------------------------------------
// Block gather (C a multiple of 128): one CTA per 64 consecutive rows.
//   * the block's CSR metadata (rowptr slice, every (col, gx, gy) triple) is staged in shared memory by ONE coalesced
//     pass: the per-row dependent chain rowptr -> colidx -> neighbour rows (three DRAM/L2 latencies in the warp-per-row
//     kernel) becomes one latency per 64 rows plus the gathers themselves;
//   * a warp issues every neighbour-row load of a batch of NB entries (3 x NB independent 16-byte loads per lane)
//     before the first FMA; 8 warps walk 8 consecutive rows at a time, so the band structure of a locally ordered
//     mesh hits L1.
// ---------------------------------------------------------------------------------------------
constexpr int GB_ROWS = 64;      // rows per CTA
constexpr int GB_NNZ = 1024;     // staged entries per CTA (entries past it are read from global memory)

struct __align__(16) GxyEnt { int col; int pad; float gx, gy; };   // (gx, gy) 8-byte aligned: one LDS.64

// NB entries: every 16-byte slice of the batch's neighbour rows is loaded before the first FMA.  The weights are read
// again from the entry at FMA time: a broadcast LDS.64 is cheaper than 2 x NB live registers.  The row strides are
// 32-bit: with 64-bit ones the C = 128 rotation instance spills at its 128-register cap.
template <bool ROT, int NB>
__device__ __forceinline__ void blk_entries(FeatAcc<float4>& a, const GxyEnt* en, const char* xb, const char* pb,
                                            int x_row_bytes, int pq_row_bytes) {
  float4 x[NB], P[NB], Q[NB];
#pragma unroll
  for (int j = 0; j < NB; ++j) {
    const int64_t col = en[j].col;
    const char* pr = pb + col * pq_row_bytes;
    x[j] = __ldg(reinterpret_cast<const float4*>(xb + col * x_row_bytes));
    P[j] = __ldg(reinterpret_cast<const float4*>(pr));
    Q[j] = ROT ? __ldg(reinterpret_cast<const float4*>(pr + x_row_bytes)) : float4{};
  }
#pragma unroll
  for (int j = 0; j < NB; ++j) feat_entry<ROT>(a, *reinterpret_cast<const float2*>(&en[j].gx), x[j], P[j], Q[j]);
}

// (16-byte entry records, unpredicated full batches -- the first version,
// with per-entry predicates and separate col / value arrays, spent half of its issue slots on bookkeeping.)
template <bool ROT, int NH>
__global__ void __launch_bounds__(256, 2)
spmm_features_blk_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                         const float2* __restrict__ vals, const float* __restrict__ xd,
                         const float* __restrict__ pq, int ld_pq, int64_t V, float* __restrict__ feat) {
  constexpr int C = 128 * NH;          // a warp covers 128 channels per pass (one float4 per lane), NH passes per row
  constexpr int x_row_bytes = C * 4;
  __shared__ int s_rp[GB_ROWS + 1];
  __shared__ GxyEnt s_e[GB_NNZ];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t base = (int64_t)blockIdx.x * GB_ROWS;
  const int nrows = (int)((V - base) < GB_ROWS ? (V - base) : GB_ROWS);
  if ((int)threadIdx.x <= nrows) s_rp[threadIdx.x] = __ldg(rowptr + base + threadIdx.x);
  __syncthreads();
  const int e0 = s_rp[0];
  const int tot = s_rp[nrows] - e0;
  const bool staged = tot <= GB_NNZ;                              // (block-uniform)
  if (staged) {
    for (int i = threadIdx.x; i < tot; i += 256) {
      const float2 g = __ldg(vals + e0 + i);
      GxyEnt en;
      en.col = __ldg(colidx + e0 + i); en.gx = g.x; en.gy = g.y; en.pad = 0;
      s_e[i] = en;
    }
  }
  __syncthreads();
  const int pq_row_bytes = ld_pq * 4;
#pragma unroll 1
  for (int rh = warp; rh < nrows * NH; rh += 8) {
    const int r = rh / NH, h = rh % NH;
    const char* xb = reinterpret_cast<const char*>(xd) + h * 512 + lane * 16;
    const char* pb = reinterpret_cast<const char*>(pq) + h * 512 + lane * 16;
    const int s = s_rp[r] - e0, e = s_rp[r + 1] - e0;
    FeatAcc<float4> a = {};
    if (staged) {
      int p = s;
#pragma unroll 1
      for (; p + 7 <= e; p += 7)                                  // full batches: 21 independent loads, no predicates
        blk_entries<ROT, 7>(a, s_e + p, xb, pb, x_row_bytes, pq_row_bytes);
#pragma unroll 1
      for (; p + 2 <= e; p += 2)                                  // remainder: pairs, then a single entry
        blk_entries<ROT, 2>(a, s_e + p, xb, pb, x_row_bytes, pq_row_bytes);
      if (p < e) blk_entries<ROT, 1>(a, s_e + p, xb, pb, x_row_bytes, pq_row_bytes);
    } else {
#pragma unroll 1
      for (int p = s; p < e; ++p) {                               // (a block with more than GB_NNZ entries)
        GxyEnt en;
        const float2 g = __ldg(vals + e0 + p);
        en.col = __ldg(colidx + e0 + p); en.gx = g.x; en.gy = g.y; en.pad = 0;
        blk_entries<ROT, 1>(a, &en, xb, pb, x_row_bytes, pq_row_bytes);
      }
    }
    *reinterpret_cast<float4*>(feat + (base + r) * C + h * 128 + lane * 4) = feat_value(a);
  }
}

// Patch variant (dn_patches, built once for resident operators): one CTA per patch of graph-adjacent rows.
// Phase 1 copies the patch's distinct neighbour rows of x_diffuse and [P|Q] into shared memory, coalesced, each row
// exactly once; phase 2 is the same gather as above but out of shared memory.  At V = 200k the plain kernel moves
// ~1.1 GB from L2 into the SMs (every neighbour row is re-fetched by ~half of the vertices that touch it: 47 % L1
// hits); here it is (distinct rows / rows) x 1.5 KB per vertex.  Entries keep their CSR order, so the result is
// bit-identical.
template <bool ROT>
__global__ void __launch_bounds__(512) spmm_features_patch_kernel(const dn_patches P, const float* __restrict__ xd,
                                                                  const float* __restrict__ pq, int ld_pq, int C,
                                                                  float* __restrict__ feat) {
  extern __shared__ float4 sm4[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int xq = C >> 2, pqq = ld_pq >> 2, rowf4 = xq + pqq;
  const int p = blockIdx.x;
  const int s0 = __ldg(P.src_ptr + p), ns = __ldg(P.src_ptr + p + 1) - s0;
  const int t0 = __ldg(P.tgt_ptr + p), nt = __ldg(P.tgt_ptr + p + 1) - t0;
  const float2* vals = reinterpret_cast<const float2*>(P.vals);

  // per-row metadata of this warp's target, one entry per lane (coalesced), fetched one round ahead so that its
  // latency hides behind the row copies (round 0) or the previous round's arithmetic
  struct Meta { int64_t row; int es, n; int lc; float2 g; };
  auto load_meta = [&](int i) {
    Meta m;
    m.row = 0; m.es = 0; m.n = 0; m.lc = 0; m.g = make_float2(0.f, 0.f);
    if (i < nt) {
      m.row = __ldg(P.tgt + t0 + i);
      m.es = __ldg(P.ent_ptr + t0 + i);
      m.n = __ldg(P.ent_ptr + t0 + i + 1) - m.es;
      if (lane < m.n) { m.lc = __ldg(P.lcol + m.es + lane); m.g = __ldg(vals + m.es + lane); }
    }
    return m;
  };
  Meta cur = load_meta(warp);

  // phase 1: distinct neighbour rows -> shared memory, four rows (12 x 16 B at C = 128) in flight per lane
  for (int r = warp; r < ns; r += 4 * nwarps) {
    int64_t row[4];
    bool ok[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      ok[u] = r + u * nwarps < ns;
      row[u] = __ldg(P.src_rows + s0 + (ok[u] ? r + u * nwarps : r));
    }
    for (int c4 = lane; c4 < xq; c4 += 32) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = ldg4(xd + row[u] * C + 4 * c4);
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (ok[u]) sm4[(size_t)(r + u * nwarps) * rowf4 + c4] = v[u];
    }
    for (int c4 = lane; c4 < pqq; c4 += 32) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = ldg4(pq + row[u] * ld_pq + 4 * c4);
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (ok[u]) sm4[(size_t)(r + u * nwarps) * rowf4 + xq + c4] = v[u];
    }
  }
  __syncthreads();

  // phase 2: the gather, out of shared memory, entries in CSR order
  for (int i = warp; i < nt; i += nwarps) {
    const Meta nxt = load_meta(i + nwarps);
    for (int c4 = lane; c4 < xq; c4 += 32) {
      FeatAcc<float4> a = {};
      for (int base = 0; base < cur.n; base += 32) {
        int lc_l = cur.lc;
        float2 g_l = cur.g;
        if (base > 0) {                                            // rows longer than a warp: next 32 entries
          lc_l = 0; g_l = make_float2(0.f, 0.f);
          if (base + lane < cur.n) { lc_l = __ldg(P.lcol + cur.es + base + lane); g_l = __ldg(vals + cur.es + base + lane); }
        }
        const int cnt = (cur.n - base) < 32 ? (cur.n - base) : 32;
        for (int e = 0; e < cnt; ++e) {
          const int lc = __shfl_sync(0xffffffffu, lc_l, e);
          float2 g;
          g.x = __shfl_sync(0xffffffffu, g_l.x, e);
          g.y = __shfl_sync(0xffffffffu, g_l.y, e);
          const float4* src = sm4 + (size_t)lc * rowf4;
          feat_entry<ROT>(a, g, src[c4], src[xq + c4], ROT ? src[2 * xq + c4] : float4{});
        }
      }
      *reinterpret_cast<float4*>(feat + cur.row * C + c4 * 4) = feat_value(a);
    }
    cur = nxt;
  }
}

// U[v] = [dd*Bre | dd*Bim | dd*gX | dd*gY],  dd = dfeat * (1 - feat^2)
template <bool ROT, class T>
__global__ void __launch_bounds__(256) features_bwd_local_kernel(
    const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const float2* __restrict__ vals,
    const float* __restrict__ xd, const float* __restrict__ pq, int ld_pq, const float* __restrict__ feat,
    const float* __restrict__ dfeat, int64_t V, int C, int G, float* __restrict__ U) {
  const auto mul = [](float d, float v) { return d * v; };
  feat_lanes<T>(rowptr, V, C, G, [&](int64_t row, int s, int e, int c) {
    const FeatAcc<T> a = gather_row<ROT, T>(colidx, vals, xd, pq, ld_pq, C, s, e, c);
    const T dd = per_ch([](float d, float f) { return d * (1.f - f * f); }, ldg_lane<T>(dfeat + row * C + c),
                        ldg_lane<T>(feat + row * C + c));
    float* u = U + row * 4 * C + c;
    *reinterpret_cast<T*>(u) = per_ch(mul, dd, a.bre);
    *reinterpret_cast<T*>(u + C) = per_ch(mul, dd, a.bim);
    *reinterpret_cast<T*>(u + 2 * C) = per_ch(mul, dd, a.gX);
    *reinterpret_cast<T*>(u + 3 * C) = per_ch(mul, dd, a.gY);
  });
}

// transpose gather over the CSR of G^T:  dxd = GX^T U1 + GY^T U2;  dP = GX^T U3 + GY^T U4;
// dQ = -GY^T U3 + GX^T U4
template <bool ROT, class T>
__global__ void __launch_bounds__(256) features_bwd_transpose_kernel(
    const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const float2* __restrict__ vals,
    const float* __restrict__ U, int64_t V, int C, int G, float* __restrict__ dxd, float* __restrict__ dP,
    float* __restrict__ dQ, int64_t ld_pq) {
  feat_lanes<T>(rowptr, V, C, G, [&](int64_t row, int s, int e, int c) {
    T ax = {}, ap = {}, aq = {};
    for (int p = s; p < e; ++p) {
      const int64_t i = __ldg(colidx + p);
      const float2 g = __ldg(vals + p);
      const float* u = U + i * 4 * C + c;
      const T u1 = ldg_lane<T>(u), u2 = ldg_lane<T>(u + C), u3 = ldg_lane<T>(u + 2 * C), u4 = ldg_lane<T>(u + 3 * C);
      ax = per_ch([g](float ax, float u1, float u2) { return ax += g.x * u1 + g.y * u2; }, ax, u1, u2);
      ap = per_ch([g](float ap, float u3, float u4) { return ap += g.x * u3 + g.y * u4; }, ap, u3, u4);
      if (ROT) aq = per_ch([g](float aq, float u3, float u4) { return aq += g.x * u4 - g.y * u3; }, aq, u3, u4);
    }
    *reinterpret_cast<T*>(dxd + row * C + c) = ax;
    *reinterpret_cast<T*>(dP + row * ld_pq + c) = ap;
    if (ROT) *reinterpret_cast<T*>(dQ + row * ld_pq + c) = aq;
  });
}

__global__ void deinterleave_vc2_kernel(const float2* __restrict__ vc2, int64_t V, int C, float* __restrict__ g01) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= V * C) return;
  const int64_t v = idx / C;
  const int c = (int)(idx % C);
  const float2 g = __ldg(vc2 + idx);
  g01[v * 2 * C + c] = g.x;
  g01[v * 2 * C + C + c] = g.y;
}

__global__ void complex_dots_tanh_kernel(const float* __restrict__ g01, const float* __restrict__ b01, int64_t V,
                                         int C, float* __restrict__ out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= V * C) return;
  const int64_t v = idx / C;
  const int c = (int)(idx % C);
  const float d = g01[v * 2 * C + c] * b01[v * 2 * C + c] + g01[v * 2 * C + C + c] * b01[v * 2 * C + C + c];
  out[idx] = tanhf(d);
}

// Launches a row-gather features kernel (threads mapped by feat_lanes) for C's lane width and for `rotations`:
// launch(rot, lane, blocks, G), rot a std::bool_constant, lane a float or float4 value.
template <class F>
int launch_feat_rows(int64_t V, int C, int rotations, F launch) {
  if (V <= 0) return DN_OK;
  if (C % 4) {                                   // float lanes: one thread per (row, channel)
    const unsigned blocks = (unsigned)((V * C + 255) / 256);
    if (rotations) launch(std::true_type{}, float{}, blocks, C);
    else launch(std::false_type{}, float{}, blocks, C);
  } else {                                       // float4 lanes: G = min(32, C / 4) rounded down to a power of two
    int G = 1;
    while (G * 2 <= 32 && G * 2 <= (C >> 2)) G *= 2;
    const int64_t warps = (V + (32 / G) - 1) / (32 / G);
    const unsigned blocks = (unsigned)((warps * 32 + 255) / 256);
    if (rotations) launch(std::true_type{}, float4{}, blocks, G);
    else launch(std::false_type{}, float4{}, blocks, G);
  }
  DN_LAUNCH_CHECK();
  return DN_OK;
}

}  // namespace

// =============================================================================================
// host launchers
// =============================================================================================
int simt_rows_gemm(const DnRowsSrc& src, const DnLayer& L, int64_t V, cudaStream_t st) {
  if (V <= 0) return DN_OK;
  if (!L.out) return DN_ERR_INVALID_ARGUMENT;
  bool vec = true;
  int ktot = 0;
  for (int i = 0; i < src.nsrc; ++i) {
    vec = vec && (src.width[i] % 4 == 0) && (src.ld[i] % 4 == 0) &&
          ((reinterpret_cast<uintptr_t>(src.ptr[i]) & 15) == 0);
    ktot += src.width[i];
  }
  if (ktot != L.K) return DN_ERR_INVALID_ARGUMENT;
  vec = vec && (L.ldw % 4 == 0) && ((reinterpret_cast<uintptr_t>(L.W) & 15) == 0) &&
        (!L.W2 || (reinterpret_cast<uintptr_t>(L.W2) & 15) == 0);
  dim3 grid((unsigned)((V + RG_BM - 1) / RG_BM), (unsigned)((L.N + RG_BN - 1) / RG_BN));
  if (vec)
    rows_gemm_kernel<true><<<grid, 256, 0, st>>>(src, L, V);
  else
    rows_gemm_kernel<false><<<grid, 256, 0, st>>>(src, L, V);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

// Row slices of a split-V reduction over V rows and `tiles` column tiles, each slice's partial `slice_floats` floats:
// slices of >= 2048 rows, at most 4 CTAs per SM over the column tiles and never more than ws holds, with the rows of a
// slice rounded up to a multiple of `round`.  Sets *P and *rps (rows per slice); DN_ERR_WORKSPACE if one slice does not fit.
static int plan_row_slices(int64_t V, int tiles, int64_t slice_floats, int64_t ws_floats, int round, int* P_out,
                           int64_t* rps_out) {
  int P = (int)((V + 2047) / 2048);
  const int maxP = (4 * dn_sm_count()) / tiles > 1 ? (4 * dn_sm_count()) / tiles : 1;
  if (P > maxP) P = maxP;
  if (P < 1) P = 1;
  while (P * slice_floats > ws_floats && P > 1) --P;
  if (P * slice_floats > ws_floats) return DN_ERR_WORKSPACE;
  int64_t rps = (V + P - 1) / P;
  rps = (rps + round - 1) / round * round;
  if (rps < round) rps = round;
  P = (int)((V + rps - 1) / rps);
  *P_out = P < 1 ? 1 : P;
  *rps_out = rps;
  return DN_OK;
}

int simt_atb_partial_st(const float* A, int64_t lda, int I, const float* B, int64_t ldb, int J, const float* scale,
                        int64_t V, float* ws, int64_t ws_floats, int* P_out, cudaStream_t st) {
  const int tiles = ((I + 63) / 64) * ((J + 63) / 64);
  int P;
  int64_t rps;
  if (plan_row_slices(V, tiles, (int64_t)I * J, ws_floats, 16, &P, &rps)) return DN_ERR_WORKSPACE;
  atb_partial_kernel<<<dim3(tiles, P), 256, 0, st>>>(A, lda, I, B, ldb, J, scale, V, rps, ws);
  DN_LAUNCH_CHECK();
  *P_out = P;
  return DN_OK;
}

int simt_atb(const float* A, int64_t lda, int I, const float* B, int64_t ldb, int J, const float* scale, int64_t V,
             float* out, int64_t ld_out, int accumulate, float* ws, int64_t ws_floats, cudaStream_t st) {
  int P = 0;
  int rc = simt_atb_partial_st(A, lda, I, B, ldb, J, scale, V, ws, ws_floats, &P, st);
  if (rc) return rc;
  return launch_reduce_partials(ws, P, nullptr, 1, I, J, out, ld_out, accumulate, st);
}

int simt_colsum(const float* A, int64_t lda, int N, int64_t V, float* out, int accumulate, float* ws,
                int64_t ws_floats, cudaStream_t st) {
  if (V <= 0) {
    if (!accumulate) DN_CUDA_TRY(cudaMemsetAsync(out, 0, sizeof(float) * N, st));
    return DN_OK;
  }
  const int tiles = (N + 31) / 32;
  int P;
  int64_t rps;
  if (plan_row_slices(V, tiles, N, ws_floats, 1, &P, &rps)) return DN_ERR_WORKSPACE;
  colsum_partial_kernel<<<dim3(P, tiles), dim3(32, 8), 0, st>>>(A, lda, N, V, rps, ws);
  DN_LAUNCH_CHECK();
  return launch_reduce_partials(ws, P, nullptr, 1, 1, N, out, N, accumulate, st);
}

int launch_spectral_scale(const float* partial, int P, const float* evals, float* time, int K, int C,
                          float* x_spec_out, float* S_out, int clamp_writeback, cudaStream_t st) {
  spectral_scale_kernel<<<(K * C + 63) / 64, 256, 0, st>>>(partial, P, evals, time, K, C, x_spec_out, S_out,
                                                            clamp_writeback);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_reduce_partials(const float* partial, int P, const int32_t* mesh_cta_begin, int n_meshes, int64_t rows,
                           int cols, float* out, int64_t ld_out, int accumulate, cudaStream_t st) {
  const int64_t n = rows * cols;
  reduce_partials_kernel<<<dim3((unsigned)((n + 255) / 256), mesh_cta_begin ? (unsigned)n_meshes : 1u), 256, 0, st>>>(
      partial, P, mesh_cta_begin, rows, cols, out, ld_out, accumulate);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_spectral_bwd(const float* gs_partial, int P, const float* evals, const float* time, const float* x_spec,
                        int K, int C, float* dS, float* grad_time, cudaStream_t st) {
  spectral_bwd_kernel<<<(C + 63) / 64, 64, 0, st>>>(gs_partial, P, evals, time, x_spec, K, C, dS, grad_time);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_spectral_time_grad_batched(const float* G, const float* x_spec, const float* evals, const float* time,
                                      int n_meshes, int K, int C, float* grad_time, cudaStream_t st) {
  spectral_time_grad_batched_kernel<<<(C + 31) / 32, dim3(32, 16), 0, st>>>(G, x_spec, evals, time, n_meshes * K, C,
                                                                           grad_time);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_csr_from_coo(const int64_t* rows, const int64_t* cols, const float* vx, const float* vy, int64_t nnz,
                        int64_t V, int32_t* rowptr, int32_t* colidx, float* vals, cudaStream_t st) {
  if (nnz == 0) {
    DN_CUDA_TRY(cudaMemsetAsync(rowptr, 0, sizeof(int32_t) * (V + 1), st));
    return DN_OK;
  }
  csr_from_coo_kernel<<<(unsigned)((nnz + 255) / 256), 256, 0, st>>>(rows, cols, vx, vy, nnz, V, rowptr, colidx, vals);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_grad_spmm_pair(const dn_csr* g, const float* x, int64_t V, int C, float* out, cudaStream_t st) {
  if (V <= 0) return DN_OK;
  const int64_t threads = V * 32;
  grad_spmm_pair_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(
      g->rowptr, g->colidx, reinterpret_cast<const float2*>(g->vals), x, V, C, out);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_spmm_features(const dn_csr* g, const float* xd, const float* pq, int rotations, int64_t V, int C,
                         float* feat, cudaStream_t st) {
  if (V <= 0) return DN_OK;
  const float2* vals = reinterpret_cast<const float2*>(g->vals);
  // the patched kernel when the host built patches for this operator (bit-identical to the plain kernel, both ROT
  // variants).  C == 128 only: that is the shape validated on the GPU; the phase-2 shuffles also assume every lane owns
  // a float4 of the row (C/4 a multiple of 32)
  if (g->patches && g->patches->n_patches > 0 && C == 128) {
    const dn_patches& P = *g->patches;
    const int ld = rotations ? 2 * C : C;
    const size_t smem = (size_t)P.max_src * (size_t)(C + ld) * 4;
    if (smem <= 227 * 1024) {
      static size_t attr_set[2] = {0, 0};
      if (smem > attr_set[rotations ? 1 : 0]) {
        DN_CUDA_TRY(rotations ? cudaFuncSetAttribute(spmm_features_patch_kernel<true>,
                                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                              : cudaFuncSetAttribute(spmm_features_patch_kernel<false>,
                                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set[rotations ? 1 : 0] = smem;
      }
      if (rotations) spmm_features_patch_kernel<true><<<(unsigned)P.n_patches, 512, smem, st>>>(P, xd, pq, ld, C, feat);
      else spmm_features_patch_kernel<false><<<(unsigned)P.n_patches, 512, smem, st>>>(P, xd, pq, ld, C, feat);
      DN_LAUNCH_CHECK();
      return DN_OK;
    }
  }
  if (C == 128 || C == 256) {
    const unsigned ctas = (unsigned)((V + GB_ROWS - 1) / GB_ROWS);
    const int ld = rotations ? 2 * C : C;
#define DN_BLK_LAUNCH(ROT_, NH_) \
    spmm_features_blk_kernel<ROT_, NH_><<<ctas, 256, 0, st>>>(g->rowptr, g->colidx, vals, xd, pq, ld, V, feat)
    if (rotations) { if (C == 128) DN_BLK_LAUNCH(true, 1); else DN_BLK_LAUNCH(true, 2); }
    else { if (C == 128) DN_BLK_LAUNCH(false, 1); else DN_BLK_LAUNCH(false, 2); }
#undef DN_BLK_LAUNCH
    DN_LAUNCH_CHECK();
    return DN_OK;
  }
  return launch_feat_rows(V, C, rotations, [&](auto rot, auto lane, unsigned blocks, int G) {
    spmm_features_kernel<decltype(rot)::value, decltype(lane)><<<blocks, 256, 0, st>>>(
        g->rowptr, g->colidx, vals, xd, pq, rot ? 2 * C : C, V, C, G, feat);
  });
}

int launch_features_bwd_local(const dn_csr* g, const float* xd, const float* pq, const float* feat,
                              const float* dfeat, int rotations, int64_t V, int C, float* U, cudaStream_t st) {
  const float2* vals = reinterpret_cast<const float2*>(g->vals);
  return launch_feat_rows(V, C, rotations, [&](auto rot, auto lane, unsigned blocks, int G) {
    features_bwd_local_kernel<decltype(rot)::value, decltype(lane)><<<blocks, 256, 0, st>>>(
        g->rowptr, g->colidx, vals, xd, pq, rot ? 2 * C : C, feat, dfeat, V, C, G, U);
  });
}

int launch_features_bwd_transpose(const dn_csr* gt, const float* U, int rotations, int64_t V, int C, float* dxd,
                                  float* dP, float* dQ, int64_t ld_pq, cudaStream_t st) {
  const float2* vals = reinterpret_cast<const float2*>(gt->vals);
  return launch_feat_rows(V, C, rotations, [&](auto rot, auto lane, unsigned blocks, int G) {
    features_bwd_transpose_kernel<decltype(rot)::value, decltype(lane)><<<blocks, 256, 0, st>>>(
        gt->rowptr, gt->colidx, vals, U, V, C, G, dxd, dP, dQ, ld_pq);
  });
}

int launch_deinterleave_vc2(const float* vc2, int64_t V, int C, float* g01, cudaStream_t st) {
  const int64_t n = V * C;
  if (n <= 0) return DN_OK;
  deinterleave_vc2_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float2*>(vc2), V, C, g01);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_complex_dots_tanh(const float* g01, const float* b01, int64_t V, int C, float* out, cudaStream_t st) {
  const int64_t n = V * C;
  if (n <= 0) return DN_OK;
  complex_dots_tanh_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(g01, b01, V, C, out);
  DN_LAUNCH_CHECK();
  return DN_OK;
}
