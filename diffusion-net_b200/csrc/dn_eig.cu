// Kernels of the Laplace-Beltrami eigensolver (Chebyshev-filtered subspace iteration, Zhou & Saad), fp64 throughout.
// The solver runs on A = M^-1/2 (L + eps I) M^-1/2, held as the Laplacian's CSR pattern with values d_v d_k L_vk plus a
// diagonal shift (dn_mesh_laplacian), on a V x n block stored row-major.  Everything here is bandwidth-bound streaming
// over that block: one warp per row for the sparse filter step, 64 x 64 output tiles for the two dense contractions.
// No atomics: the reductions over V are split into partial sums that are added in a fixed order, so every result is
// bitwise reproducible.
//
// Every step has one __device__ body, run by a single-mesh kernel and by its batched form (dn_eig_batch): mesh b owns
// rows [row_begin[b], row_begin[b + 1]) of every block and of one block-diagonal CSR.  The kernels differ only in how
// they find their rows, coefficients and output slot.  A single mesh's reductions are split into eig_splits(V) row
// ranges; a batch's row tiles (DN_EIG_TILE_ROWS) and reduction slices (DN_EIG_SLICE_ROWS) are cut inside each mesh from
// its first row, so what a mesh's rows receive -- and the order its partial sums are added in -- depends on that mesh
// alone, not on which meshes share the batch.  Meshes with active[b] == 0 are skipped by every batched kernel.
#include <type_traits>

#include "dn_internal.h"

namespace {

constexpr int kTile = 64, kChunk = 32;
static_assert(DN_EIG_TILE_ROWS == kTile, "the batched rotate owns one 64-row tile per CTA");
static_assert(DN_EIG_SLICE_ROWS % DN_EIG_TILE_ROWS == 0, "slices are whole tiles");

// out[row] = alpha * (A Y)[row] + beta * Y[row] + gamma * Y_prev[row] over columns [0, n) of the caller's slice
// (n <= 32 * NC); lane l owns columns l, l + 32, ...  The row's pattern and values are broadcast to the warp.
// coef() returns (alpha, beta, gamma); it is called after the product, so a batched kernel reads its mesh's
// coefficients only then and does not hold them in registers across the row.
template <int NC, class Coef>
__device__ __forceinline__ void eig_filter_row(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                                               const double* __restrict__ avals, const double* __restrict__ adiag,
                                               int64_t row, int n, const double* __restrict__ Y,
                                               const double* __restrict__ Yp, int64_t ld, Coef coef,
                                               double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  double acc[NC];
  const double* yr = Y + row * ld;
  const double dg = adiag[row];
#pragma unroll
  for (int q = 0; q < NC; ++q) {
    const int c = lane + 32 * q;
    acc[q] = c < n ? dg * yr[c] : 0.0;
  }
  const int s = rowptr[row], e = rowptr[row + 1];
  for (int p = s; p < e; ++p) {
    const double a = avals[p];
    const double* yc = Y + (int64_t)colidx[p] * ld;
#pragma unroll
    for (int q = 0; q < NC; ++q) {
      const int c = lane + 32 * q;
      if (c < n) acc[q] = fma(a, yc[c], acc[q]);
    }
  }
  const double3 k = coef();
  double* o = out + row * ld;
  const double* pr = Yp ? Yp + row * ld : nullptr;
#pragma unroll
  for (int q = 0; q < NC; ++q) {
    const int c = lane + 32 * q;
    if (c < n) {
      double r = k.x * acc[q] + k.y * yr[c];
      if (pr) r += k.z * pr[c];
      o[c] = r;
    }
  }
}

// P[i][j] = sum over rows v in [r0, r1) of X[v][i] * Y[v][j] (P: m x n) on the CTA's 64 x 64 output tile
// (i0 = 64 blockIdx.y, j0 = 64 blockIdx.x); thread (tx, ty) owns i = i0 + ty + 16 a, j = j0 + tx + 16 b.
__device__ __forceinline__ void eig_gram_tile(const double* __restrict__ X, int64_t ldx, const double* __restrict__ Y,
                                              int64_t ldy, int64_t r0, int64_t r1, int m, int n,
                                              double* __restrict__ P) {
  __shared__ double xs[kChunk][kTile], ys[kChunk][kTile];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int i0 = blockIdx.y * kTile, j0 = blockIdx.x * kTile;
  double acc[4][4] = {};
  for (int64_t v0 = r0; v0 < r1; v0 += kChunk) {
    for (int e = t; e < kChunk * kTile; e += 256) {
      const int r = e / kTile, c = e % kTile;
      const bool rok = v0 + r < r1;
      xs[r][c] = (rok && i0 + c < m) ? X[(v0 + r) * ldx + i0 + c] : 0.0;
      ys[r][c] = (rok && j0 + c < n) ? Y[(v0 + r) * ldy + j0 + c] : 0.0;
    }
    __syncthreads();
#pragma unroll 4
    for (int r = 0; r < kChunk; ++r) {
      double xa[4], yb[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) xa[a] = xs[r][ty + 16 * a];
#pragma unroll
      for (int b = 0; b < 4; ++b) yb[b] = ys[r][tx + 16 * b];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = fma(xa[a], yb[b], acc[a][b]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int i = i0 + ty + 16 * a, j = j0 + tx + 16 * b;
      if (i < m && j < n) P[(int64_t)i * n + j] = acc[a][b];
    }
}

// sum_{p0 <= p < p1} partial[p][e], p ascending; optionally its square root
__device__ __forceinline__ double eig_sum_partials(const double* __restrict__ partial, int p0, int p1, int64_t count,
                                                   int64_t e, int take_sqrt) {
  double s = 0.0;
  for (int p = p0; p < p1; ++p) s += partial[(int64_t)p * count + e];
  return take_sqrt ? sqrt(s) : s;
}

// Z = beta * Z + X C on rows [v0, min(v0 + 64, v_end)) and the CTA's 64 columns (j0 = 64 blockIdx.x):
// X (rows x kd, ldx), C (kd x n, ldc), Z (rows x n, ldz)
__device__ __forceinline__ void eig_rotate_tile(const double* __restrict__ X, int64_t ldx, const double* __restrict__ Cm,
                                                int64_t ldc, int64_t v0, int64_t v_end, int kd, int n, double beta,
                                                double* __restrict__ Z, int64_t ldz) {
  __shared__ double xs[kTile][kChunk + 1], cs[kChunk][kTile];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int j0 = blockIdx.x * kTile;
  double acc[4][4] = {};
  for (int k0 = 0; k0 < kd; k0 += kChunk) {
    for (int e = t; e < kTile * kChunk; e += 256) {
      const int r = e / kChunk, c = e % kChunk;
      xs[r][c] = (v0 + r < v_end && k0 + c < kd) ? X[(v0 + r) * ldx + k0 + c] : 0.0;
      const int r2 = e / kTile, c2 = e % kTile;
      cs[r2][c2] = (k0 + r2 < kd && j0 + c2 < n) ? Cm[(int64_t)(k0 + r2) * ldc + j0 + c2] : 0.0;
    }
    __syncthreads();
#pragma unroll 4
    for (int kk = 0; kk < kChunk; ++kk) {
      double xa[4], cb[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) xa[a] = xs[ty + 16 * a][kk];
#pragma unroll
      for (int b = 0; b < 4; ++b) cb[b] = cs[kk][tx + 16 * b];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = fma(xa[a], cb[b], acc[a][b]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int64_t v = v0 + ty + 16 * a;
      const int j = j0 + tx + 16 * b;
      if (v < v_end && j < n) {
        double* z = Z + v * ldz + j;
        *z = beta == 0.0 ? acc[a][b] : fma(beta, *z, acc[a][b]);
      }
    }
}

// partial[c] = sum over rows v in [r0, r1) of (W[v][c] - theta[c] Q[v][c])^2 for the CTA's 32 columns
// (c = 32 blockIdx.x + tx); 8 row lanes, lane ty summing rows r0 + ty, r0 + ty + 8, ..., then the lanes in order
__device__ __forceinline__ void eig_resid_cols(const double* __restrict__ W, int64_t ldw, const double* __restrict__ Q,
                                               int64_t ldq, const double* __restrict__ theta, int64_t r0, int64_t r1,
                                               int n, double* __restrict__ partial) {
  __shared__ double part[8][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  double s = 0.0;
  if (c < n) {
    const double th = theta[c];
    for (int64_t v = r0 + ty; v < r1; v += 8) {
      const double d = W[v * ldw + c] - th * Q[v * ldq + c];
      s = fma(d, d, s);
    }
  }
  part[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && c < n) {
    double r = 0.0;
    for (int i = 0; i < 8; ++i) r += part[i][tx];
    partial[c] = r;
  }
}

// *sign = sign of the largest-magnitude entry of rows [r0, r1) of column c of phi = M^-1/2 Y (lowest row on ties;
// +1 for 0), r1 the index of "no row"
__device__ __forceinline__ void eig_colsign_col(const double* __restrict__ Y, int64_t ldy, int c,
                                                const double* __restrict__ mass, int32_t r0, int32_t r1,
                                                double* __restrict__ sign) {
  __shared__ double bv[256], bx[256];
  __shared__ int32_t bi[256];
  const int t = threadIdx.x;
  double best = -1.0, bval = 0.0;
  int32_t bidx = r1;
  for (int32_t v = r0 + t; v < r1; v += 256) {
    const double x = Y[(int64_t)v * ldy + c] / sqrt(mass[v]);
    if (fabs(x) > best) { best = fabs(x); bidx = v; bval = x; }   // ascending v per thread: the first maximum stays
  }
  bv[t] = best;
  bi[t] = bidx;
  bx[t] = bval;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (t < o) {
      const bool take = bv[t + o] > bv[t] || (bv[t + o] == bv[t] && bi[t + o] < bi[t]);
      if (take) { bv[t] = bv[t + o]; bi[t] = bi[t + o]; bx[t] = bx[t + o]; }
    }
    __syncthreads();
  }
  if (t == 0) *sign = bx[0] < 0.0 ? -1.0 : 1.0;
}

// sign[i] * Y[v][cols[i]] / sqrt(mass[v])
__device__ __forceinline__ double eig_gather_entry(const double* __restrict__ Y, int64_t ldy,
                                                   const int32_t* __restrict__ cols, const double* __restrict__ sign,
                                                   const double* __restrict__ mass, int64_t v, int i) {
  return sign[i] * (Y[v * ldy + cols[i]] / sqrt(mass[v]));
}

// ---- single mesh: rows [0, V) --------------------------------------------------------------------------------------

template <int NC>
__global__ void __launch_bounds__(256) eig_filter_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                                                         const double* __restrict__ avals, const double* __restrict__ adiag,
                                                         int64_t V, int n, const double* __restrict__ Y,
                                                         const double* __restrict__ Yp, int64_t ld, double alpha,
                                                         double beta, double gamma, double* __restrict__ out) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row < V)
    eig_filter_row<NC>(rowptr, colidx, avals, adiag, row, n, Y, Yp, ld, [=] { return make_double3(alpha, beta, gamma); },
                       out);
}

// split blockIdx.z = rows [z rows_per, (z + 1) rows_per) into partial[z]
__global__ void __launch_bounds__(256) eig_gram_partial_kernel(const double* __restrict__ X, int64_t ldx,
                                                               const double* __restrict__ Y, int64_t ldy, int64_t V, int m,
                                                               int n, int64_t rows_per, double* __restrict__ partial) {
  const int64_t r0 = (int64_t)blockIdx.z * rows_per, r1 = r0 + rows_per < V ? r0 + rows_per : V;
  eig_gram_tile(X, ldx, Y, ldy, r0, r1, m, n, partial + (int64_t)blockIdx.z * m * n);
}

__global__ void eig_reduce_kernel(const double* __restrict__ partial, int P, int64_t count, int take_sqrt,
                                  double* __restrict__ out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < count) out[e] = eig_sum_partials(partial, 0, P, count, e, take_sqrt);
}

__global__ void __launch_bounds__(256) eig_rotate_kernel(const double* __restrict__ X, int64_t ldx,
                                                         const double* __restrict__ Cm, int64_t ldc, int64_t V, int kd, int n,
                                                         double beta, double* __restrict__ Z, int64_t ldz) {
  eig_rotate_tile(X, ldx, Cm, ldc, (int64_t)blockIdx.y * kTile, V, kd, n, beta, Z, ldz);
}

__global__ void __launch_bounds__(256) eig_resid_partial_kernel(const double* __restrict__ W, int64_t ldw,
                                                                const double* __restrict__ Q, int64_t ldq,
                                                                const double* __restrict__ theta, int64_t V, int n,
                                                                int64_t rows_per, double* __restrict__ partial) {
  const int64_t r0 = (int64_t)blockIdx.y * rows_per, r1 = r0 + rows_per < V ? r0 + rows_per : V;
  eig_resid_cols(W, ldw, Q, ldq, theta, r0, r1, n, partial + (int64_t)blockIdx.y * n);
}

// column cols[blockIdx.x]
__global__ void __launch_bounds__(256) eig_colsign_kernel(const double* __restrict__ Y, int64_t ldy,
                                                          const int32_t* __restrict__ cols, const double* __restrict__ mass,
                                                          int64_t V, double* __restrict__ sign) {
  eig_colsign_col(Y, ldy, cols[blockIdx.x], mass, 0, (int32_t)V, sign + blockIdx.x);
}

// one thread per entry of the V x k output
__global__ void eig_gather_kernel(const double* __restrict__ Y, int64_t ldy, const int32_t* __restrict__ cols,
                                  const double* __restrict__ sign, const double* __restrict__ mass, int64_t V, int k,
                                  double* __restrict__ out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= V * k) return;
  out[e] = eig_gather_entry(Y, ldy, cols, sign, mass, e / k, (int)(e % k));
}

// row splits of the partial sums: a function of V alone (so equal inputs reduce in the same order), 4096 rows or more
int eig_splits(int64_t V) {
  int64_t p = V / 4096;
  return (int)(p < 1 ? 1 : (p > 64 ? 64 : p));
}

// ---- batch of meshes -----------------------------------------------------------------------------------------------

// (alpha, beta, gamma) per mesh; 8 warps = 8 rows per CTA, 8 CTAs per 64-row tile
template <int NC>
__global__ void __launch_bounds__(256) eig_filter_batched_kernel(const int32_t* __restrict__ rowptr,
                                                                 const int32_t* __restrict__ colidx,
                                                                 const double* __restrict__ avals,
                                                                 const double* __restrict__ adiag, dn_eig_batch bt, int n,
                                                                 const double* __restrict__ Y, const double* __restrict__ Yp,
                                                                 int64_t ld, const double* __restrict__ alpha,
                                                                 const double* __restrict__ beta,
                                                                 const double* __restrict__ gamma,
                                                                 const int32_t* __restrict__ active, double* __restrict__ out) {
  const int tile = blockIdx.x >> 3;
  const int b = bt.tile_mesh[tile];
  if (active && !active[b]) return;
  const int64_t row = (int64_t)bt.row_begin[b] + (int64_t)(tile - bt.tile_begin[b]) * DN_EIG_TILE_ROWS +
                      (blockIdx.x & 7) * 8 + (threadIdx.x >> 5);
  if (row < bt.row_begin[b + 1])
    eig_filter_row<NC>(rowptr, colidx, avals, adiag, row, n, Y, Yp, ld,
                       [=] { return make_double3(alpha[b], beta[b], gamma[b]); }, out);
}

// slice blockIdx.z of its mesh into partial[z]
__global__ void __launch_bounds__(256) eig_gram_batched_kernel(const double* __restrict__ X, int64_t ldx,
                                                               const double* __restrict__ Y, int64_t ldy, dn_eig_batch bt,
                                                               int m, int n, const int32_t* __restrict__ active,
                                                               double* __restrict__ partial) {
  const int b = bt.slice_mesh[blockIdx.z];
  if (active && !active[b]) return;
  const int64_t r0 = (int64_t)bt.row_begin[b] + (int64_t)(blockIdx.z - bt.slice_begin[b]) * DN_EIG_SLICE_ROWS;
  const int64_t re = bt.row_begin[b + 1], r1 = r0 + DN_EIG_SLICE_ROWS < re ? r0 + DN_EIG_SLICE_ROWS : re;
  eig_gram_tile(X, ldx, Y, ldy, r0, r1, m, n, partial + (int64_t)blockIdx.z * m * n);
}

// out[b][e] over the slices of mesh b = blockIdx.y
__global__ void eig_reduce_batched_kernel(const double* __restrict__ partial, dn_eig_batch bt, int64_t count, int take_sqrt,
                                          const int32_t* __restrict__ active, double* __restrict__ out) {
  const int b = blockIdx.y;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= count || (active && !active[b])) return;
  out[(int64_t)b * count + e] = eig_sum_partials(partial, bt.slice_begin[b], bt.slice_begin[b + 1], count, e, take_sqrt);
}

// tile blockIdx.y with its mesh's own kd x n C
__global__ void __launch_bounds__(256) eig_rotate_batched_kernel(const double* __restrict__ X, int64_t ldx,
                                                                 const double* __restrict__ Cm, dn_eig_batch bt, int kd, int n,
                                                                 double beta, const int32_t* __restrict__ active,
                                                                 double* __restrict__ Z, int64_t ldz) {
  const int b = bt.tile_mesh[blockIdx.y];
  if (active && !active[b]) return;
  const int64_t v0 = (int64_t)bt.row_begin[b] + (int64_t)(blockIdx.y - bt.tile_begin[b]) * kTile;
  eig_rotate_tile(X, ldx, Cm + (int64_t)b * kd * n, n, v0, bt.row_begin[b + 1], kd, n, beta, Z, ldz);
}

// slice blockIdx.y of its mesh with the mesh's own theta (n per mesh)
__global__ void __launch_bounds__(256) eig_resid_batched_kernel(const double* __restrict__ W, int64_t ldw,
                                                                const double* __restrict__ Q, int64_t ldq,
                                                                const double* __restrict__ theta, dn_eig_batch bt, int n,
                                                                const int32_t* __restrict__ active,
                                                                double* __restrict__ partial) {
  const int b = bt.slice_mesh[blockIdx.y];
  if (active && !active[b]) return;
  const int64_t r0 = (int64_t)bt.row_begin[b] + (int64_t)(blockIdx.y - bt.slice_begin[b]) * DN_EIG_SLICE_ROWS;
  const int64_t re = bt.row_begin[b + 1], r1 = r0 + DN_EIG_SLICE_ROWS < re ? r0 + DN_EIG_SLICE_ROWS : re;
  eig_resid_cols(W, ldw, Q, ldq, theta + (int64_t)b * n, r0, r1, n, partial + (int64_t)blockIdx.y * n);
}

// column blockIdx.x of mesh blockIdx.y: cols and sign are (n_meshes, k)
__global__ void __launch_bounds__(256) eig_colsign_batched_kernel(const double* __restrict__ Y, int64_t ldy,
                                                                  const int32_t* __restrict__ cols,
                                                                  const double* __restrict__ mass, dn_eig_batch bt,
                                                                  double* __restrict__ sign) {
  const int b = blockIdx.y;
  const unsigned i = b * gridDim.x + blockIdx.x;
  eig_colsign_col(Y, ldy, cols[i], mass, bt.row_begin[b], bt.row_begin[b + 1], sign + i);
}

// the rows of tile blockIdx.x, b its mesh
__global__ void __launch_bounds__(256) eig_gather_batched_kernel(const double* __restrict__ Y, int64_t ldy,
                                                                 const int32_t* __restrict__ cols,
                                                                 const double* __restrict__ sign,
                                                                 const double* __restrict__ mass, dn_eig_batch bt, int k,
                                                                 double* __restrict__ out) {
  const int b = bt.tile_mesh[blockIdx.x];
  const int64_t v0 = (int64_t)bt.row_begin[b] + (int64_t)(blockIdx.x - bt.tile_begin[b]) * DN_EIG_TILE_ROWS;
  const int64_t left = bt.row_begin[b + 1] - v0;
  const int rows = (int)(left < DN_EIG_TILE_ROWS ? left : DN_EIG_TILE_ROWS);
  for (int e = threadIdx.x; e < rows * k; e += 256) {
    const int64_t v = v0 + e / k;
    const int i = e % k;
    out[v * k + i] = eig_gather_entry(Y, ldy, cols, sign, mass, v, b * k + i);
  }
}

// Calls launch(std::integral_constant<int, NC>(), w, Y + c0, Y_prev + c0, out + c0) on column slices [c0, c0 + w) of at
// most 256 columns (8 per lane), NC = ceil(w / 32): the one instantiation switch of both filter launchers.
template <class Launch>
int eig_filter_slices(int n, const double* Y, const double* Yp, double* out, Launch launch) {
  for (int c0 = 0; c0 < n; c0 += 256) {
    const int w = n - c0 < 256 ? n - c0 : 256;
    const double* y = Y + c0;
    const double* yp = Yp ? Yp + c0 : nullptr;
    double* o = out + c0;
    switch ((w + 31) / 32) {
      case 1: launch(std::integral_constant<int, 1>(), w, y, yp, o); break;
      case 2: launch(std::integral_constant<int, 2>(), w, y, yp, o); break;
      case 3: launch(std::integral_constant<int, 3>(), w, y, yp, o); break;
      case 4: launch(std::integral_constant<int, 4>(), w, y, yp, o); break;
      case 5: launch(std::integral_constant<int, 5>(), w, y, yp, o); break;
      case 6: launch(std::integral_constant<int, 6>(), w, y, yp, o); break;
      case 7: launch(std::integral_constant<int, 7>(), w, y, yp, o); break;
      default: launch(std::integral_constant<int, 8>(), w, y, yp, o); break;
    }
    DN_LAUNCH_CHECK();
  }
  return DN_OK;
}

}  // namespace

int64_t eig_gram_ws_bytes(int64_t V, int m, int n) { return 8ll * eig_splits(V) * m * n; }
int64_t eig_resid_ws_bytes(int64_t V, int n) { return 8ll * eig_splits(V) * n; }

int launch_eig_filter(const int32_t* rowptr, const int32_t* colidx, const double* avals, const double* adiag, int64_t V,
                      int n, const double* Y, const double* Yp, int64_t ld, double alpha, double beta, double gamma,
                      double* out, cudaStream_t st) {
  if (V <= 0 || n <= 0) return DN_OK;
  const unsigned blocks = (unsigned)((V * 32 + 255) / 256);
  return eig_filter_slices(n, Y, Yp, out, [&](auto nc, int w, const double* y, const double* yp, double* o) {
    eig_filter_kernel<decltype(nc)::value><<<blocks, 256, 0, st>>>(rowptr, colidx, avals, adiag, V, w, y, yp, ld, alpha,
                                                                   beta, gamma, o);
  });
}

int launch_eig_gram(const double* X, int64_t ldx, const double* Y, int64_t ldy, int64_t V, int m, int n, double* out,
                    double* ws, cudaStream_t st) {
  if (m <= 0 || n <= 0) return DN_OK;
  if (V <= 0) {
    DN_CUDA_TRY(cudaMemsetAsync(out, 0, sizeof(double) * m * n, st));
    return DN_OK;
  }
  const int P = eig_splits(V);
  const int64_t rows_per = (V + P - 1) / P;
  dim3 grid((unsigned)((n + kTile - 1) / kTile), (unsigned)((m + kTile - 1) / kTile), (unsigned)P);
  eig_gram_partial_kernel<<<grid, 256, 0, st>>>(X, ldx, Y, ldy, V, m, n, rows_per, ws);
  DN_LAUNCH_CHECK();
  const int64_t cnt = (int64_t)m * n;
  eig_reduce_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(ws, P, cnt, 0, out);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_eig_rotate(const double* X, int64_t ldx, const double* Cm, int64_t ldc, int64_t V, int kd, int n, double beta,
                      double* Z, int64_t ldz, cudaStream_t st) {
  if (V <= 0 || n <= 0) return DN_OK;
  dim3 grid((unsigned)((n + kTile - 1) / kTile), (unsigned)((V + kTile - 1) / kTile));
  eig_rotate_kernel<<<grid, 256, 0, st>>>(X, ldx, Cm, ldc, V, kd, n, beta, Z, ldz);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_eig_residual_norms(const double* W, int64_t ldw, const double* Q, int64_t ldq, const double* theta, int64_t V,
                              int n, double* out, double* ws, cudaStream_t st) {
  if (n <= 0) return DN_OK;
  if (V <= 0) {
    DN_CUDA_TRY(cudaMemsetAsync(out, 0, sizeof(double) * n, st));
    return DN_OK;
  }
  const int P = eig_splits(V);
  const int64_t rows_per = (V + P - 1) / P;
  eig_resid_partial_kernel<<<dim3((unsigned)((n + 31) / 32), (unsigned)P), 256, 0, st>>>(W, ldw, Q, ldq, theta, V, n,
                                                                                        rows_per, ws);
  DN_LAUNCH_CHECK();
  eig_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ws, P, n, 1, out);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_eig_finalize(const double* Y, int64_t ldy, const int32_t* cols, int k, const double* mass, int64_t V,
                        double* out, double* sign_ws, cudaStream_t st) {
  if (V <= 0 || k <= 0) return DN_OK;
  eig_colsign_kernel<<<(unsigned)k, 256, 0, st>>>(Y, ldy, cols, mass, V, sign_ws);
  DN_LAUNCH_CHECK();
  eig_gather_kernel<<<(unsigned)((V * k + 255) / 256), 256, 0, st>>>(Y, ldy, cols, sign_ws, mass, V, k, out);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int64_t eig_gram_batched_ws_bytes(int n_slices, int m, int n) { return 8ll * n_slices * m * n; }
int64_t eig_resid_batched_ws_bytes(int n_slices, int n) { return 8ll * n_slices * n; }

int launch_eig_filter_batched(const int32_t* rowptr, const int32_t* colidx, const double* avals, const double* adiag,
                              const dn_eig_batch* bt, int n, const double* Y, const double* Yp, int64_t ld,
                              const double* alpha, const double* beta, const double* gamma, const int32_t* active,
                              double* out, cudaStream_t st) {
  if (bt->n_tiles <= 0 || n <= 0) return DN_OK;
  const unsigned blocks = (unsigned)bt->n_tiles * 8u;
  return eig_filter_slices(n, Y, Yp, out, [&](auto nc, int w, const double* y, const double* yp, double* o) {
    eig_filter_batched_kernel<decltype(nc)::value><<<blocks, 256, 0, st>>>(rowptr, colidx, avals, adiag, *bt, w, y, yp, ld,
                                                                           alpha, beta, gamma, active, o);
  });
}

int launch_eig_gram_batched(const double* X, int64_t ldx, const double* Y, int64_t ldy, const dn_eig_batch* bt, int m, int n,
                            const int32_t* active, double* out, double* ws, cudaStream_t st) {
  if (m <= 0 || n <= 0 || bt->n_meshes <= 0) return DN_OK;
  dim3 grid((unsigned)((n + kTile - 1) / kTile), (unsigned)((m + kTile - 1) / kTile), (unsigned)bt->n_slices);
  eig_gram_batched_kernel<<<grid, 256, 0, st>>>(X, ldx, Y, ldy, *bt, m, n, active, ws);
  DN_LAUNCH_CHECK();
  const int64_t cnt = (int64_t)m * n;
  eig_reduce_batched_kernel<<<dim3((unsigned)((cnt + 255) / 256), (unsigned)bt->n_meshes), 256, 0, st>>>(ws, *bt, cnt, 0,
                                                                                                       active, out);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_eig_rotate_batched(const double* X, int64_t ldx, const double* Cm, const dn_eig_batch* bt, int kd, int n,
                              double beta, const int32_t* active, double* Z, int64_t ldz, cudaStream_t st) {
  if (bt->n_tiles <= 0 || n <= 0) return DN_OK;
  dim3 grid((unsigned)((n + kTile - 1) / kTile), (unsigned)bt->n_tiles);
  eig_rotate_batched_kernel<<<grid, 256, 0, st>>>(X, ldx, Cm, *bt, kd, n, beta, active, Z, ldz);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_eig_residual_norms_batched(const double* W, int64_t ldw, const double* Q, int64_t ldq, const double* theta,
                                      const dn_eig_batch* bt, int n, const int32_t* active, double* out, double* ws,
                                      cudaStream_t st) {
  if (n <= 0 || bt->n_meshes <= 0) return DN_OK;
  eig_resid_batched_kernel<<<dim3((unsigned)((n + 31) / 32), (unsigned)bt->n_slices), 256, 0, st>>>(W, ldw, Q, ldq, theta,
                                                                                                   *bt, n, active, ws);
  DN_LAUNCH_CHECK();
  eig_reduce_batched_kernel<<<dim3((unsigned)((n + 255) / 256), (unsigned)bt->n_meshes), 256, 0, st>>>(ws, *bt, n, 1,
                                                                                                     active, out);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_eig_finalize_batched(const double* Y, int64_t ldy, const int32_t* cols, int k, const double* mass,
                                const dn_eig_batch* bt, double* out, double* sign_ws, cudaStream_t st) {
  if (bt->n_tiles <= 0 || k <= 0) return DN_OK;
  eig_colsign_batched_kernel<<<dim3((unsigned)k, (unsigned)bt->n_meshes), 256, 0, st>>>(Y, ldy, cols, mass, *bt, sign_ws);
  DN_LAUNCH_CHECK();
  eig_gather_batched_kernel<<<(unsigned)bt->n_tiles, 256, 0, st>>>(Y, ldy, cols, sign_ws, mass, *bt, k, out);
  DN_LAUNCH_CHECK();
  return DN_OK;
}
