// Kernels of the Laplace-Beltrami eigensolver (Chebyshev-filtered subspace iteration, Zhou & Saad), fp64 throughout.
// The solver runs on A = M^-1/2 (L + eps I) M^-1/2, held as the Laplacian's CSR pattern with values d_v d_k L_vk plus a
// diagonal shift (dn_mesh_laplacian), on a V x n block stored row-major.  Everything here is bandwidth-bound streaming
// over that block: one warp per row for the sparse filter step, 64 x 64 output tiles for the two dense contractions.
// No atomics: the reductions over V are split into partial sums that are added in a fixed order, so every result is
// bitwise reproducible.
#include "dn_internal.h"

namespace {

// Y_out = alpha * (A Y) + beta * Y + gamma * Y_prev over columns [0, 32 * NC) of the caller's slice (n <= 32 * NC);
// lane l owns columns l, l + 32, ...  The row's pattern and values are broadcast to the warp.
template <int NC>
__global__ void __launch_bounds__(256) eig_filter_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                                                         const double* __restrict__ avals, const double* __restrict__ adiag,
                                                         int64_t V, int n, const double* __restrict__ Y,
                                                         const double* __restrict__ Yp, int64_t ld, double alpha,
                                                         double beta, double gamma, double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= V) return;
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
  double* o = out + row * ld;
  const double* pr = Yp ? Yp + row * ld : nullptr;
#pragma unroll
  for (int q = 0; q < NC; ++q) {
    const int c = lane + 32 * q;
    if (c < n) {
      double r = alpha * acc[q] + beta * yr[c];
      if (pr) r += gamma * pr[c];
      o[c] = r;
    }
  }
}

constexpr int kTile = 64, kChunk = 32;

// partial[p][i][j] = sum over rows v of split p of X[v][i] * Y[v][j]; CTA (bx, by, p) owns the 64 x 64 output tile
// (i0 = 64 by, j0 = 64 bx); thread (tx, ty) owns i = i0 + ty + 16 a, j = j0 + tx + 16 b.
__global__ void __launch_bounds__(256) eig_gram_partial_kernel(const double* __restrict__ X, int64_t ldx,
                                                               const double* __restrict__ Y, int64_t ldy, int64_t V, int m,
                                                               int n, int64_t rows_per, double* __restrict__ partial) {
  __shared__ double xs[kChunk][kTile], ys[kChunk][kTile];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int i0 = blockIdx.y * kTile, j0 = blockIdx.x * kTile;
  const int64_t r0 = (int64_t)blockIdx.z * rows_per, r1 = r0 + rows_per < V ? r0 + rows_per : V;
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
  double* P = partial + (int64_t)blockIdx.z * m * n;
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int i = i0 + ty + 16 * a, j = j0 + tx + 16 * b;
      if (i < m && j < n) P[(int64_t)i * n + j] = acc[a][b];
    }
}

// out[e] = sum_{p < P} partial[p][e], p ascending; optionally its square root
__global__ void eig_reduce_kernel(const double* __restrict__ partial, int P, int64_t count, int take_sqrt,
                                  double* __restrict__ out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= count) return;
  double s = 0.0;
  for (int p = 0; p < P; ++p) s += partial[(int64_t)p * count + e];
  out[e] = take_sqrt ? sqrt(s) : s;
}

// Z = beta * Z + X C: X (V x kd, ldx), C (kd x n, ldc), Z (V x n, ldz); CTA owns 64 rows x 64 columns of Z
__global__ void __launch_bounds__(256) eig_rotate_kernel(const double* __restrict__ X, int64_t ldx,
                                                         const double* __restrict__ Cm, int64_t ldc, int64_t V, int kd, int n,
                                                         double beta, double* __restrict__ Z, int64_t ldz) {
  __shared__ double xs[kTile][kChunk + 1], cs[kChunk][kTile];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int64_t v0 = (int64_t)blockIdx.y * kTile;
  const int j0 = blockIdx.x * kTile;
  double acc[4][4] = {};
  for (int k0 = 0; k0 < kd; k0 += kChunk) {
    for (int e = t; e < kTile * kChunk; e += 256) {
      const int r = e / kChunk, c = e % kChunk;
      xs[r][c] = (v0 + r < V && k0 + c < kd) ? X[(v0 + r) * ldx + k0 + c] : 0.0;
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
      if (v < V && j < n) {
        double* z = Z + v * ldz + j;
        *z = beta == 0.0 ? acc[a][b] : fma(beta, *z, acc[a][b]);
      }
    }
}

// partial[p][c] = sum over rows of split p of (W[v][c] - theta[c] Q[v][c])^2; block = 32 columns x 8 row lanes
__global__ void __launch_bounds__(256) eig_resid_partial_kernel(const double* __restrict__ W, int64_t ldw,
                                                                const double* __restrict__ Q, int64_t ldq,
                                                                const double* __restrict__ theta, int64_t V, int n,
                                                                int64_t rows_per, double* __restrict__ partial) {
  __shared__ double part[8][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per, r1 = r0 + rows_per < V ? r0 + rows_per : V;
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
    partial[(int64_t)blockIdx.y * n + c] = r;
  }
}

// sign[i] = sign of the largest-magnitude entry of column i of phi = M^-1/2 Y[:, cols[i]] (lowest row on ties; +1 for 0)
__global__ void __launch_bounds__(256) eig_colsign_kernel(const double* __restrict__ Y, int64_t ldy,
                                                          const int32_t* __restrict__ cols, const double* __restrict__ mass,
                                                          int64_t V, double* __restrict__ sign) {
  __shared__ double bv[256], bx[256];
  __shared__ int32_t bi[256];
  const int t = threadIdx.x;
  const int c = cols[blockIdx.x];
  double best = -1.0, bval = 0.0;
  int32_t bidx = (int32_t)V;
  for (int32_t v = t; v < (int32_t)V; v += 256) {
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
  if (t == 0) sign[blockIdx.x] = bx[0] < 0.0 ? -1.0 : 1.0;
}

// out[v][i] = sign[i] * Y[v][cols[i]] / sqrt(mass[v])
__global__ void eig_gather_kernel(const double* __restrict__ Y, int64_t ldy, const int32_t* __restrict__ cols,
                                  const double* __restrict__ sign, const double* __restrict__ mass, int64_t V, int k,
                                  double* __restrict__ out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= V * k) return;
  const int64_t v = e / k;
  const int i = (int)(e % k);
  out[e] = sign[i] * (Y[v * ldy + cols[i]] / sqrt(mass[v]));
}

// row splits of the partial sums: a function of V alone (so equal inputs reduce in the same order), 4096 rows or more
int eig_splits(int64_t V) {
  int64_t p = V / 4096;
  return (int)(p < 1 ? 1 : (p > 64 ? 64 : p));
}


// ---------------------------------------------------------------------------------------------
// The same steps over a batch of meshes (dn_eig_batch): mesh b owns rows [row_begin[b], row_begin[b + 1]) of every block
// and of one block-diagonal CSR.  Row tiles (DN_EIG_TILE_ROWS) and reduction slices (DN_EIG_SLICE_ROWS) are cut inside
// each mesh from its first row, so what a mesh's rows receive -- and the order its partial sums are added in -- depends
// on that mesh alone, not on which meshes share the batch.  Meshes with active[b] == 0 are skipped by every kernel.
// ---------------------------------------------------------------------------------------------
static_assert(DN_EIG_TILE_ROWS == kTile, "the batched rotate owns one 64-row tile per CTA");
static_assert(DN_EIG_SLICE_ROWS % DN_EIG_TILE_ROWS == 0, "slices are whole tiles");

// eig_filter_kernel with (alpha, beta, gamma) per mesh; 8 warps = 8 rows per CTA, 8 CTAs per 64-row tile
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
  const int lane = threadIdx.x & 31;
  const int tile = blockIdx.x >> 3;
  const int b = bt.tile_mesh[tile];
  if (active && !active[b]) return;
  const int64_t row = (int64_t)bt.row_begin[b] + (int64_t)(tile - bt.tile_begin[b]) * DN_EIG_TILE_ROWS +
                      (blockIdx.x & 7) * 8 + (threadIdx.x >> 5);
  if (row >= bt.row_begin[b + 1]) return;
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
  const double al = alpha[b], be = beta[b], ga = gamma[b];
  double* o = out + row * ld;
  const double* pr = Yp ? Yp + row * ld : nullptr;
#pragma unroll
  for (int q = 0; q < NC; ++q) {
    const int c = lane + 32 * q;
    if (c < n) {
      double r = al * acc[q] + be * yr[c];
      if (pr) r += ga * pr[c];
      o[c] = r;
    }
  }
}

// eig_gram_partial_kernel on slice blockIdx.z: partial[slice][i][j] over the slice's rows
__global__ void __launch_bounds__(256) eig_gram_batched_kernel(const double* __restrict__ X, int64_t ldx,
                                                               const double* __restrict__ Y, int64_t ldy, dn_eig_batch bt,
                                                               int m, int n, const int32_t* __restrict__ active,
                                                               double* __restrict__ partial) {
  __shared__ double xs[kChunk][kTile], ys[kChunk][kTile];
  const int b = bt.slice_mesh[blockIdx.z];
  if (active && !active[b]) return;
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int i0 = blockIdx.y * kTile, j0 = blockIdx.x * kTile;
  const int64_t r0 = (int64_t)bt.row_begin[b] + (int64_t)(blockIdx.z - bt.slice_begin[b]) * DN_EIG_SLICE_ROWS;
  const int64_t re = bt.row_begin[b + 1], r1 = r0 + DN_EIG_SLICE_ROWS < re ? r0 + DN_EIG_SLICE_ROWS : re;
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
      for (int c = 0; c < 4; ++c) yb[c] = ys[r][tx + 16 * c];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][c] = fma(xa[a], yb[c], acc[a][c]);
    }
    __syncthreads();
  }
  double* P = partial + (int64_t)blockIdx.z * m * n;
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int i = i0 + ty + 16 * a, j = j0 + tx + 16 * c;
      if (i < m && j < n) P[(int64_t)i * n + j] = acc[a][c];
    }
}

// out[b][e] = sum of partial[s][e] over the slices s of mesh b, ascending; optionally its square root
__global__ void eig_reduce_batched_kernel(const double* __restrict__ partial, dn_eig_batch bt, int64_t count, int take_sqrt,
                                          const int32_t* __restrict__ active, double* __restrict__ out) {
  const int b = blockIdx.y;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= count || (active && !active[b])) return;
  double s = 0.0;
  for (int p = bt.slice_begin[b]; p < bt.slice_begin[b + 1]; ++p) s += partial[(int64_t)p * count + e];
  out[(int64_t)b * count + e] = take_sqrt ? sqrt(s) : s;
}

// eig_rotate_kernel on tile blockIdx.y with the mesh's own C
__global__ void __launch_bounds__(256) eig_rotate_batched_kernel(const double* __restrict__ X, int64_t ldx,
                                                                 const double* __restrict__ Cm, dn_eig_batch bt, int kd, int n,
                                                                 double beta, const int32_t* __restrict__ active,
                                                                 double* __restrict__ Z, int64_t ldz) {
  __shared__ double xs[kTile][kChunk + 1], cs[kChunk][kTile];
  const int b = bt.tile_mesh[blockIdx.y];
  if (active && !active[b]) return;
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int64_t v0 = (int64_t)bt.row_begin[b] + (int64_t)(blockIdx.y - bt.tile_begin[b]) * kTile, V = bt.row_begin[b + 1];
  const int j0 = blockIdx.x * kTile;
  Cm += (int64_t)b * kd * n;
  double acc[4][4] = {};
  for (int k0 = 0; k0 < kd; k0 += kChunk) {
    for (int e = t; e < kTile * kChunk; e += 256) {
      const int r = e / kChunk, c = e % kChunk;
      xs[r][c] = (v0 + r < V && k0 + c < kd) ? X[(v0 + r) * ldx + k0 + c] : 0.0;
      const int r2 = e / kTile, c2 = e % kTile;
      cs[r2][c2] = (k0 + r2 < kd && j0 + c2 < n) ? Cm[(int64_t)(k0 + r2) * n + j0 + c2] : 0.0;
    }
    __syncthreads();
#pragma unroll 4
    for (int kk = 0; kk < kChunk; ++kk) {
      double xa[4], cb[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) xa[a] = xs[ty + 16 * a][kk];
#pragma unroll
      for (int c = 0; c < 4; ++c) cb[c] = cs[kk][tx + 16 * c];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][c] = fma(xa[a], cb[c], acc[a][c]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int64_t v = v0 + ty + 16 * a;
      const int j = j0 + tx + 16 * c;
      if (v < V && j < n) {
        double* z = Z + v * ldz + j;
        *z = beta == 0.0 ? acc[a][c] : fma(beta, *z, acc[a][c]);
      }
    }
}

// eig_resid_partial_kernel on slice blockIdx.y with the mesh's own theta (n per mesh)
__global__ void __launch_bounds__(256) eig_resid_batched_kernel(const double* __restrict__ W, int64_t ldw,
                                                                const double* __restrict__ Q, int64_t ldq,
                                                                const double* __restrict__ theta, dn_eig_batch bt, int n,
                                                                const int32_t* __restrict__ active,
                                                                double* __restrict__ partial) {
  __shared__ double part[8][32];
  const int b = bt.slice_mesh[blockIdx.y];
  if (active && !active[b]) return;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  const int64_t r0 = (int64_t)bt.row_begin[b] + (int64_t)(blockIdx.y - bt.slice_begin[b]) * DN_EIG_SLICE_ROWS;
  const int64_t re = bt.row_begin[b + 1], r1 = r0 + DN_EIG_SLICE_ROWS < re ? r0 + DN_EIG_SLICE_ROWS : re;
  double s = 0.0;
  if (c < n) {
    const double th = theta[(int64_t)b * n + c];
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
    partial[(int64_t)blockIdx.y * n + c] = r;
  }
}

// eig_colsign_kernel for column blockIdx.x of mesh blockIdx.y: cols and sign are (n_meshes, k)
__global__ void __launch_bounds__(256) eig_colsign_batched_kernel(const double* __restrict__ Y, int64_t ldy,
                                                                  const int32_t* __restrict__ cols,
                                                                  const double* __restrict__ mass, dn_eig_batch bt,
                                                                  double* __restrict__ sign) {
  __shared__ double bv[256], bx[256];
  __shared__ int32_t bi[256];
  const int t = threadIdx.x, b = blockIdx.y;
  const int c = cols[b * gridDim.x + blockIdx.x];
  const int32_t r0 = bt.row_begin[b], r1 = bt.row_begin[b + 1];
  double best = -1.0, bval = 0.0;
  int32_t bidx = r1;
  for (int32_t v = r0 + t; v < r1; v += 256) {
    const double x = Y[(int64_t)v * ldy + c] / sqrt(mass[v]);
    if (fabs(x) > best) { best = fabs(x); bidx = v; bval = x; }
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
  if (t == 0) sign[b * gridDim.x + blockIdx.x] = bx[0] < 0.0 ? -1.0 : 1.0;
}

// out[v][i] = sign[b][i] * Y[v][cols[b][i]] / sqrt(mass[v]) for the rows v of tile blockIdx.x, b its mesh
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
    out[v * k + i] = sign[b * k + i] * (Y[v * ldy + cols[b * k + i]] / sqrt(mass[v]));
  }
}

}  // namespace

int64_t eig_gram_ws_bytes(int64_t V, int m, int n) { return 8ll * eig_splits(V) * m * n; }
int64_t eig_resid_ws_bytes(int64_t V, int n) { return 8ll * eig_splits(V) * n; }

int launch_eig_filter(const int32_t* rowptr, const int32_t* colidx, const double* avals, const double* adiag, int64_t V,
                      int n, const double* Y, const double* Yp, int64_t ld, double alpha, double beta, double gamma,
                      double* out, cudaStream_t st) {
  if (V <= 0 || n <= 0) return DN_OK;
  const unsigned blocks = (unsigned)((V * 32 + 255) / 256);
  for (int c0 = 0; c0 < n; c0 += 256) {               // column slices of at most 256 (8 per lane)
    const int w = n - c0 < 256 ? n - c0 : 256;
    const double* y = Y + c0;
    const double* yp = Yp ? Yp + c0 : nullptr;
    double* o = out + c0;
#define DN_FILTER(NC) eig_filter_kernel<NC><<<blocks, 256, 0, st>>>(rowptr, colidx, avals, adiag, V, w, y, yp, ld, alpha, \
                                                                   beta, gamma, o)
    switch ((w + 31) / 32) {
      case 1: DN_FILTER(1); break;
      case 2: DN_FILTER(2); break;
      case 3: DN_FILTER(3); break;
      case 4: DN_FILTER(4); break;
      case 5: DN_FILTER(5); break;
      case 6: DN_FILTER(6); break;
      case 7: DN_FILTER(7); break;
      default: DN_FILTER(8); break;
    }
#undef DN_FILTER
    DN_LAUNCH_CHECK();
  }
  return DN_OK;
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
  for (int c0 = 0; c0 < n; c0 += 256) {
    const int w = n - c0 < 256 ? n - c0 : 256;
    const double* y = Y + c0;
    const double* yp = Yp ? Yp + c0 : nullptr;
    double* o = out + c0;
#define DN_FILTER(NC) eig_filter_batched_kernel<NC><<<blocks, 256, 0, st>>>(rowptr, colidx, avals, adiag, *bt, w, y, yp, ld, \
                                                                           alpha, beta, gamma, active, o)
    switch ((w + 31) / 32) {
      case 1: DN_FILTER(1); break;
      case 2: DN_FILTER(2); break;
      case 3: DN_FILTER(3); break;
      case 4: DN_FILTER(4); break;
      case 5: DN_FILTER(5); break;
      case 6: DN_FILTER(6); break;
      case 7: DN_FILTER(7); break;
      default: DN_FILTER(8); break;
    }
#undef DN_FILTER
    DN_LAUNCH_CHECK();
  }
  return DN_OK;
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
