// Kernels for the two data-side neighbours of the block (SURVEY.md section 8f, items 2 and 3):
//   * heat-kernel-signature input features   (reference geometry.py:600-628, compute_hks)
//   * CSC (the reference's on-disk operator cache, geometry.py:548-568) -> device CSR, i.e. a sparse transpose
// Both are HBM-bound index/streaming work: plain coalesced SIMT, no tensor cores.
#include "dn_internal.h"
#include <type_traits>

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
    for (int s = 0; s < 16; ++s) coef[j][s] = (s < S) ? dn_heat(ev, scales[s < S ? s : 0]) : 0.f;
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
      acc = fmaf(dn_heat(evals[k], t), f * f, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) out[row * S + s] = acc;
  }
}

// ---------------------------------------------------------------------------------------------
// sparse transpose of the shared-pattern CSR (int32 indices, interleaved (x, y) values); the count / scan / row-sort
// kernels also build the mesh Laplacian and the vertex -> face incidence below
// ---------------------------------------------------------------------------------------------
template <typename I>
__global__ void tr_count_kernel(const I* __restrict__ colidx, int64_t nnz, int32_t* __restrict__ cnt) {
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

// Row payloads of the sort below.  Ties (equal column) are ordered by value_less so that rows filled by atomics in
// arbitrary order come out in one deterministic order; the transposes never have ties (their input has unique entries).
struct NoVal {};                      // keys only (vertex -> face incidence)
struct LapVal { double w, a; };       // one directed half of a face corner: cotan weight w and a sixth of the face area
__device__ __forceinline__ bool value_less(const float2&, const float2&) { return false; }
__device__ __forceinline__ bool value_less(const LapVal& x, const LapVal& y) {
  return x.w < y.w || (x.w == y.w && x.a < y.a);
}

// the atomics above land entries of one output row in arbitrary order: sort each row by column (rows are short --
// vertex degree + 1 on meshes, 31 on point clouds -- so one thread per row with an insertion sort)
template <typename T>
__global__ void tr_sort_rows_kernel(const int32_t* __restrict__ rowptr_t, int64_t V, int32_t* __restrict__ colidx_t,
                                    T* __restrict__ vals_t) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= V) return;
  const int s = rowptr_t[row], e = rowptr_t[row + 1];
  for (int i = s + 1; i < e; ++i) {
    const int32_t ck = colidx_t[i];
    T vk{};
    if constexpr (!std::is_same<T, NoVal>::value) vk = vals_t[i];
    auto after = [&](int j) {             // entry j sorts after the one being inserted
      if (colidx_t[j] != ck) return colidx_t[j] > ck;
      if constexpr (std::is_same<T, NoVal>::value) return false;
      else return value_less(vk, vals_t[j]);
    };
    int j = i - 1;
    while (j >= s && after(j)) {
      colidx_t[j + 1] = colidx_t[j];
      if constexpr (!std::is_same<T, NoVal>::value) vals_t[j + 1] = vals_t[j];
      --j;
    }
    colidx_t[j + 1] = ck;
    if constexpr (!std::is_same<T, NoVal>::value) vals_t[j + 1] = vk;
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

// ---------------------------------------------------------------------------------------------
// Mesh Laplacian and lumped mass (reference geometry.py:322-329): the cotan Laplacian with cot = (u.v) / (|u x v| +
// denom_eps) per face corner, L_jk = -1/2 sum cot, L_jj = -sum_k L_jk, and the barycentric vertex areas.  fp64.
// Pattern as scipy's coo -> csc of the reference: the diagonal of every vertex a face references plus both directions
// of every face edge, duplicates summed, explicit zeros kept.  Each corner's weight is computed once and scattered to
// (j, k) and (k, j) together with a sixth of the face area (every vertex of a face receives two such halves); rows are
// sorted by (column, value) so that every sum runs in one fixed order and L is exactly symmetric.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double3 ld3(const double* p, int64_t i) { return make_double3(p[3 * i], p[3 * i + 1], p[3 * i + 2]); }
__device__ __forceinline__ double3 sub3(double3 a, double3 b) { return make_double3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ double dot3(double3 a, double3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ double3 cross3(double3 a, double3 b) {
  return make_double3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
__device__ __forceinline__ double norm3(double3 a) { return sqrt(dot3(a, a)); }

__device__ __forceinline__ bool face_ok(const int64_t* f, int64_t V) {
  return f[0] >= 0 && f[0] < V && f[1] >= 0 && f[1] < V && f[2] >= 0 && f[2] < V;
}

// per face: 2 directed entries per corner whose opposite edge has two distinct ends; marks referenced vertices
__global__ void lap_count_kernel(const int64_t* __restrict__ faces, int64_t F, int64_t V, int32_t* __restrict__ cnt,
                                 int32_t* __restrict__ ref) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F || !face_ok(faces + 3 * f, V)) return;
  const int64_t* t = faces + 3 * f;
  for (int c = 0; c < 3; ++c) {
    const int64_t i = t[c], j = t[(c + 1) % 3], k = t[(c + 2) % 3];
    ref[i] = 1;
    if (j != k) { atomicAdd(cnt + j + 1, 1); atomicAdd(cnt + k + 1, 1); }
  }
}

// A corner whose opposite edge is a single vertex (a face with a repeated index) adds -w, -w, +w, +w to that vertex's
// diagonal in the reference, i.e. nothing, and its face has zero area: it is skipped.
__global__ void lap_fill_kernel(const double* __restrict__ verts, const int64_t* __restrict__ faces, int64_t F, int64_t V,
                                double denom_eps, const int32_t* __restrict__ rawptr, int32_t* __restrict__ cursor,
                                int32_t* __restrict__ rawcol, LapVal* __restrict__ rawval) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F || !face_ok(faces + 3 * f, V)) return;
  const int64_t* t = faces + 3 * f;
  const double3 p0 = ld3(verts, t[0]);
  const double area6 = 0.5 * norm3(cross3(sub3(ld3(verts, t[1]), p0), sub3(ld3(verts, t[2]), p0))) / 6.0;
  for (int c = 0; c < 3; ++c) {
    const int64_t i = t[c], j = t[(c + 1) % 3], k = t[(c + 2) % 3];
    if (j == k) continue;
    const double3 pi = ld3(verts, i), u = sub3(ld3(verts, j), pi), v = sub3(ld3(verts, k), pi);
    const double w = 0.5 * (dot3(u, v) / (norm3(cross3(u, v)) + denom_eps));
    int dst = rawptr[j] + atomicAdd(cursor + j, 1);
    rawcol[dst] = (int32_t)k;
    rawval[dst] = LapVal{w, area6};
    dst = rawptr[k] + atomicAdd(cursor + k, 1);
    rawcol[dst] = (int32_t)j;
    rawval[dst] = LapVal{w, area6};
  }
}

// per row (sorted): number of distinct columns + the diagonal -> cnt[v + 1]; the vertex area (before the eps shift)
__global__ void lap_rows_kernel(const int32_t* __restrict__ rawptr, const int32_t* __restrict__ rawcol,
                                const LapVal* __restrict__ rawval, const int32_t* __restrict__ ref, int64_t V,
                                int32_t* __restrict__ cnt, double* __restrict__ area) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int s = rawptr[v], e = rawptr[v + 1];
  int n = ref[v] ? 1 : 0;
  double a = 0.0;
  for (int p = s; p < e; ++p) {
    if (p == s || rawcol[p] != rawcol[p - 1]) ++n;
    a += rawval[p].a;
  }
  cnt[v + 1] = n;
  area[v] = a;
}

// mass += eps * mean(mass) per mesh, one block each, fixed summation order; block b owns rows [row_begin[b],
// row_begin[b + 1]) (all V rows without row_begin)
__global__ void __launch_bounds__(1024) lap_mass_shift_kernel(double* __restrict__ mass, const int32_t* __restrict__ row_begin,
                                                              int64_t V, double eps) {
  __shared__ double part[1024];
  const int t = threadIdx.x;
  if (row_begin) {
    mass += row_begin[blockIdx.x];
    V = row_begin[blockIdx.x + 1] - row_begin[blockIdx.x];
  }
  double s = 0.0;
  for (int64_t i = t; i < V; i += 1024) s += mass[i];
  part[t] = s;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (t < o) part[t] += part[t + o];
    __syncthreads();
  }
  const double shift = eps * (part[0] / (double)V);
  for (int64_t i = t; i < V; i += 1024) mass[i] += shift;
}

// Merge the sorted raw row into the final CSR row (diagonal at its column position), and the operator the eigensolver
// runs on, A = M^-1/2 (L + eps I) M^-1/2, as A_vals (same pattern: d_v d_k L_vk) + A_diag (eps / m_v).  Row bound of
// Gershgorin's theorem -> max into bound_bits; NaN counts -> nan_out[0] (L rows) and nan_out[1] (mass entries).  With
// row_begin (n_meshes + 1 row offsets of a batch of meshes) the bound and the NaN counts are kept per mesh.
__global__ void lap_emit_kernel(const int32_t* __restrict__ rawptr, const int32_t* __restrict__ rawcol,
                                const LapVal* __restrict__ rawval, const int32_t* __restrict__ ref,
                                const double* __restrict__ mass, int64_t V, double eps, const int32_t* __restrict__ rowptr,
                                int32_t* __restrict__ colidx, double* __restrict__ lvals, double* __restrict__ avals,
                                double* __restrict__ adiag, unsigned long long* __restrict__ bound_bits,
                                int32_t* __restrict__ nan_out, int n_meshes, const int32_t* __restrict__ row_begin) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  if (row_begin) {                      // the vertex's mesh b: bound_bits[b], nan_out[2 b .. 2 b + 1]
    int lo = 0, hi = n_meshes - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (row_begin[mid] <= v) lo = mid; else hi = mid - 1;
    }
    bound_bits += lo;
    nan_out += 2 * lo;
  }
  const int s = rawptr[v], e = rawptr[v + 1];
  const double dv = 1.0 / sqrt(mass[v]);
  double diag = 0.0;
  for (int p = s; p < e; ++p) diag += rawval[p].w;
  int out = rowptr[v];
  bool diag_done = !ref[v], bad = false;
  double rowsum = 0.0;
  const double shift = eps * dv * dv;
  auto emit = [&](int32_t col, double l) {
    colidx[out] = col;
    lvals[out] = l;
    const double a = (dv * (col == v ? dv : 1.0 / sqrt(mass[col]))) * l;   // d_v d_k commutes: A is symmetric too
    if (avals) avals[out] = a;
    rowsum += fabs(col == v ? a + shift : a);
    bad |= isnan(l);
    ++out;
  };
  for (int p = s; p < e;) {
    const int32_t col = rawcol[p];
    double w = 0.0;
    for (; p < e && rawcol[p] == col; ++p) w += rawval[p].w;
    if (!diag_done && col > v) { emit((int32_t)v, diag); diag_done = true; }
    emit(col, -w);
  }
  if (!diag_done) emit((int32_t)v, diag);
  if (!ref[v]) rowsum += fabs(shift);
  if (adiag) adiag[v] = shift;
  if (bad) atomicAdd(nan_out, 1);
  if (isnan(mass[v])) atomicAdd(nan_out + 1, 1);
  if (!isnan(rowsum)) atomicMax(bound_bits, (unsigned long long)__double_as_longlong(rowsum));   // >= 0: bits order as values
}

// ---------------------------------------------------------------------------------------------
// Vertex normals and tangent frames (reference geometry.py:101-177).  Unit face normals (divide-eps 1e-6) summed per
// vertex in face order over the vertex -> face incidence (count / scan / fill / sort), then normalised without eps: a
// vertex no face with a nonzero normal touches gets NaN and is counted (the host applies the reference's remedy).
// Frames: basis candidate e_x unless |n.e_x| >= 0.9 (then e_y), projected to the tangent plane, normalised
// (divide-eps 1e-6), basisY = n x basisX.
// ---------------------------------------------------------------------------------------------
__global__ void vf_fill_kernel(const int64_t* __restrict__ faces, int64_t F, const int32_t* __restrict__ rowptr,
                               int32_t* __restrict__ cursor, int32_t* __restrict__ inc) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= 3 * F) return;
  const int64_t v = faces[s];
  inc[rowptr[v] + atomicAdd(cursor + v, 1)] = (int32_t)(s / 3);
}

__global__ void vf_normals_kernel(const double* __restrict__ verts, const int64_t* __restrict__ faces,
                                  const int32_t* __restrict__ rowptr, const int32_t* __restrict__ inc, int64_t V,
                                  double* __restrict__ normals, int32_t* __restrict__ n_bad) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  double3 n = make_double3(0.0, 0.0, 0.0);
  for (int p = rowptr[v]; p < rowptr[v + 1]; ++p) {
    const int64_t* t = faces + 3 * (int64_t)inc[p];
    const double3 p0 = ld3(verts, t[0]);
    const double3 r = cross3(sub3(ld3(verts, t[1]), p0), sub3(ld3(verts, t[2]), p0));
    const double d = norm3(r) + 1e-6;
    n.x += r.x / d; n.y += r.y / d; n.z += r.z / d;
  }
  const double l = norm3(n);
  n.x /= l; n.y /= l; n.z /= l;
  normals[3 * v] = n.x; normals[3 * v + 1] = n.y; normals[3 * v + 2] = n.z;
  if (isnan(n.x) || isnan(n.y) || isnan(n.z)) atomicAdd(n_bad, 1);
}

__global__ void vf_frames_kernel(const double* __restrict__ normals, int64_t V, double* __restrict__ frames) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const double3 n = ld3(normals, v);
  double3 b = fabs(n.x) < 0.9 ? make_double3(1.0, 0.0, 0.0) : make_double3(0.0, 1.0, 0.0);
  const double d = dot3(b, n);
  b = make_double3(b.x - n.x * d, b.y - n.y * d, b.z - n.z * d);
  const double l = norm3(b) + 1e-6;
  b = make_double3(b.x / l, b.y / l, b.z / l);
  const double3 y = cross3(n, b);
  double* o = frames + 9 * v;
  o[0] = b.x; o[1] = b.y; o[2] = b.z;
  o[3] = y.x; o[4] = y.y; o[5] = y.z;
  o[6] = n.x; o[7] = n.y; o[8] = n.z;
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

namespace {
template <typename T>
T* carve(char*& p, int64_t count) {
  T* r = reinterpret_cast<T*>(p);
  p += (count * (int64_t)sizeof(T) + 255) / 256 * 256;
  return r;
}
}  // namespace

int64_t mesh_laplacian_ws_bytes(int64_t F, int64_t V) { return 120 * F + 12 * V + 2048; }
int64_t vertex_frames_ws_bytes(int64_t F, int64_t V) { return 12 * F + 8 * V + 1024; }

// row_begin == nullptr: one mesh.  Otherwise the union of n_meshes meshes (faces index the union's rows): every kernel but
// the mass shift and the emit is per face or per row and runs on the union unchanged.
static int mesh_laplacian_impl(const double* verts, const int64_t* faces, int64_t F, int64_t V, int n_meshes,
                               const int32_t* row_begin, double eps, int32_t* rowptr, int32_t* colidx, double* lvals,
                               double* mass, double* avals, double* adiag, double* bound, int32_t* nan_out, void* ws,
                               cudaStream_t st) {
  DN_CUDA_TRY(cudaMemsetAsync(rowptr, 0, sizeof(int32_t) * (V + 1), st));
  DN_CUDA_TRY(cudaMemsetAsync(bound, 0, sizeof(double) * n_meshes, st));
  DN_CUDA_TRY(cudaMemsetAsync(nan_out, 0, 2 * sizeof(int32_t) * n_meshes, st));
  if (V <= 0) return DN_OK;
  char* p = static_cast<char*>(ws);
  int32_t* rawcol = carve<int32_t>(p, 6 * F);
  LapVal* rawval = carve<LapVal>(p, 6 * F);
  int32_t* rawptr = carve<int32_t>(p, V + 1);
  int32_t* cursor = carve<int32_t>(p, V);
  int32_t* ref = carve<int32_t>(p, V);
  DN_CUDA_TRY(cudaMemsetAsync(rawptr, 0, sizeof(int32_t) * (V + 1), st));
  DN_CUDA_TRY(cudaMemsetAsync(cursor, 0, sizeof(int32_t) * V, st));
  DN_CUDA_TRY(cudaMemsetAsync(ref, 0, sizeof(int32_t) * V, st));
  const unsigned vb = (unsigned)((V + 255) / 256), fb = (unsigned)((F + 255) / 256);
  if (F > 0) {
    lap_count_kernel<<<fb, 256, 0, st>>>(faces, F, V, rawptr, ref);
    DN_LAUNCH_CHECK();
  }
  tr_scan_kernel<<<1, 1024, 0, st>>>(rawptr, V + 1);
  DN_LAUNCH_CHECK();
  if (F > 0) {
    lap_fill_kernel<<<fb, 256, 0, st>>>(verts, faces, F, V, 1e-10, rawptr, cursor, rawcol, rawval);
    DN_LAUNCH_CHECK();
  }
  tr_sort_rows_kernel<<<vb, 256, 0, st>>>(rawptr, V, rawcol, rawval);
  DN_LAUNCH_CHECK();
  lap_rows_kernel<<<vb, 256, 0, st>>>(rawptr, rawcol, rawval, ref, V, rowptr, mass);
  DN_LAUNCH_CHECK();
  tr_scan_kernel<<<1, 1024, 0, st>>>(rowptr, V + 1);
  DN_LAUNCH_CHECK();
  lap_mass_shift_kernel<<<(unsigned)n_meshes, 1024, 0, st>>>(mass, row_begin, V, eps);
  DN_LAUNCH_CHECK();
  lap_emit_kernel<<<vb, 256, 0, st>>>(rawptr, rawcol, rawval, ref, mass, V, eps, rowptr, colidx, lvals, avals, adiag,
                                      reinterpret_cast<unsigned long long*>(bound), nan_out, n_meshes, row_begin);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_mesh_laplacian(const double* verts, const int64_t* faces, int64_t F, int64_t V, double eps, int32_t* rowptr,
                          int32_t* colidx, double* lvals, double* mass, double* avals, double* adiag, double* bound,
                          int32_t* nan_out, void* ws, cudaStream_t st) {
  return mesh_laplacian_impl(verts, faces, F, V, 1, nullptr, eps, rowptr, colidx, lvals, mass, avals, adiag, bound, nan_out,
                             ws, st);
}

int launch_mesh_laplacian_batched(const double* verts, const int64_t* faces, int64_t F, int64_t V, int n_meshes,
                                  const int32_t* row_begin, double eps, int32_t* rowptr, int32_t* colidx, double* lvals,
                                  double* mass, double* avals, double* adiag, double* bound, int32_t* nan_out, void* ws,
                                  cudaStream_t st) {
  if (n_meshes <= 0) return DN_OK;
  return mesh_laplacian_impl(verts, faces, F, V, n_meshes, row_begin, eps, rowptr, colidx, lvals, mass, avals, adiag, bound,
                             nan_out, ws, st);
}

int launch_vertex_frames(const double* verts, const int64_t* faces, int64_t F, int64_t V, const double* normals_in,
                         double* normals_out, double* frames, int32_t* n_bad, void* ws, cudaStream_t st) {
  DN_CUDA_TRY(cudaMemsetAsync(n_bad, 0, sizeof(int32_t), st));
  if (V <= 0) return DN_OK;
  const unsigned vb = (unsigned)((V + 255) / 256);
  if (!normals_in) {
    char* p = static_cast<char*>(ws);
    int32_t* rowptr = carve<int32_t>(p, V + 1);
    int32_t* cursor = carve<int32_t>(p, V);
    int32_t* inc = carve<int32_t>(p, 3 * F);
    DN_CUDA_TRY(cudaMemsetAsync(rowptr, 0, sizeof(int32_t) * (V + 1), st));
    DN_CUDA_TRY(cudaMemsetAsync(cursor, 0, sizeof(int32_t) * V, st));
    if (F > 0) {
      tr_count_kernel<<<(unsigned)((3 * F + 255) / 256), 256, 0, st>>>(faces, 3 * F, rowptr);
      DN_LAUNCH_CHECK();
    }
    tr_scan_kernel<<<1, 1024, 0, st>>>(rowptr, V + 1);
    DN_LAUNCH_CHECK();
    if (F > 0) {
      vf_fill_kernel<<<(unsigned)((3 * F + 255) / 256), 256, 0, st>>>(faces, F, rowptr, cursor, inc);
      DN_LAUNCH_CHECK();
    }
    tr_sort_rows_kernel<<<vb, 256, 0, st>>>(rowptr, V, inc, static_cast<NoVal*>(nullptr));
    DN_LAUNCH_CHECK();
    vf_normals_kernel<<<vb, 256, 0, st>>>(verts, faces, rowptr, inc, V, normals_out, n_bad);
    DN_LAUNCH_CHECK();
    normals_in = normals_out;
  }
  vf_frames_kernel<<<vb, 256, 0, st>>>(normals_in, V, frames);
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
