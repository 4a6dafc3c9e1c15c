// Fused classification head: z = X W^T + b, log_softmax and the NLL loss per row (optionally with a label-smoothed
// target), forward and backward, on wgmma.  The (R x n_class) logits, probabilities and logit gradients live only in
// registers and shared memory.  Also the rows the head runs on for face / edge outputs (element mean) and for
// whole-shape outputs (mass-weighted mean per mesh).
//
// Every kernel runs 256 threads: two warpgroups of 64 rows each own the 128 rows of a CTA tile (rows of X, or classes
// of W in the weight-gradient kernel).  A 128-wide tile of the other operand streams through a B image in shared memory
// in 32-deep K stages, in the K-major layout of the chain kernels (kmajor_off, dn_tc_ptx.cuh) with N = 128; 3xTF32 keeps
// a hi image and a lo image.
#include <math.h>
#include "dn_internal.h"
#include "dn_tc_ptx.cuh"

using namespace tc;

namespace {

constexpr int HT = 128;                   // CTA rows, class-tile width and MMA N
constexpr int KS = 32;                    // K per B stage
constexpr int NTHR = 256;
constexpr uint32_t LBO = HT * 16;
constexpr int B_IMG = KS * HT * 4;        // one tf32 image of a stage

__host__ __device__ constexpr int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

// element (k, n) of a stage's B image
template <int MODE>
__device__ __forceinline__ void b_put(uint8_t* img, int k, int n, float v) {
  const uint32_t off = kmajor_off<MODE>(k, n, HT);
  if constexpr (MODE == MODE_BF16) {
    *reinterpret_cast<uint16_t*>(img + off) = (uint16_t)(pack_bf16x2(v, 0.f) & 0xFFFFu);
  } else {
    float hi, lo;
    split_tf32(v, hi, lo);
    *reinterpret_cast<float*>(img + off) = hi;
    if (MODE == MODE_TF32X3) *reinterpret_cast<float*>(img + B_IMG + off) = lo;
  }
}

// Every B stage reaches shared memory by TMA as a raw fp32 box with the 128-byte swizzle, through a two-slot ring
// (one mbarrier per slot, stage q + 2 in flight while stage q is consumed); all threads then convert it into the MMA
// image.  The swizzle makes both sides of the conversion free of bank conflicts: a warp writes 128 consecutive bytes of
// the image and reads 8 rows x 4 floats of the raw box whose 16-byte chunks the swizzle spreads over all banks.
constexpr int RAW_BYTES = KS * HT * 4;    // one raw stage (16 KB)

// raw (row, col) of a box with 128-byte rows (32 floats) and the 128-byte swizzle
__device__ __forceinline__ float raw_at(const uint8_t* raw, int row, int col) {
  return *reinterpret_cast<const float*>(raw + row * 128 + ((((col >> 2) ^ row) & 7) << 4) + (col & 3) * 4);
}

// image coordinates of the w-th word a thread converts: consecutive w are consecutive image words (TF32 layout)
__device__ __forceinline__ void img_coords(int w, int& kl, int& n) {
  kl = (w >> 9) * 4 + (w & 3);
  n = ((w >> 5) & 15) * 8 + ((w >> 2) & 7);
}

// rows stage: B(k, n) = src row n, column k: one {32, 128} box (TMA zero-fills rows and columns outside the source)
template <int MODE>
__device__ void convert_rows(uint8_t* img, const uint8_t* raw) {
  for (int w = threadIdx.x; w < KS * HT; w += NTHR) {
    int k, n;
    img_coords(w, k, n);
    b_put<MODE>(img, k, n, raw_at(raw, n, k));
  }
}

// columns stage: B(k, n) = src row k, column n, from four {32, 32} boxes (box j holds n in [32 j, 32 j + 32)); zero
// outside k < nk, n < nn (boxes wholly outside the source are not loaded).  For the TF32 engines the K order inside every
// 8-group is permuted to match A fragments taken from an accumulator (tf32_k_slot, mma_dz).
template <int MODE>
__device__ void convert_cols(uint8_t* img, const uint8_t* raw, int nk, int nn) {
  for (int w = threadIdx.x; w < KS * HT; w += NTHR) {
    int kl, n;
    img_coords(w, kl, n);
    const int k = MODE == MODE_BF16 ? kl : tf32_slot_k(kl);
    const float v = (k < nk && n < nn) ? raw_at(raw + (n >> 5) * (RAW_BYTES / 4), k, n & 31) : 0.f;
    b_put<MODE>(img, kl, n, v);
  }
}

// The stage sequence of a CTA: `ntiles` tiles, tile t = nst rows stages of map a (rows a0 + 128 t, columns KS i) then
// ncol columns stages of map b (rows b0 + 128 t + KS j, columns c0 .. c0 + 127).
struct Seq {
  int64_t a0, b0, ntiles;
  int nst, ncol, c0;
  int64_t b_rows;    // rows of map b's source
  int b_cols;        // columns of map b's source
};

struct Ring {
  uint8_t* raw;      // 2 slots of RAW_BYTES, 1024-byte aligned
  uint32_t bar;      // 2 mbarriers
  int64_t q;         // next stage to consume
};

__device__ __forceinline__ void ring_issue(const Ring& rg, const Seq& sq, const CUtensorMap* amap, const CUtensorMap* bmap,
                                           int64_t q) {
  const int per = sq.nst + sq.ncol;
  const int64_t t = q / per;
  if (t >= sq.ntiles) return;
  const int i = (int)(q % per);
  const uint32_t bar = rg.bar + 8 * (uint32_t)(q & 1), dst = smem_u32(rg.raw + (q & 1) * RAW_BYTES);
  if (i < sq.nst) {
    mbar_arrive_expect_tx(bar, RAW_BYTES);
    tma_tile_2d_g2s(dst, amap, KS * i, (int)(sq.a0 + HT * t), bar);
    return;
  }
  const int64_t row = sq.b0 + HT * t + KS * (i - sq.nst);
  int nbox = 0;
  for (int j = 0; j < 4; ++j) nbox += (row < sq.b_rows && sq.c0 + 32 * j < sq.b_cols) ? 1 : 0;
  if (nbox == 0) { mbar_arrive(bar); return; }
  mbar_arrive_expect_tx(bar, nbox * (RAW_BYTES / 4));
  for (int j = 0; j < 4; ++j)
    if (row < sq.b_rows && sq.c0 + 32 * j < sq.b_cols)
      tma_tile_2d_g2s(dst + j * (RAW_BYTES / 4), bmap, sq.c0 + 32 * j, (int)row, bar);
}

// one stage: wait for its box, convert it into the image once every warpgroup's MMAs on the image are done, then hand
// the raw slot to stage q + 2
template <typename Convert>
__device__ __forceinline__ void ring_next(Ring& rg, const Seq& sq, const CUtensorMap* amap, const CUtensorMap* bmap,
                                          uint8_t* img, Convert convert) {
  mbar_wait(rg.bar + 8 * (uint32_t)(rg.q & 1), (uint32_t)((rg.q >> 1) & 1));
  __syncthreads();
  convert(img, rg.raw + (rg.q & 1) * RAW_BYTES);
  fence_proxy_async();
  __syncthreads();
  if (threadIdx.x == 0) ring_issue(rg, sq, amap, bmap, rg.q + 2);
  ++rg.q;
}

// acc (+)= A * B image over the first `steps` K slices of a stage (k8 TF32, k16 bf16); frag(s, ah, al) forms the A
// fragment of slice s.  Every fragment is formed before wgmma_fence.
template <int MODE, typename Frag>
__device__ __forceinline__ void mma_stage(float* acc, uint32_t sb, bool first, int steps, Frag frag) {
  constexpr int STEPS = MODE == MODE_BF16 ? KS / 16 : KS / 8;
  uint32_t ah[STEPS][4], al[STEPS][4];
#pragma unroll
  for (int s = 0; s < STEPS; ++s) frag(s, ah[s], al[s]);
#pragma unroll
  for (int s = 0; s < STEPS; ++s) {
    fence_frag4(ah[s]);
    if (MODE == MODE_TF32X3) fence_frag4(al[s]);
  }
  wgmma_fence();
#pragma unroll
  for (int s = 0; s < STEPS; ++s) {
    if (s >= steps) break;
    mma_step<MODE, HT>(acc, ah[s], al[s], sb + s * 2 * LBO, B_IMG, LBO, (!first || s > 0) ? 1u : 0u);
  }
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int j = 0; j < 8; ++j) fence_acc8(acc + 8 * j);
}

// rows [r0, r0 + nr) of src (R x C, row stride C) into the shared tile As (128 x (C + 4)), zero rows past nr
__device__ void load_tile(float* As, const float* __restrict__ src, int64_t r0, int nr, int C) {
  const int lda = C + 4, q = C / 4;
  for (int i = threadIdx.x; i < HT * q; i += NTHR) {
    const int r = i / q, c = 4 * (i % q);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < nr) v = __ldg(reinterpret_cast<const float4*>(src + (r0 + r) * C + c));
    *reinterpret_cast<float4*>(As + r * lda + c) = v;
  }
}

// acc = As (this warp's rows) x src[n0 .. n0 + nn)^T over the full C: the 128-wide logit tile, bias not added
template <int MODE>
__device__ __forceinline__ void logit_tile(float* acc, const float* As, int C, int r, Ring& rg, const Seq& sq,
                                           const CUtensorMap* amap, const CUtensorMap* bmap, uint8_t* img) {
  const uint32_t sb = smem_u32(img);
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, lda = C + 4;
  for (int k0 = 0; k0 < C; k0 += KS) {
    const int nk = C - k0 < KS ? C - k0 : KS;
    ring_next(rg, sq, amap, bmap, img, [](uint8_t* im, const uint8_t* raw) { convert_rows<MODE>(im, raw); });
    // A = rows r + g, r + g + 8 of the shared tile, columns k0 ..
    const float* a0 = As + (r + g) * lda + k0;
    const float* a1 = a0 + 8 * lda;
    mma_stage<MODE>(acc, sb, k0 == 0, MODE == MODE_BF16 ? nk / 16 : nk / 8, [&](int s, uint32_t* ah, uint32_t* al) {
      if constexpr (MODE == MODE_BF16) {
        const int c = 16 * s + 2 * t;
        const float x[8] = {a0[c], a0[c + 1], a1[c], a1[c + 1], a0[c + 8], a0[c + 9], a1[c + 8], a1[c + 9]};
        frag_bf16(x, ah);
      } else {
        const int c = 8 * s + t;
        const float x[4] = {a0[c], a1[c], a0[c + 4], a1[c + 4]};
        frag_tf32(x, ah, al);
      }
    });
  }
}

// acc (+)= Z[:, 32 ch, 32 ch + 32) * B_ch for ch = CH .. 3: Z is this warpgroup's 64 x 128 accumulator z as the A operand
// (columns of z = K), B_ch the next columns stage (source rows k0 + 32 ch .. of `extent` rows, columns c0 .. c0 + nc).
// `first`: chunk 0 starts the sum.
template <int MODE, int CH = 0>
__device__ __forceinline__ void mma_dz(float* acc, const float* z, int64_t k0, int64_t extent, int nc, bool first,
                                       Ring& rg, const Seq& sq, const CUtensorMap* amap, const CUtensorMap* bmap,
                                       uint8_t* img) {
  const int64_t rem = extent - (k0 + KS * CH);
  const int nk = (int)(rem < KS ? rem : KS);   // <= 0: no row of the stage is in the source
  ring_next(rg, sq, amap, bmap, img, [=](uint8_t* im, const uint8_t* raw) { convert_cols<MODE>(im, raw, nk, nc); });
  constexpr int STEPS = MODE == MODE_BF16 ? KS / 16 : KS / 8;
  mma_stage<MODE>(acc, smem_u32(img), first && CH == 0, STEPS, [&](int s, uint32_t* ah, uint32_t* al) {
    if constexpr (MODE == MODE_BF16) {
      frag_bf16(z + 4 * (4 * CH + 2 * s), ah);
    } else {
      const float* zb = z + 4 * (4 * CH + s);
      const float x[4] = {zb[0], zb[2], zb[1], zb[3]};
      frag_tf32(x, ah, al);
    }
  });
  if constexpr (CH + 1 < HT / KS) mma_dz<MODE, CH + 1>(acc, z, k0, extent, nc, first, rg, sq, amap, bmap, img);
}

// shared memory: the raw ring (1024-byte aligned for the swizzle), the A tile, the B image, per-row factors, mbarriers
struct HeadSmem {
  Ring rg;
  float* As;
  uint8_t* img;
  float* rows;
};

__device__ __forceinline__ HeadSmem head_smem_carve(uint8_t* smem, int C, const Seq& sq, const CUtensorMap* amap,
                                                    const CUtensorMap* bmap) {
  HeadSmem h;
  uint8_t* base = smem + ((1024 - (smem_u32(smem) & 1023)) & 1023);
  h.rg.raw = base;
  h.As = reinterpret_cast<float*>(base + 2 * RAW_BYTES);
  h.img = base + 2 * RAW_BYTES + (size_t)HT * (C + 4) * 4;
  h.rows = reinterpret_cast<float*>(h.img + 2 * B_IMG);
  h.rg.bar = smem_u32(h.rows + 3 * HT);
  h.rg.q = 0;
  if (threadIdx.x == 0) {
    mbar_init(h.rg.bar, 1);
    mbar_init(h.rg.bar + 8, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    ring_issue(h.rg, sq, amap, bmap, 0);
    ring_issue(h.rg, sq, amap, bmap, 1);
  }
  return h;
}

// per-row factor of the logit gradient: dZ = coef * (softmax - onehot); 0 for padding and ignored rows, NaN for a label
// outside [0, n_class)
__device__ __forceinline__ float row_coef(int64_t lab, float g, int n_class, int64_t ignore_index, bool valid) {
  if (!valid || lab == ignore_index) return 0.f;
  if (lab < 0 || lab >= n_class) return __int_as_float(0x7fc00000);
  return g;
}

struct HeadArgs {
  const float* X;
  const float* W;
  const float* b;
  const int64_t* labels;
  const float* lse;       // bwd: saved by the forward
  const float* g;         // bwd: upstream per-row weight
  int64_t R;
  int C, n_class;
  int64_t ignore_index;
  float* nll;             // fwd
  int64_t* argmax;        // fwd
  float* lse_out;         // fwd
  float* dX;              // bwd
  float* dWp;             // bwd: [S][n_class][C] partials
  float* dbp;             // bwd: [S][n_class]
  int S;                  // row splits of the weight-gradient kernel
  // label smoothing (set_smoothing): the target is ls_on for the label and ls_off = s / (n_class - 1) for every other
  // class; ls_label = ls_on - ls_off.  Without smoothing ls_on = 1 and ls_off = 0 exactly, so the logit gradient
  // g (softmax - target) is the one-hot expression bit for bit.
  int smooth;
  float ls_on, ls_off, ls_label;
  CUtensorMap amap;       // logits' B source (W: forward and dX; X: dW), {32, 128} boxes
  CUtensorMap bmap;       // dX / dW's B source (W / X), {32, 32} boxes
};

// at most 128 registers: two CTAs share an SM wherever their shared memory fits (C up to about 96)
template <int MODE>
__global__ void __launch_bounds__(NTHR, 2) linear_nll_fwd_kernel(const __grid_constant__ HeadArgs p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const Seq sq{0, 0, cdiv(p.n_class, HT), (int)cdiv(p.C, KS), 0, 0, 0, 0};
  HeadSmem hs = head_smem_carve(smem, p.C, sq, &p.amap, &p.bmap);
  float* As = hs.As;
  uint8_t* img = hs.img;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, t = lane & 3;
  const int r = (warp >> 2) * 64 + (warp & 3) * 16;        // rows r + g, r + g + 8 of the tile
  const int64_t row0 = (int64_t)blockIdx.x * HT;
  const int nr = p.R - row0 < HT ? (int)(p.R - row0) : HT;
  load_tile(As, p.X, row0, nr, p.C);
  const int64_t rows[2] = {row0 + r + (lane >> 2), row0 + r + (lane >> 2) + 8};
  int64_t lab[2];
  float m[2], s[2], zl[2], best[2], dm[2];
  int bi[2];
  bool bad[2];
  float cnt = 0.f;     // smoothing: this thread's valid columns so far
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    lab[h] = rows[h] < p.R ? p.labels[rows[h]] : p.ignore_index;
    m[h] = -INFINITY; s[h] = 0.f; zl[h] = 0.f; best[h] = -INFINITY; bi[h] = 0; bad[h] = false; dm[h] = 0.f;
  }
  float acc[64];
  for (int64_t n0 = 0; n0 < p.n_class; n0 += HT) {
    const int nn = p.n_class - n0 < HT ? (int)(p.n_class - n0) : HT;
    logit_tile<MODE>(acc, As, p.C, r, hs.rg, sq, &p.amap, &p.bmap, img);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      // online log-sum-exp over the valid columns (padding columns are skipped, not set to -inf)
      float tmax = -INFINITY;
#pragma unroll
      for (int b = 0; b < 16; ++b)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * b + 2 * t + e;
          if (c < nn) {
            const float z = acc[4 * b + 2 * h + e] + (p.b ? __ldg(p.b + n0 + c) : 0.f);
            acc[4 * b + 2 * h + e] = z;
            if (!isfinite(z)) bad[h] = true;
            tmax = fmaxf(tmax, z);
            if (z > best[h]) { best[h] = z; bi[h] = (int)(n0 + c); }
            if (n0 + c == lab[h]) zl[h] = z;
          }
        }
      tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 1));
      tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 2));
      const float mn = fmaxf(m[h], tmax);
      float sum = s[h] * expf(m[h] - mn);
      // smoothing: the running sum_j (m - z_j) over this thread's columns, moved to the new max; every term is >= 0,
      // so the smoothed loss needs no difference of large sums
      if (p.smooth && cnt > 0.f) dm[h] += cnt * (mn - m[h]);
#pragma unroll
      for (int b = 0; b < 16; ++b)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (8 * b + 2 * t + e < nn) {
            sum += expf(acc[4 * b + 2 * h + e] - mn);
            if (p.smooth) dm[h] += mn - acc[4 * b + 2 * h + e];
          }
      m[h] = mn;
      s[h] = sum;
    }
    // this thread's columns of the tile are 8 b + 2 t + e < nn
    if (p.smooth) cnt += (float)(cdiv(max(nn - 2 * t, 0), 8) + cdiv(max(nn - 2 * t - 1, 0), 8));
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      s[h] += __shfl_xor_sync(0xffffffffu, s[h], o);
      zl[h] += __shfl_xor_sync(0xffffffffu, zl[h], o);
      bad[h] = __shfl_xor_sync(0xffffffffu, (int)bad[h], o) != 0;
      if (p.smooth) dm[h] += __shfl_xor_sync(0xffffffffu, dm[h], o);
      const float ob = __shfl_xor_sync(0xffffffffu, best[h], o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi[h], o);
      if (ob > best[h] || (ob == best[h] && oi < bi[h])) { best[h] = ob; bi[h] = oi; }
    }
    if (t == 0 && rows[h] < p.R) {
      const float nan = __int_as_float(0x7fc00000);
      const float lse = bad[h] ? nan : m[h] + logf(s[h]);
      float nll = lse - zl[h];
      // smoothed: sum_j t_j (lse - z_j) = ls_label (lse - z_label) + ls_off sum_j (lse - z_j), and
      // sum_j (lse - z_j) = sum_j (m - z_j) + n_class log(sum-exp)
      if (p.smooth) nll = p.ls_label * nll + p.ls_off * (dm[h] + (float)p.n_class * logf(s[h]));
      if (lab[h] == p.ignore_index) nll = 0.f;
      else if (lab[h] < 0 || lab[h] >= p.n_class) nll = nan;
      p.nll[rows[h]] = nll;
      p.lse_out[rows[h]] = lse;
      p.argmax[rows[h]] = bi[h];
    }
  }
}

// dX[:, c0 .. c0 + 128) = sum over class tiles of dZ_tile W_tile[:, c0 ..]; grid (row tiles, column halves)
template <int MODE>
__global__ void __launch_bounds__(NTHR, 1) linear_nll_dx_kernel(const __grid_constant__ HeadArgs p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int c0 = blockIdx.y * HT, nc = p.C - c0 < HT ? p.C - c0 : HT;
  const Seq sq{0, 0, cdiv(p.n_class, HT), (int)cdiv(p.C, KS), HT / KS, c0, p.n_class, p.C};
  HeadSmem hs = head_smem_carve(smem, p.C, sq, &p.amap, &p.bmap);
  float* As = hs.As;
  uint8_t* img = hs.img;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, t = lane & 3;
  const int r = (warp >> 2) * 64 + (warp & 3) * 16;
  const int64_t row0 = (int64_t)blockIdx.x * HT;
  const int nr = p.R - row0 < HT ? (int)(p.R - row0) : HT;
  load_tile(As, p.X, row0, nr, p.C);
  const int64_t rows[2] = {row0 + r + (lane >> 2), row0 + r + (lane >> 2) + 8};
  int64_t lab[2];
  float coef[2], lse[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const bool v = rows[h] < p.R;
    lab[h] = v ? p.labels[rows[h]] : p.ignore_index;
    coef[h] = row_coef(lab[h], v ? p.g[rows[h]] : 0.f, p.n_class, p.ignore_index, v);
    lse[h] = v ? p.lse[rows[h]] : 0.f;
  }
  float z[64], acc[64];
  for (int64_t n0 = 0; n0 < p.n_class; n0 += HT) {
    const int nn = p.n_class - n0 < HT ? (int)(p.n_class - n0) : HT;
    logit_tile<MODE>(z, As, p.C, r, hs.rg, sq, &p.amap, &p.bmap, img);
#pragma unroll
    for (int b = 0; b < 16; ++b)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int c = 8 * b + 2 * t + (e & 1), h = e >> 1;
        float d = 0.f;
        if (c < nn && coef[h] != 0.f) {
          const float zz = z[4 * b + e] + (p.b ? __ldg(p.b + n0 + c) : 0.f);
          d = coef[h] * (expf(zz - lse[h]) - (n0 + c == lab[h] ? p.ls_on : p.ls_off));
        }
        z[4 * b + e] = d;
      }
    mma_dz<MODE>(acc, z, n0, p.n_class, nc, n0 == 0, hs.rg, sq, &p.amap, &p.bmap, img);
  }
#pragma unroll
  for (int b = 0; b < 16; ++b)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = 8 * b + 2 * t + (e & 1), h = e >> 1;
      if (c < nc && rows[h] < p.R) p.dX[rows[h] * p.C + c0 + c] = acc[4 * b + e];
    }
}

// Weight and bias gradient partials: CTA (class tile, column half, row split s) sums dZ^T X over the row tiles of split
// s, recomputing the transposed logit tile W_tile X_rows^T.  dbp is written by the column-half-0 CTAs.
template <int MODE>
__global__ void __launch_bounds__(NTHR, 1) linear_nll_dw_kernel(const __grid_constant__ HeadArgs p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, t = lane & 3;
  const int r = (warp >> 2) * 64 + (warp & 3) * 16;
  const int64_t n0 = (int64_t)blockIdx.x * HT;
  const int nn = p.n_class - n0 < HT ? (int)(p.n_class - n0) : HT;
  const int c0 = blockIdx.y * HT, nc = p.C - c0 < HT ? p.C - c0 : HT;
  const int split = blockIdx.z;
  const int64_t RT = cdiv(p.R, HT);
  const int64_t t_begin = RT * split / p.S, t_end = RT * (split + 1) / p.S;
  const Seq sq{HT * t_begin, HT * t_begin, t_end - t_begin, (int)cdiv(p.C, KS), HT / KS, c0, p.R, p.C};
  HeadSmem hs = head_smem_carve(smem, p.C, sq, &p.amap, &p.bmap);
  float* As = hs.As;
  uint8_t* img = hs.img;
  float* rcoef = hs.rows;
  float* rlse = rcoef + HT;
  int* rlab = reinterpret_cast<int*>(rlse + HT);
  load_tile(As, p.W, n0, nn, p.C);
  const int cls[2] = {r + (lane >> 2), r + (lane >> 2) + 8};
  float bias[2], dbs[2] = {0.f, 0.f};
#pragma unroll
  for (int h = 0; h < 2; ++h) bias[h] = (p.b && cls[h] < nn) ? p.b[n0 + cls[h]] : 0.f;
  float z[64], acc[64];
  for (int64_t rt = t_begin; rt < t_end; ++rt) {
    const int64_t row0 = rt * HT;
    const int nr = p.R - row0 < HT ? (int)(p.R - row0) : HT;
    // the tile's per-row factors go to shared memory (read after logit_tile's barriers); kept in registers for all 32
    // columns of a thread they would spill
    if (threadIdx.x < HT) {
      const int c = threadIdx.x;
      const bool v = c < nr;
      const int64_t lab = v ? __ldg(p.labels + row0 + c) : p.ignore_index;
      rcoef[c] = row_coef(lab, v ? __ldg(p.g + row0 + c) : 0.f, p.n_class, p.ignore_index, v);
      rlse[c] = v ? __ldg(p.lse + row0 + c) : 0.f;
      rlab[c] = (lab >= n0 && lab < n0 + nn) ? (int)(lab - n0) : -1;
    }
    logit_tile<MODE>(z, As, p.C, r, hs.rg, sq, &p.amap, &p.bmap, img);
#pragma unroll
    for (int b = 0; b < 16; ++b)
#pragma unroll
      for (int e2 = 0; e2 < 2; ++e2) {
        const int c = 8 * b + 2 * t + e2;
        const float coef = rcoef[c], lse = rlse[c];
        const int lab = rlab[c];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float d = 0.f;
          if (cls[h] < nn && coef != 0.f)
            d = coef * (expf(z[4 * b + 2 * h + e2] + bias[h] - lse) - (cls[h] == lab ? p.ls_on : p.ls_off));
          z[4 * b + 2 * h + e2] = d;
          dbs[h] += d;
        }
      }
    mma_dz<MODE>(acc, z, row0, p.R, nc, rt == t_begin, hs.rg, sq, &p.amap, &p.bmap, img);
  }
  float* dw = p.dWp + (int64_t)split * p.n_class * p.C;
#pragma unroll
  for (int b = 0; b < 16; ++b)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = 8 * b + 2 * t + (e & 1), h = e >> 1;
      if (c < nc && cls[h] < nn) dw[(n0 + cls[h]) * p.C + c0 + c] = acc[4 * b + e];
    }
  if (blockIdx.y == 0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      dbs[h] += __shfl_xor_sync(0xffffffffu, dbs[h], 1);
      dbs[h] += __shfl_xor_sync(0xffffffffu, dbs[h], 2);
      if (t == 0 && cls[h] < nn) p.dbp[(int64_t)split * p.n_class + n0 + cls[h]] = dbs[h];
    }
  }
}

// dW = sum_s dWp[s], db = sum_s dbp[s], in split order (OVERWRITTEN)
__global__ void linear_nll_reduce_kernel(const float* __restrict__ dWp, const float* __restrict__ dbp, int S,
                                         int64_t nw, int64_t nb, float* dW, float* db) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nw + nb; i += (int64_t)gridDim.x * blockDim.x) {
    const bool w = i < nw;
    const float* src = w ? dWp + i : dbp + (i - nw);
    const int64_t stride = w ? nw : nb;
    float s = 0.f;
    for (int k = 0; k < S; ++k) s += src[k * stride];
    if (w) dW[i] = s;
    else if (db) db[i - nw] = s;
  }
}

// out[e][c] = (sum_j x[elems[e][j]][c]) / k, corners summed in order j = 0 .. k-1
__global__ void element_mean_fwd_kernel(const float* __restrict__ x, int C, const int64_t* __restrict__ elems, int64_t E,
                                        int k, float* out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < E * C; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e = i / C;
    const int c = (int)(i % C);
    float s = 0.f;
    for (int j = 0; j < k; ++j) s += __ldg(x + __ldg(elems + e * k + j) * C + c);
    out[i] = s / (float)k;
  }
}

// grad_x[v][c] = sum over the CSR entries of v (element ids, in list order) of grad_out[e][c] / k
__global__ void element_mean_bwd_kernel(const float* __restrict__ g, int C, const int32_t* __restrict__ rowptr,
                                        const int32_t* __restrict__ ent, int64_t V, int k, float* gx) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < V * C; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = i / C;
    const int c = (int)(i % C);
    float s = 0.f;
    for (int j = rowptr[v]; j < rowptr[v + 1]; ++j) s += __ldg(g + (int64_t)ent[j] * C + c) / (float)k;
    gx[i] = s;
  }
}

// ---- mass-weighted mean over segments of rows (outputs_at = 'global_mean') ----
// Segment b is rows [begin[b], begin[b] + rows[b]); it begins on a 128-row tile, and tile_seg[t] names the segment of
// tile t (-1: none).  Rows outside every segment are never read.  The partial pass gives every CTA POOL_TILES
// consecutive tiles; a run of them in one segment is summed into the slots of the run's last tile t:
// wx[t][c] = sum mass[v] x[v][c], wm[t] = sum mass[v].  The reduction pass sums a segment's runs in tile order.
constexpr int POOL_TILES = 2;     // small runs: a single 200k-row mesh gives ~6 CTAs per SM, evenly spread
constexpr int POOL_THR = 256;
constexpr int POOL_RTHR = 1024;   // reduction CTA: up to 1024 / (C / 4) slices of a segment's runs

__device__ __forceinline__ int pool_seg(const int32_t* __restrict__ tile_seg, int n_seg, int64_t t) {
  const int s = __ldg(tile_seg + t);
  return s < n_seg ? s : -1;
}

// thread layout over C / 4 float4 columns: lane j of row group r (rows r, r + rg, ..); threads past q * rg idle
struct PoolLanes {
  int q, rg, j, r;
  __device__ PoolLanes(int C, int nthr) {
    q = C >> 2;
    rg = nthr / q < HT ? nthr / q : HT;
    j = threadIdx.x % q;
    r = threadIdx.x / q;
  }
};

__global__ void __launch_bounds__(POOL_THR) global_mean_pool_partial_kernel(
    const float* __restrict__ x, int C, const float* __restrict__ mass, int64_t V, const int32_t* __restrict__ begin,
    const int32_t* __restrict__ rows, const int32_t* __restrict__ tile_seg, int n_seg, float* wx, float* wm) {
  __shared__ float4 red[POOL_THR];
  __shared__ float redm[POOL_THR];
  const PoolLanes l(C, POOL_THR);
  const bool lead = l.r < l.rg;
  const int64_t n_tiles = cdiv(V, HT);
  const int64_t t0 = (int64_t)blockIdx.x * POOL_TILES;
  const int64_t t1 = t0 + POOL_TILES < n_tiles ? t0 + POOL_TILES : n_tiles;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float am = 0.f;
  int s = pool_seg(tile_seg, n_seg, t0);
  for (int64_t t = t0; t < t1; ++t) {
    const int s_next = t + 1 < t1 ? pool_seg(tile_seg, n_seg, t + 1) : -2;
    if (s >= 0 && lead) {
      const int64_t b = __ldg(begin + s);
      int64_t e = b + __ldg(rows + s);
      e = e < V ? e : V;
      const int64_t v1 = HT * t + HT < e ? HT * t + HT : e;
#pragma unroll 8
      for (int64_t v = HT * t + l.r; v < v1; v += l.rg) {
        if (v < b) continue;
        const float m = __ldg(mass + v);
        const float4 xv = __ldg(reinterpret_cast<const float4*>(x + v * C) + l.j);
        acc.x += m * xv.x; acc.y += m * xv.y; acc.z += m * xv.z; acc.w += m * xv.w;
        am += m;
      }
    }
    if (s >= 0 && s_next != s) {   // the run ends at tile t: fold the row groups in order
      red[threadIdx.x] = acc;
      redm[threadIdx.x] = am;
      __syncthreads();
      if (threadIdx.x < l.q) {
        float4 f = red[l.j];
        for (int k = 1; k < l.rg; ++k) {
          const float4 o = red[k * l.q + l.j];
          f.x += o.x; f.y += o.y; f.z += o.z; f.w += o.w;
        }
        reinterpret_cast<float4*>(wx + t * C)[l.j] = f;
        if (l.j == 0) {
          float fm = redm[0];
          for (int k = 1; k < l.rg; ++k) fm += redm[k * l.q];
          wm[t] = fm;
        }
      }
      __syncthreads();
      acc = make_float4(0.f, 0.f, 0.f, 0.f);
      am = 0.f;
    }
    s = s_next;
  }
}

// pooled[b] = (sum of segment b's runs) / (its mass sum), the runs split over rg slices in a fixed order; one CTA per
// segment.  msum[b] (the mass sum) is what the backward needs.
__global__ void __launch_bounds__(POOL_RTHR) global_mean_pool_reduce_kernel(
    const float* __restrict__ wx, const float* __restrict__ wm, int64_t V, int C, const int32_t* __restrict__ begin,
    const int32_t* __restrict__ rows, float* pooled, float* msum) {
  __shared__ float4 red[POOL_RTHR];
  __shared__ float redm[POOL_RTHR];
  const PoolLanes l(C, POOL_RTHR);
  const int sg = blockIdx.x;
  const int64_t b = __ldg(begin + sg), e = b + __ldg(rows + sg);
  const int64_t tb = b / HT, te = cdiv(e < V ? e : V, HT);
  // run k of the segment ends at tile min(POOL_TILES k + POOL_TILES - 1, te - 1), k = tb / POOL_TILES ..
  const int64_t k0 = tb / POOL_TILES, k1 = te > tb ? (te - 1) / POOL_TILES + 1 : k0;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float am = 0.f;
  if (l.r < l.rg) {
#pragma unroll 4
    for (int64_t k = k0 + l.r; k < k1; k += l.rg) {
      const int64_t t = POOL_TILES * k + POOL_TILES - 1 < te - 1 ? POOL_TILES * k + POOL_TILES - 1 : te - 1;
      const float4 o = __ldg(reinterpret_cast<const float4*>(wx + t * C) + l.j);
      acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w;
      am += __ldg(wm + t);
    }
  }
  red[threadIdx.x] = acc;
  redm[threadIdx.x] = am;
  __syncthreads();
  if (threadIdx.x < l.q) {
    float4 f = red[l.j];
    float fm = redm[l.j];
    for (int k = 1; k < l.rg; ++k) {
      const float4 o = red[k * l.q + l.j];
      f.x += o.x; f.y += o.y; f.z += o.z; f.w += o.w;
      fm += redm[k * l.q + l.j];
    }
    reinterpret_cast<float4*>(pooled + (int64_t)sg * C)[l.j] = make_float4(f.x / fm, f.y / fm, f.z / fm, f.w / fm);
    if (l.j == 0) msum[sg] = fm;
  }
}

// grad_x[v] = mass[v] / msum[b] grad_pooled[b] on the rows of segment b, 0 on every other row
__global__ void global_mean_pool_bwd_kernel(const float* __restrict__ g, const float* __restrict__ mass,
                                            const float* __restrict__ msum, int64_t V, int C,
                                            const int32_t* __restrict__ begin, const int32_t* __restrict__ rows,
                                            const int32_t* __restrict__ tile_seg, int n_seg, float* gx) {
  const int q = C >> 2;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < V * q; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = i / q;
    const int j = (int)(i % q);
    const int s = pool_seg(tile_seg, n_seg, v / HT);
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
    if (s >= 0) {
      const int64_t b = __ldg(begin + s);
      if (v >= b && v < b + __ldg(rows + s)) {
        const float w = __ldg(mass + v) / __ldg(msum + s);
        const float4 gv = __ldg(reinterpret_cast<const float4*>(g + (int64_t)s * C) + j);
        o = make_float4(w * gv.x, w * gv.y, w * gv.z, w * gv.w);
      }
    }
    reinterpret_cast<float4*>(gx)[i] = o;
  }
}

size_t head_smem(int C) { return 1024 + 2 * RAW_BYTES + (size_t)HT * (C + 4) * 4 + 2 * B_IMG + 3 * HT * 4 + 16; }

// target of the reference's label_smoothing_log_loss: 1 - s on the label, s / (n_class - 1) elsewhere (s in [0, 1], and
// n_class >= 2 when s > 0: the caller checks)
void set_smoothing(HeadArgs& a, float s) {
  a.smooth = s > 0.f;
  a.ls_on = 1.f;
  a.ls_off = 0.f;
  a.ls_label = 1.f;
  if (a.smooth) {
    const double off = (double)s / (a.n_class - 1);
    a.ls_on = (float)(1.0 - s);
    a.ls_off = (float)off;
    a.ls_label = (float)(1.0 - s - off);
  }
}

template <typename K>
int launch(K kernel, dim3 grid, int C, const HeadArgs& a, cudaStream_t st) {
  const size_t sm = head_smem(C);
  DN_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  kernel<<<grid, NTHR, sm, st>>>(a);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

template <int MODE>
int launch_bwd(dim3 gx, dim3 gw, int C, const HeadArgs& a, const HeadArgs& aw, cudaStream_t st) {
  const int rc = launch(linear_nll_dx_kernel<MODE>, gx, C, a, st);
  return rc ? rc : launch(linear_nll_dw_kernel<MODE>, gw, C, aw, st);
}

}  // namespace

int head_splits(int64_t R, int C, int n_class) {
  const int64_t tiles = cdiv(n_class, HT) * cdiv(C, HT);
  int64_t s = cdiv(2ll * dn_sm_count(), tiles);
  const int64_t rt = cdiv(R, HT);
  if (s > rt) s = rt;
  if (s > 1024) s = 1024;
  return (int)(s < 1 ? 1 : s);
}

int64_t head_ws_bytes(int64_t R, int C, int n_class) {
  return 4ll * head_splits(R, C, n_class) * n_class * (C + 1);
}

int64_t pool_ws_bytes(int64_t V, int C) { return 4ll * cdiv(V, HT) * (C + 1); }

int launch_global_mean_fwd(const float* x, const float* mass, int64_t V, int C, const int32_t* begin,
                           const int32_t* rows, const int32_t* tile_seg, int n_seg, float* pooled, float* msum,
                           void* ws, cudaStream_t st) {
  float* wx = static_cast<float*>(ws);
  float* wm = wx + cdiv(V, HT) * C;
  global_mean_pool_partial_kernel<<<(unsigned)cdiv(cdiv(V, HT), POOL_TILES), POOL_THR, 0, st>>>(
      x, C, mass, V, begin, rows, tile_seg, n_seg, wx, wm);
  DN_LAUNCH_CHECK();
  global_mean_pool_reduce_kernel<<<(unsigned)n_seg, POOL_RTHR, 0, st>>>(wx, wm, V, C, begin, rows, pooled, msum);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_global_mean_bwd(const float* g, const float* mass, const float* msum, int64_t V, int C,
                           const int32_t* begin, const int32_t* rows, const int32_t* tile_seg, int n_seg, float* gx,
                           cudaStream_t st) {
  const int64_t blocks = cdiv(V * (C / 4), 256);
  global_mean_pool_bwd_kernel<<<(unsigned)(blocks < 8192 ? blocks : 8192), 256, 0, st>>>(g, mass, msum, V, C, begin,
                                                                                       rows, tile_seg, n_seg, gx);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_linear_nll_fwd(const float* X, const float* W, const float* b, const int64_t* labels, int64_t R, int C,
                          int n_class, int64_t ignore_index, float label_smoothing, float* nll, int64_t* argmax,
                          float* lse, int passes, cudaStream_t st) {
  HeadArgs a{};
  a.X = X; a.W = W; a.b = b; a.labels = labels; a.R = R; a.C = C; a.n_class = n_class; a.ignore_index = ignore_index;
  a.nll = nll; a.argmax = argmax; a.lse_out = lse;
  set_smoothing(a, label_smoothing);
  if (!encode_tensor_map_f32(&a.amap, W, n_class, C, C, 32, HT, true)) return DN_ERR_UNSUPPORTED;
  a.bmap = a.amap;
  const dim3 grid((unsigned)cdiv(R, HT));
  if (passes == DN_PASSES_BF16) return launch(linear_nll_fwd_kernel<MODE_BF16>, grid, C, a, st);
  if (passes == 1) return launch(linear_nll_fwd_kernel<MODE_TF32>, grid, C, a, st);
  return launch(linear_nll_fwd_kernel<MODE_TF32X3>, grid, C, a, st);
}

int launch_linear_nll_bwd(const float* X, const float* W, const float* b, const int64_t* labels, const float* lse,
                          const float* g, int64_t R, int C, int n_class, int64_t ignore_index, float label_smoothing,
                          float* dX, float* dW, float* db, void* ws, int passes, cudaStream_t st) {
  HeadArgs a{};
  a.X = X; a.W = W; a.b = b; a.labels = labels; a.lse = lse; a.g = g; a.R = R; a.C = C; a.n_class = n_class;
  a.ignore_index = ignore_index; a.dX = dX;
  set_smoothing(a, label_smoothing);
  a.S = head_splits(R, C, n_class);
  a.dWp = static_cast<float*>(ws);
  a.dbp = a.dWp + (int64_t)a.S * n_class * C;
  HeadArgs aw = a;       // the weight-gradient kernel streams X, the dX kernel W
  // fp32 [rows][C] in boxes of 32 columns with the 128-byte swizzle
  if (!encode_tensor_map_f32(&a.amap, W, n_class, C, C, 32, HT, true) ||
      !encode_tensor_map_f32(&a.bmap, W, n_class, C, C, 32, KS, true) ||
      !encode_tensor_map_f32(&aw.amap, X, R, C, C, 32, HT, true) ||
      !encode_tensor_map_f32(&aw.bmap, X, R, C, C, 32, KS, true))
    return DN_ERR_UNSUPPORTED;
  const dim3 gx((unsigned)cdiv(R, HT), (unsigned)cdiv(C, HT));
  const dim3 gw((unsigned)cdiv(n_class, HT), (unsigned)cdiv(C, HT), (unsigned)a.S);
  const int rc = passes == DN_PASSES_BF16 ? launch_bwd<MODE_BF16>(gx, gw, C, a, aw, st)
                 : passes == 1             ? launch_bwd<MODE_TF32>(gx, gw, C, a, aw, st)
                                           : launch_bwd<MODE_TF32X3>(gx, gw, C, a, aw, st);
  if (rc) return rc;
  const int64_t nw = (int64_t)n_class * C;
  const int64_t blocks = cdiv(nw + n_class, 256);
  linear_nll_reduce_kernel<<<(unsigned)(blocks < 4096 ? blocks : 4096), 256, 0, st>>>(a.dWp, a.dbp, a.S, nw, n_class,
                                                                                      dW, db);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_element_mean_fwd(const float* x, int C, const int64_t* elems, int64_t E, int k, float* out,
                            cudaStream_t st) {
  const int64_t blocks = cdiv(E * C, 256);
  element_mean_fwd_kernel<<<(unsigned)(blocks < 8192 ? (blocks > 0 ? blocks : 1) : 8192), 256, 0, st>>>(x, C, elems, E,
                                                                                                      k, out);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int launch_element_mean_bwd(const float* g, int C, const int32_t* rowptr, const int32_t* ent, int64_t V, int k,
                            float* gx, cudaStream_t st) {
  const int64_t blocks = cdiv(V * C, 256);
  element_mean_bwd_kernel<<<(unsigned)(blocks < 8192 ? (blocks > 0 ? blocks : 1) : 8192), 256, 0, st>>>(g, C, rowptr,
                                                                                                      ent, V, k, gx);
  DN_LAUNCH_CHECK();
  return DN_OK;
}
