// Inline-PTX wrappers for the Hopper (sm_90a) features the tensor-core engine uses:
// mbarrier, bulk and tiled TMA copies, proxy fences and warpgroup MMA (wgmma) with the A operand in registers; and the
// MMA step every tensor-core kernel (dn_tc.cu, dn_head.cu) shares: engine mode, A fragments, the MMAs of one K slice and
// the B-image layout.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "dn_internal.h"

namespace tc {

// The engine a tensor-core kernel instance runs, keyed on the pass count of the engine (`passes`, dn_internal.h):
// 1xTF32, 3xTF32 (lo*hi + hi*lo + hi*hi) or bf16.
enum { MODE_TF32 = 1, MODE_TF32X3 = 3, MODE_BF16 = DN_PASSES_BF16 };

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier -------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.shared::cta.b64 st, [%0];\n}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n}" ::"r"(bar), "r"(bytes)
               : "memory");
}
// Spin on the phase parity; traps (instead of hanging the GPU) if nothing arrives for ~2 s.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  long long t0 = 0;
  for (uint32_t it = 0;; ++it) {
    asm volatile(
        "{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) return;
    if ((it & 1023u) == 1023u) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000ll) __trap();
    }
  }
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// generic-proxy smem writes -> visible to the async proxy (wgmma / TMA reads)
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// brings the 128-byte line holding `p` into L2 (a hint: no register, no completion to wait for)
__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}
// named barrier over `count` threads (a multiple of 32)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// warpgroup register budget hand-off (every warp of the warpgroup executes it)
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// ---- bulk TMA copy global -> shared, completion on an mbarrier ----------------------------------
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst_smem, const void* src_gmem, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src_gmem), "r"(bytes), "r"(bar)
               : "memory");
}
// 2-D tiled TMA copy of the box at (column c0, row c1) of the tensor map `tmap` (a __grid_constant__ kernel parameter)
// into shared memory; elements outside the tensor are zero-filled and still counted in the transaction bytes
__device__ __forceinline__ void tma_tile_2d_g2s(uint32_t dst_smem, const void* tmap, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          dst_smem),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}

// ---- tiled TMA store shared -> global, bulk-group completion --------------------------------------
// 2-D tiled store of the box at (column c0, row c1) of `tmap` from shared memory; elements outside the tensor are not
// written.  The stores a thread issued since its last commit form one bulk group.
__device__ __forceinline__ void tma_tile_2d_s2g(const void* tmap, int c0, int c1, uint32_t src_smem) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];" ::"l"(
                   reinterpret_cast<uint64_t>(tmap)),
               "r"(c0), "r"(c1), "r"(src_smem)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's bulk groups still read their shared-memory source (the source may be rewritten)
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// at most N of this thread's bulk groups are incomplete (their global writes are done)
template <int N>
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// ---- wgmma ------------------------------------------------------------------------------------
// shared-memory matrix descriptor, no swizzle, K-major: core matrices of 8 rows x 16 bytes;
//   LBO = byte distance between core matrices adjacent in K, SBO = between 8-row groups
// bits: [0,14) addr>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [62,64) layout = 0 (no swizzle)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
__device__ __forceinline__ void fence_acc8(float* d) {
  asm volatile("" : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
               :: "memory");
}
// pins an A fragment ahead of the next wgmma_fence: without it the compiler may form the fragment (a convert, a
// subtraction) after the fence, right before its MMA, and ptxas then inserts a warpgroup arrive before every MMA
__device__ __forceinline__ void fence_frag4(uint32_t* a) {
  asm volatile("" : "+r"(a[0]), "+r"(a[1]), "+r"(a[2]), "+r"(a[3]) :: "memory");
}

// D[64 x 16] (+)= A[64 x 8] (registers, tf32) * B[8 x 16] (smem descriptor, K-major tf32), fp32 accumulate.
//   A fragment of lane (g = lane / 4, t = lane % 4) in warp w: a0 (16w+g, t), a1 (16w+g+8, t), a2 (16w+g, t+4),
//   a3 (16w+g+8, t+4);  D fragment: d[4b + {0,1,2,3}] = (16w+g, 8b+2t), (16w+g, 8b+2t+1), (16w+g+8, 8b+2t), (16w+g+8, 8b+2t+1)
__device__ __forceinline__ void wgmma_tf32_n16(float* d, const uint32_t* a, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %13, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate)
      : "memory");
}
// D[64 x 16] (+)= A[64 x 16] (registers, bf16 pairs) * B[16 x 16] (smem descriptor, K-major bf16), fp32 accumulate.
//   a0 = (16w+g, 2t..2t+1), a1 = (16w+g+8, 2t..2t+1), a2 = (16w+g, 2t+8..2t+9), a3 = (16w+g+8, 2t+8..2t+9)
__device__ __forceinline__ void wgmma_bf16_n16(float* d, const uint32_t* a, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %13, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate)
      : "memory");
}

// Full-width forms: D[64 x N] (+)= A * B[K x N] in one instruction (N = 128 or 256; N / 2 accumulators per lane).  B is
// the same K-major canonical layout with 8-row groups 128 B apart, so one descriptor at the operand's base covers all N
// columns, and the D fragment is the n16 fragments laid end to end: d[4b + {0,1,2,3}] belongs to 8-column block b.
#define DN_ACC8(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), \
                   "+f"(d[o + 6]), "+f"(d[o + 7])
#define DN_ACC64 DN_ACC8(0), DN_ACC8(8), DN_ACC8(16), DN_ACC8(24), DN_ACC8(32), DN_ACC8(40), DN_ACC8(48), DN_ACC8(56)
#define DN_ACC128 DN_ACC64, DN_ACC8(64), DN_ACC8(72), DN_ACC8(80), DN_ACC8(88), DN_ACC8(96), DN_ACC8(104), DN_ACC8(112), \
                  DN_ACC8(120)
#define DN_REGS64 \
  "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15," \
  "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31," \
  "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47," \
  "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
#define DN_REGS128 DN_REGS64 "," \
  "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79," \
  "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95," \
  "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111," \
  "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
// one wrapper: name, instruction, D register list, operand numbers of A / descriptor / scale-d, trailing immediates
#define DN_WGMMA_WIDE(NAME, INSTR, REGS, A, DESC, SCALE_D, IMM, ACC)                                                  \
  __device__ __forceinline__ void NAME(float* d, const uint32_t* a, uint64_t b_desc, uint32_t accumulate) {         \
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, " SCALE_D ", 0;\n" INSTR " {" REGS "}, {" A "}, " DESC ", p, " \
                 IMM ";\n}"                                                                                          \
                 : ACC                                                                                             \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate)                        \
                 : "memory");                                                                                      \
  }
DN_WGMMA_WIDE(wgmma_tf32_n128, "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32", DN_REGS64, "%64,%65,%66,%67",
              "%68", "%69", "1, 1", DN_ACC64)
DN_WGMMA_WIDE(wgmma_tf32_n256, "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32", DN_REGS128,
              "%128,%129,%130,%131", "%132", "%133", "1, 1", DN_ACC128)
DN_WGMMA_WIDE(wgmma_bf16_n128, "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16", DN_REGS64, "%64,%65,%66,%67",
              "%68", "%69", "1, 1, 0", DN_ACC64)
DN_WGMMA_WIDE(wgmma_bf16_n256, "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16", DN_REGS128,
              "%128,%129,%130,%131", "%132", "%133", "1, 1, 0", DN_ACC128)
#undef DN_WGMMA_WIDE
#undef DN_REGS128
#undef DN_REGS64
#undef DN_ACC128
#undef DN_ACC64
#undef DN_ACC8

// one MMA over the whole N-wide accumulator (N = 16, 128 or 256); `accumulate` = 0 starts a new sum (D = A B)
template <int N>
__device__ __forceinline__ void wgmma_tf32(float* d, const uint32_t* a, uint64_t b_desc, uint32_t accumulate) {
  static_assert(N == 16 || N == 128 || N == 256, "wgmma_tf32: unsupported width");
  if constexpr (N == 16) wgmma_tf32_n16(d, a, b_desc, accumulate);
  else if constexpr (N == 128) wgmma_tf32_n128(d, a, b_desc, accumulate);
  else wgmma_tf32_n256(d, a, b_desc, accumulate);
}
template <int N>
__device__ __forceinline__ void wgmma_bf16(float* d, const uint32_t* a, uint64_t b_desc, uint32_t accumulate) {
  static_assert(N == 16 || N == 128 || N == 256, "wgmma_bf16: unsupported width");
  if constexpr (N == 16) wgmma_bf16_n16(d, a, b_desc, accumulate);
  else if constexpr (N == 128) wgmma_bf16_n128(d, a, b_desc, accumulate);
  else wgmma_bf16_n256(d, a, b_desc, accumulate);
}

// two fp32 -> packed bf16x2 (round to nearest even): `lo` in bits [0,16), `hi` in bits [16,32)
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// error-compensated split  x ~= hi + lo  with hi, lo exactly representable in TF32
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  uint32_t h, l;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(x));
  hi = __uint_as_float(h);
  const float r = x - hi;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(r));
  lo = __uint_as_float(l);
}

// cheaper split for activations: hi = x rounded to TF32 (round-half-up on the magnitude bits); lo = x - hi is exact
// in fp32 and the MMA reads only its top 19 bits.  Non-finite inputs stay non-finite.
__device__ __forceinline__ void split_tf32_fast(float x, float& hi, float& lo) {
  hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
  lo = x - hi;
}

// ---- one MMA step of the tensor-core kernels -------------------------------------------------------------------
// A operand of one k8 TF32 slice from its four values in fragment order (a0 .. a3 of wgmma_tf32_n16): the hi and lo
// registers of the split x = hi + lo (the 1xTF32 engine issues hi only)
__device__ __forceinline__ void frag_tf32(const float* x, uint32_t* ah, uint32_t* al) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float h, l;
    split_tf32_fast(x[i], h, l);
    ah[i] = __float_as_uint(h);
    al[i] = __float_as_uint(l);
  }
}
// A operand of one k16 bf16 slice from its eight values in fragment order: a_i = (x[2i], x[2i + 1]) (wgmma_bf16_n16)
__device__ __forceinline__ void frag_bf16(const float* x, uint32_t* a) {
#pragma unroll
  for (int i = 0; i < 4; ++i) a[i] = pack_bf16x2(x[2 * i], x[2 * i + 1]);
}

// acc[64 x N] (+)= A * B over one K slice (k8 TF32, k16 bf16): one MMA, or for 3xTF32 lo*B_hi, hi*B_lo, hi*B_hi.  B is
// a K-major image at b_addr (kmajor_off, K groups lbo bytes apart), its 3xTF32 lo image lo_offset bytes further.
// `accumulate` = 0 starts a new sum.  The caller forms the fragments and fences, commits and waits.
template <int MODE, int N>
__device__ __forceinline__ void mma_step(float* acc, const uint32_t* ah, const uint32_t* al, uint32_t b_addr,
                                         uint32_t lo_offset, uint32_t lbo, uint32_t accumulate) {
  const uint64_t dh = make_desc(b_addr, lbo, 128);
  if constexpr (MODE == MODE_BF16) {
    wgmma_bf16<N>(acc, ah, dh, accumulate);
  } else if constexpr (MODE == MODE_TF32X3) {
    wgmma_tf32<N>(acc, al, dh, accumulate);
    wgmma_tf32<N>(acc, ah, make_desc(b_addr + lo_offset, lbo, 128), 1u);
    wgmma_tf32<N>(acc, ah, dh, 1u);
  } else {
    wgmma_tf32<N>(acc, ah, dh, accumulate);
  }
}

// Byte offset of element (k, n) in an N-column B image in the K-major canonical layout (no swizzle): core matrices of
// 8 columns x 16 bytes of K, 8-column groups 128 B apart, K groups (4 tf32 / 8 bf16) N * 16 B apart.
template <int MODE>
__host__ __device__ __forceinline__ uint32_t kmajor_off(int k, int n, int N) {
  if constexpr (MODE == MODE_BF16) return (k >> 3) * N * 16 + (n >> 3) * 128 + (n & 7) * 16 + (k & 7) * 2;
  else return (k >> 2) * N * 16 + (n >> 3) * 128 + (n & 7) * 16 + (k & 3) * 4;
}
// TF32 B images whose A operand is an accumulator fragment (columns 2t, 2t + 1 of a lane in every 8-column block) store
// K permuted inside every group of 8: slot s < 4 holds k = 2s, slot 4 + s holds k = 2s + 1.  The fragment of k8 slice
// b is then z[4b], z[4b + 2], z[4b + 1], z[4b + 3].  (bf16 fragments already match the accumulator layout.)
__host__ __device__ __forceinline__ int tf32_k_slot(int k) {
  const int j = k & 7;
  return (k & ~7) | ((j & 1) ? 4 + (j >> 1) : (j >> 1));
}
__host__ __device__ __forceinline__ int tf32_slot_k(int s) {
  const int j = s & 7;
  return (s & ~7) | (j < 4 ? 2 * j : 2 * (j - 4) + 1);
}

}  // namespace tc
