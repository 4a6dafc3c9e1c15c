// Hopper tensor-core engine (sm_90a): the dense contractions of the DiffusionNetBlock path.
//
//   tc_rows_chain       fused chain of affine layers over 128- or 192-vertex row tiles
//                       (from_basis [+ complex-linear P|Q], MiniMLP + skip)      layers.py:56-67,229-239
//   tc_to_basis_partial split-V  Phi^T (M x)                                      geometry.py:572-583
//
// Arithmetic: warpgroup MMAs (wgmma) with fp32 accumulation in registers.  TF32 engines: "3x" mode splits every
// operand x = hi + lo (both exactly TF32) and issues lo*hi + hi*lo + hi*hi, recovering fp32-grade products; "1x"
// issues hi*hi only.  bf16 engine: one bf16 pass.
//
// Data movement: weights are pre-split and pre-laid-out in the wgmma canonical (no-swizzle, K-major) layout by a
// small pack kernel and streamed per 16-wide K stage with bulk TMA copies (cp.async.bulk + mbarrier complete_tx).
// The A operand of every MMA is in registers.  For the first layer of a chain it is read from a shared-memory ring
// that a second producer lane fills from HBM with 2-D tiled TMA copies (8 columns x a tile's rows per copy), running
// ahead of the consumers across layers and tiles; every later layer's A is the previous layer's accumulator fragment
// (three-warpgroup chains: read back from the shared-memory staging buffer the epilogue wrote it to).
#include "dn_internal.h"
#include "dn_tc_ptx.cuh"
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_bf16.h>
#include <string.h>

namespace {

using namespace tc;

constexpr int KC = 16;                          // k-elements per weight stage
constexpr int W_RING_BYTES = 128 * 1024;        // weight ring: as many stages of the instantiation's width as fit
constexpr int W_NST_MAX = 8;                    // ... but no deeper than this
constexpr int A_NST_MAX = 8;                  // activation stages in flight (64 KiB per SM)
constexpr int SMEM_OPTIN = 232448;              // sm_90 opt-in dynamic shared memory per block
constexpr int OUT_ROWS = 64;                    // rows of an output / residual box: one consumer warpgroup's rows
constexpr int OUT_BOX_BYTES = 8 * OUT_ROWS * 4; // 8 columns x 64 rows, [64 rows][8 floats]
constexpr int RES_ROWS = 16;                    // three-warpgroup chains: a residual box is one consumer warp's rows

// Shared memory of rows_chain_kernel<MODE, NMAX, WIDE, CWG> (CWG consumer warpgroups of 64 rows: a tile is 64 CWG
// rows).  Weight ring: a slot holds one K stage of an NMAX-wide layer as the producer streams it (tf32x3: hi | lo
// images, 8 bytes per weight; tf32: hi, 4; bf16: 2), as many as fit in W_RING_BYTES, at most 8.  (With 16 slots for
// the narrower stages, repeated bf16 mesh-batch forwards once gave differing bits; the cause was not found, so the
// depth stays at 8.)  The first layer's activations: 16-column x (64 CWG)-row fp32 stages, each two 8-column boxes of
// [64 CWG rows][8 floats].  The TF32 chains at NMAX <= 128 also hold one output / residual staging buffer per consumer
// warpgroup (64 rows x NMAX fp32, 32 KiB at NMAX = 128).  Two consumer warpgroups: where everything does not fit the
// opt-in limit (tc3x at NMAX = 128 only), the weight ring gives up two slots and the activation ring one: 6 weight and
// 7 activation slots measured slightly faster than 5 and 8 (DESIGN.md §5).  At NMAX = 128 / 256: tc3x 6 slots of
// 16 KiB / 4 of 32 KiB; tc1x 8 of 8 KiB / 8 of 16 KiB; bf16 8 of 4 KiB / 8 of 8 KiB.  Three consumer warpgroups (full-
// width TF32 at NMAX = 128): 64 KiB of weight slots (tc3x 4 of 16 KiB, tc1x 8 of 8 KiB), 5 activation slots of
// 12 KiB and 96 KiB of staging.  `set_chain_smem` and the launch both read SMEM.
template <int MODE, int NMAX, int CWG = 2>
struct ChainRing {
  static_assert(CWG == 2 || (CWG == 3 && NMAX == 128 && MODE != MODE_BF16), "rows_chain_kernel: unsupported variant");
  static constexpr int TILE = 64 * CWG;                  // vertex rows per tile
  static constexpr int THREADS = 128 * CWG + 128;        // consumer warpgroups, then the producer warpgroup
  static constexpr int A_BOX = 8 * TILE * 4;
  static constexpr int A_STAGE = 2 * A_BOX;
  static constexpr int STAGE = KC * NMAX * (MODE == MODE_TF32X3 ? 8 : MODE == MODE_TF32 ? 4 : 2);
  static constexpr int W_BYTES = CWG == 2 ? W_RING_BYTES : W_RING_BYTES / 2;
  static constexpr int NST_FULL = W_BYTES / STAGE < W_NST_MAX ? W_BYTES / STAGE : W_NST_MAX;
  static constexpr int A_NST_FULL = CWG == 2 ? A_NST_MAX : 5;
  // (bf16 stores from registers: with the staging buffer two identical bf16 calls at V = 200k + 37 gave different
  // bits, and the cause was not found)
  static constexpr int STG = NMAX <= 128 && MODE != MODE_BF16 ? CWG * OUT_ROWS * NMAX * 4 : 0;
  // every layer's bias, staged once per CTA (NMAX = 256 chains run a single layer)
  static constexpr int BIAS = (NMAX <= 128 ? DN_MAX_LAYERS : 1) * NMAX * 4;
  static constexpr int RBARS = CWG;   // residual barriers: one per consumer warpgroup
  static constexpr int bars(int nst, int anst) { return 8 * (2 * nst + 2 * anst + RBARS); }   // full / empty, residual
  static constexpr int bytes(int nst, int anst) { return nst * STAGE + anst * A_STAGE + STG + BIAS + bars(nst, anst); }
  static constexpr bool kFull = bytes(NST_FULL, A_NST_FULL) <= SMEM_OPTIN;
  static constexpr int NST = kFull ? NST_FULL : NST_FULL - 2;
  static constexpr int A_NST = kFull ? A_NST_FULL : A_NST_FULL - 1;
  static constexpr int BARS = bars(NST, A_NST);
  static constexpr int SMEM = bytes(NST, A_NST);
  static_assert(SMEM <= SMEM_OPTIN, "rows_chain_kernel: shared memory over the opt-in limit");
  static_assert(CWG == 2 || kFull, "rows_chain_kernel: the three-warpgroup rings are sized to fit");
};

// bytes of one packed K stage of an N-wide layer: tf32 hi image (KC * N * 4) then lo image; bf16 uses the first quarter
__host__ __device__ __forceinline__ int64_t stage_stride(int N) { return (int64_t)KC * N * 8; }
__host__ __device__ __forceinline__ int64_t packed_bytes(int K, int N) {
  return (((K + KC - 1) / KC) * stage_stride(N) + 255) / 256 * 256;
}

// ---------------------------------------------------------------------------------------------
// weight pack: W -> K stages, each K-major canonical (no swizzle): 16-byte core rows, 8-row groups 128 B apart,
// k-groups N * 16 B apart.
//   fmt 0 (tf32): k-groups of 4; inside every group of 8 k the columns are stored in the order 0,2,4,6,1,3,5,7 so
//     that an accumulator fragment (two adjacent columns per lane) is directly the A fragment of the next layer
//   fmt 2 (bf16): k-groups of 8 in natural order (the bf16 A fragment already matches the accumulator)
// ---------------------------------------------------------------------------------------------
struct PackJob {
  const float* W;
  const float* W2;
  float* dst;
  int64_t ldw;
  int n_split, w_trans, K, N, blk0, fmt;
};
constexpr int kMaxPackJobs = 3 + DN_MAX_LAYERS;   // every dense layer of a block: from_basis, [P|Q] (two at most), MLP
struct PackJobs {
  PackJob j[kMaxPackJobs];
  int n;
  // optional: job 0's matrix is the spectral multiplier of every mesh (TcSpectral; layers.py:48-49, 62-64), formed here
  // instead of by a separate launch; sp_blocks blocks per mesh, sp_stride floats between the meshes' packed matrices
  TcSpectral sp;
  int sp_blocks;
  int64_t sp_stride;
};

__device__ __forceinline__ void pack_store(float* dst, int fmt, int N, int k, int n, float w) {
  char* base = reinterpret_cast<char*>(dst) + (int64_t)(k / KC) * stage_stride(N);
  const int kk = k % KC;
  if (fmt == 2) {
    *reinterpret_cast<__nv_bfloat16*>(base + kmajor_off<MODE_BF16>(kk, n, N)) = __float2bfloat16_rn(w);
    return;
  }
  float hi, lo;
  split_tf32(w, hi, lo);
  char* q = base + kmajor_off<MODE_TF32>(tf32_k_slot(kk), n, N);
  *reinterpret_cast<float*>(q) = hi;
  *reinterpret_cast<float*>(q + (int64_t)KC * N * 4) = lo;
}

// all weight matrices of a block forward in one launch (blocks are assigned to jobs by blk0)
__global__ void pack_weights_kernel(const __grid_constant__ PackJobs jobs) {
  int n, k;
  float w;
  if (jobs.sp.partial && (int)blockIdx.x < jobs.sp_blocks * jobs.sp.n_meshes) {
    // spectral job (job 0, blocks [0, sp_blocks * n_meshes)): a block = 32 consecutive elements (n fastest: coalesced)
    // of mesh b x 8 slices of its partial sums.  It is most of the launch, so it skips the job search below.
    const PackJob& J = jobs.j[0];
    const int K = J.K, N = J.N;
    __shared__ float red[8][33];
    const int b = jobs.sp.n_meshes > 1 ? (int)blockIdx.x / jobs.sp_blocks : 0;
    const int e = threadIdx.x & 31, sl = threadIdx.x >> 5;
    const int idx = ((int)blockIdx.x - b * jobs.sp_blocks) * 32 + e;
    if (jobs.sp.plain) {
      if (sl != 0 || idx >= K * N) return;
      pack_store(J.dst + b * jobs.sp_stride, J.fmt, N, idx / N, idx % N, jobs.sp.partial[(int64_t)b * K * N + idx]);
      return;
    }
    const int p0 = jobs.sp.mesh_cta_begin ? jobs.sp.mesh_cta_begin[b] : 0;
    const int p1 = jobs.sp.mesh_cta_begin ? jobs.sp.mesh_cta_begin[b + 1] : jobs.sp.P;
    float acc = 0.f;
    if (idx < K * N) {
      const float* pp = jobs.sp.partial + idx;
      const int64_t stride = (int64_t)K * N;
      for (int q = p0 + sl; q < p1; q += 8) acc += pp[(int64_t)q * stride];
    }
    red[sl][e] = acc;
    __syncthreads();
    if (sl != 0 || idx >= K * N) return;
    k = idx / N; n = idx % N;
    const float sum = pairwise_sum<8>(&red[0][e], 33);
    const float t = dn_clamp_time(jobs.sp.time[n]);
    w = dn_heat(jobs.sp.evals[(int64_t)b * K + k], t) * sum;
    pack_store(J.dst + b * jobs.sp_stride, J.fmt, N, k, n, w);
    if (jobs.sp.sum_out) jobs.sp.sum_out[(int64_t)b * K * N + idx] = sum;
    // the in-place clamp of the reference, written back by mesh 0 only: every other reader of t[n] in this launch reads
    // either value (max(t, 1e-8) is idempotent)
    if (b == 0 && k == K - 1 && !jobs.sp.no_clamp_writeback) jobs.sp.time[n] = t;
    return;
  }
  int ji = 0;
#pragma unroll
  for (int i = 1; i < kMaxPackJobs; ++i)
    if (i < jobs.n && (int)blockIdx.x >= jobs.j[i].blk0) ji = i;
  const PackJob& J = jobs.j[ji];
  const int K = J.K, N = J.N;
  const int idx = ((int)blockIdx.x - J.blk0) * blockDim.x + threadIdx.x;
  if (idx >= K * N) return;
  n = idx / K; k = idx % K;
  if (J.w_trans) w = (J.W2 && k >= J.n_split) ? J.W2[(int64_t)(k - J.n_split) * J.ldw + n] : J.W[(int64_t)k * J.ldw + n];
  else if (J.W2 && n >= J.n_split) w = J.W2[(int64_t)(n - J.n_split) * J.ldw + k];
  else w = J.W[(int64_t)n * J.ldw + k];
  pack_store(J.dst, J.fmt, N, k, n, w);
}

// ---------------------------------------------------------------------------------------------
// fused affine chain over 128-row tiles
// ---------------------------------------------------------------------------------------------
struct HcLayer {
  const float* wpack;
  const float* bias;
  const float* emul;
  const float* relu_mask;
  const float* row_scale;
  const float* residual;
  int64_t ld_res;
  float res_scale;
  float* out;
  int64_t ld_out;
  int K, N, relu, sibling;
};

struct HcParams {
  CUtensorMap amap[DN_MAX_SRC];   // layer 0's sources: fp32 [V rows][width], 8 x 128 boxes, rows >= V zero-filled
  // TF32 engines, NMAX <= 128: each layer's `out` and `residual` as fp32 [V rows][N] (row stride ld_out / ld_res), 8 x 64 boxes;
  // rows >= V are not written (out) or zero-filled (residual)
  CUtensorMap omap[DN_MAX_LAYERS];
  CUtensorMap rmap[DN_MAX_LAYERS];
  DnRowsSrc src;
  HcLayer layer[DN_MAX_LAYERS];
  int n_layers;
  int64_t V;
  const int32_t* tile_group;   // optional (mesh batches): layer 0 of tile t streams packed matrix tile_group[t]
  int64_t group_stride;        //   (floats between the packed matrices)
  const float* head_w;         // optional linear head behind the last layer (DiffusionNet.last_lin, layers.py:366-370)
  const float* head_b;
  float* head_out;
  int64_t ld_head_out;
  int head_n;
};
static_assert(sizeof(HcParams) <= 4096, "HcParams must fit the 4 KiB kernel parameter space");

// Both consumer warpgroups own 64 rows of the tile each and share the weight stages; one lane of warpgroup 2 streams
// the stages with bulk TMA (that warpgroup hands its registers to the consumers with setmaxnreg).  A second lane
// (warp 9) copies layer 0's activations of every tile into an A_NST-deep ring of 16-column stages with 2-D TMA: box h
// of a stage holds columns 8h .. 8h+7 as [128 rows][8 floats], so the 32 bytes a row contributes are contiguous and a
// half-warp's float2 reads (rows g = 0..3 of its warp, columns 2t, 2t+1) cover 128 consecutive bytes: every bank once,
// no conflict and no swizzle.  A stage whose columns lie in two sources (widths that are multiples of 8, not of 16)
// is two boxes from two tensor maps.  Consumers read their fragments, issue the stage's MMAs and release the slot
// (a proxy fence, then one arrival per warp); the producer meanwhile runs ahead into the next tile's first layer while
// the consumers are in the epilogue and the later layers.  The weight ring (ChainRing) is as deep as the
// instantiation's stage width allows.
// Per lane, the accumulator of an N-wide layer holds rows (16w+g, 16w+g+8) x columns (8b+2t, 8b+2t+1)
// for every 8-column block b: after the epilogue these values are the next layer's A fragments (columns of a 16-wide
// K stage: tf32 steps use the permuted weight order of pack_store, bf16 steps the natural one).  NMAX <= 128 chains
// any number of layers; NMAX = 256 runs a single layer (its accumulator alone takes 128 registers).
// WIDE: every layer is exactly NMAX wide (so every later layer's K is NMAX too).  Widths and trip counts are then
// compile-time and each k8 slice of a pass is one m64nNMAXk8 MMA over the whole accumulator; otherwise the layer is
// covered by N / 16 m64n16 MMAs per slice and pass.
// Outputs (TF32, NMAX <= 128): each consumer warpgroup writes a layer's result into its own staging buffer, laid out like
// the activation ring (box b = columns 8b .. 8b+7 as [64 rows][8 floats], so a warp's float2 writes cover 256
// contiguous bytes), and one elected lane stores the boxes with 2-D TMA (rows >= V clipped by the tensor map) and goes
// on.  A layer's residual comes into the same buffer by TMA, issued before the layer's MMAs; each lane reads its
// residual from the slot it then overwrites with the result.  Ordering: every thread that touched the buffer fences
// (generic -> async proxy) and passes the warpgroup's named barrier before the store is issued; before the buffer is
// written again (an epilogue, or a residual load) the elected lane waits until the previous stores have read it; and in
// the CTA's last tile it waits for its stores to complete before it goes on.  NMAX = 256 chains (their staging tile
// would not fit next to the rings) and the bf16 engine (ChainRing::STG) store from registers.
// CWG = 3 (full-width TF32 chains at NMAX = 128 without a sibling layer or tile groups): three consumer warpgroups
// share each weight stage, so a tile is 192 rows, a stage feeds 18 MMAs instead of 12 and the weights cross L2 a third
// less often; warpgroup 3 holds the producers.  The registers (160 per consumer) do not hold the activations as well:
// every layer's result goes to the staging buffer, and the next layer forms its A fragments there with the reads
// layer 0 uses on the activation ring.  A lane reads and writes only its own (row, column) pairs there (the accumulator
// layout is the A-fragment layout), so no barrier separates an epilogue from the next layer's reads.  A layer's
// residual can then no longer come into the buffer before its MMAs: each warp, once it has formed stage c's fragments,
// loads its own 16 rows of residual columns 16c .. 16c + 15 by TMA into the two boxes it has just read, on its
// warpgroup's residual mbarrier.  The head reads the finished rows from the buffer.
template <int MODE, int NMAX, bool WIDE, int CWG = 2>
__global__ void __launch_bounds__(ChainRing<MODE, NMAX, CWG>::THREADS, 1) rows_chain_kernel(const __grid_constant__ HcParams p) {
  constexpr bool kChain = NMAX <= 128;
  constexpr bool kStage = ChainRing<MODE, NMAX, CWG>::STG > 0;   // outputs and residuals through shared memory
  constexpr bool kSmemAct = CWG == 3;   // later layers' activations and the residual in the staging buffer
  static_assert(!kSmemAct || (WIDE && kStage), "rows_chain_kernel: three consumer warpgroups need full-width staging");
  constexpr int NB = NMAX / 16;
  using Ring = ChainRing<MODE, NMAX, CWG>;
  constexpr int NST = Ring::NST, STAGE_BYTES = Ring::STAGE, A_NST = Ring::A_NST;
  constexpr int TILE = Ring::TILE, A_BOX_BYTES = Ring::A_BOX, A_STAGE_BYTES = Ring::A_STAGE;
  constexpr int NCW = 4 * CWG;   // consumer warps: arrivals per ring slot
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* aring = smem + NST * STAGE_BYTES;
  uint8_t* stage_out = aring + A_NST * A_STAGE_BYTES;
  float* sbias = reinterpret_cast<float*>(stage_out + Ring::STG);
  uint64_t* bars = reinterpret_cast<uint64_t*>(stage_out + Ring::STG + Ring::BIAS);
  const uint32_t full = smem_u32(bars), empty = smem_u32(bars + NST);
  const uint32_t afull = smem_u32(bars + 2 * NST), aempty = smem_u32(bars + 2 * NST + A_NST);
  const uint32_t rfull = smem_u32(bars + 2 * NST + 2 * A_NST);   // residual loaded, one per consumer warpgroup
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < NST; ++i) { mbar_init(full + 8 * i, 1); mbar_init(empty + 8 * i, NCW); }
    for (int i = 0; i < A_NST; ++i) { mbar_init(afull + 8 * i, 1); mbar_init(aempty + 8 * i, NCW); }
    for (int i = 0; i < Ring::RBARS; ++i) mbar_init(rfull + 8 * i, CWG == 2 ? 1 : 4);
    fence_barrier_init();
  }
  __syncthreads();
  const int L = p.n_layers;
  const int64_t ntiles = (p.V + TILE - 1) / TILE;

  if (warp >= NCW) {
    setmaxnreg_dec<CWG == 2 ? 40 : 24>();
    if (warp == NCW + 1 && lane == 0) {
      // ===================== layer-0 activation producer =====================
      const int K0 = p.layer[0].K, nst0 = (K0 + KC - 1) / KC;
      uint32_t s = 0, ph = 0;
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
        for (int c = 0; c < nst0; ++c) {
          const int nbox = c * KC + 8 < K0 ? 2 : 1;   // a half stage (K % 16 == 8) is one box
          mbar_wait(aempty + 8 * s, ph ^ 1);
          mbar_arrive_expect_tx(afull + 8 * s, (uint32_t)(nbox * A_BOX_BYTES));
          for (int h = 0; h < nbox; ++h) {
            int kc = c * KC + 8 * h, sidx = 0;
            while (sidx + 1 < p.src.nsrc && kc >= p.src.width[sidx]) { kc -= p.src.width[sidx]; ++sidx; }
            tma_tile_2d_g2s(smem_u32(aring + s * A_STAGE_BYTES + h * A_BOX_BYTES), &p.amap[sidx], kc,
                            (int)(tile * TILE), afull + 8 * s);
          }
          if (++s == A_NST) { s = 0; ph ^= 1; }
        }
    }
    // ===================== weight producer =====================
    if (warp == NCW && lane == 0) {
      uint32_t s = 0, ph = 0;
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
        for (int l = 0; l < L; ++l) {
          const HcLayer& Lr = p.layer[l];
          const int nst = (Lr.K + KC - 1) / KC;
          const int64_t sstride = stage_stride(Lr.N);
          const uint32_t bytes = (uint32_t)(MODE == MODE_TF32X3 ? sstride : (MODE == MODE_TF32 ? sstride / 2 : sstride / 4));
          const char* w = reinterpret_cast<const char*>(Lr.wpack);
          if (l == 0 && p.tile_group) w += (int64_t)__ldg(p.tile_group + tile) * p.group_stride * 4;
          for (int c = 0; c < nst; ++c) {
            mbar_wait(empty + 8 * s, ph ^ 1);
            mbar_arrive_expect_tx(full + 8 * s, bytes);
            tma_bulk_g2s(smem_u32(smem + s * STAGE_BYTES), w + c * sstride, bytes, full + 8 * s);
            if (++s == NST) { s = 0; ph ^= 1; }
          }
        }
    }
    return;
  }

  // ===================== consumers =====================
  setmaxnreg_inc<CWG == 2 ? 232 : 160>();
  // The biases go to shared memory once per CTA.  Read from global memory in the epilogue they were one round trip per
  // column block (the epilogue's loads are kept in series, see below), and the residual and output traffic of the
  // tiles evicts them from L1: the two hidden-layer epilogues of the MiniMLP took about 10,000 cycles each that way.
  for (int l = 0; l < L; ++l) {
    const HcLayer& Lr = p.layer[l];
    if (!Lr.bias) continue;
    for (int n = threadIdx.x; n < Lr.N; n += 128 * CWG) sbias[l * NMAX + n] = __ldg(Lr.bias + n);
  }
  named_bar_sync(1, 128 * CWG);               // the consumers' copies are done (the producers do not take part)
  const int g = lane >> 2, t = lane & 3;
  const int rloc = (warp >> 2) * 64 + (warp & 3) * 16 + g;
  // output / residual staging (NMAX <= 128)
  const int wg = warp >> 2;
  const bool elected = (threadIdx.x & 127) == 0;   // issues the warpgroup's TMA loads and stores
  // box b (columns 8b .. 8b+7, [64 rows][8 floats]) of this warpgroup's buffer
  auto stg_box = [&](int b) { return reinterpret_cast<float*>(stage_out) + (wg * NMAX + 8 * b) * OUT_ROWS; };
  float acc[NB * 8];
  float act[kChain && !kSmemAct ? NB * 8 : 1];
  uint32_t s = 0, ph = 0, as = 0, aph = 0, rph = 0;

  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t r0 = tile * TILE + rloc, r1 = r0 + 8;
    const bool ok0 = r0 < p.V, ok1 = r1 < p.V;
    const int row0 = (int)(tile * TILE) + wg * OUT_ROWS;   // this warpgroup's first row (V < 2^31 - 256)
    for (int l = 0; l < L; ++l) {
      const HcLayer& Lr = p.layer[l];
      const int N = WIDE ? NMAX : Lr.N, nb = N / 16;
      const int K = (WIDE && l > 0) ? NMAX : Lr.K, nst = (K + KC - 1) / KC;
      const uint32_t lbo = (uint32_t)N * 16;
      int prev = -1;
      // kSmemAct: the stores of the layer before (in the previous tile, for layer 0) read the buffer this layer's
      // residual loads and epilogue write
      const bool pred_stored = kSmemAct && p.layer[l > 0 ? l - 1 : L - 1].out != nullptr;
      // kSmemAct: this warp's residual columns 16c .. 16c + 15 come into boxes 2c, 2c + 1 of its 16 rows, once every
      // lane's reads of them (generic proxy) are ordered before the async-proxy write; a warp wholly past V loads
      // nothing (its rows are not stored).  The warpgroup's residual barrier takes one arrival per warp, each with
      // its own bytes.
      auto residual_load = [&](int c) {
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) {
          const int wrow0 = row0 + (warp & 3) * RES_ROWS;
          if (c == 0) {
            if (wrow0 < p.V) mbar_arrive_expect_tx(rfull + 8 * wg, (uint32_t)(N / 8 * RES_ROWS * 32));
            else mbar_arrive(rfull + 8 * wg);
          }
          if (wrow0 < p.V)
            for (int h = 0; h < 2; ++h)
              tma_tile_2d_g2s(smem_u32(stg_box(2 * c + h) + (warp & 3) * RES_ROWS * 8), &p.rmap[l], 16 * c + 8 * h,
                              wrow0, rfull + 8 * wg);
        }
      };
      if constexpr (kSmemAct) {
        if (pred_stored && Lr.residual) {
          if (elected) bulk_wait_read<0>();
          named_bar_sync(2 + wg, 128);
        }
      } else if constexpr (kStage) {
        // the residual rows come into the staging buffer while the layer's MMAs run, once the buffer's last stores
        // have read it (issued a layer or more ago); a warpgroup wholly past V loads nothing (its rows are not stored)
        if (Lr.residual && elected) {
          bulk_wait_read<0>();
          if (row0 < p.V) {
            mbar_arrive_expect_tx(rfull + 8 * wg, (uint32_t)(Lr.N / 8 * OUT_BOX_BYTES));
            for (int b = 0; b < Lr.N / 8; ++b)
              tma_tile_2d_g2s(smem_u32(stg_box(b)), &p.rmap[l], 8 * b, row0, rfull + 8 * wg);
          } else {
            mbar_arrive(rfull + 8 * wg);
          }
        }
      }
      // The epilogue reads the rows' emul and relu-mask values (NMAX = 256: also the residual) from global memory one
      // column block after the other (their loads cannot all be in flight at once: the registers do not fit), so each
      // is a round trip.  Asking L2 for those rows now, while this layer's MMAs run, makes every one of those round
      // trips an L2 hit.  The four lanes that share a row pair ask for one 128-byte line each of every 512 bytes; lane 0
      // also for the row's end.
      auto prefetch_rows = [&](const float* base, int64_t ld) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!(h ? ok1 : ok0)) continue;
          const char* row = reinterpret_cast<const char*>(base + (h ? r1 : r0) * ld);
          for (int b = 128 * t; b < N * 4; b += 512) prefetch_l2(row + b);
          if (t == 0) prefetch_l2(row + N * 4 - 4);
        }
      };
      if (!kStage && Lr.residual) prefetch_rows(Lr.residual, Lr.ld_res);
      if (Lr.emul) prefetch_rows(Lr.emul, N);
      if (Lr.relu_mask) prefetch_rows(Lr.relu_mask, N);
      // one K stage: q[0], q[1] = rows (r0, r1) x columns (2t, 2t+1); q[2], q[3] the same 8 columns further.  All A
      // fragments of the stage are formed before wgmma_fence, so the MMAs read registers the fence already covers and
      // ptxas has no reason to order them.  One commit group per stage, at most two stages in flight -- except in the
      // full-width TF32 chains: there the accumulator, the activations and two stages of fragments do not fit in the
      // register budget together (ptxas spills or serializes), so each stage waits for its own MMAs (up to six
      // full-width MMAs per stage; the other consumer warpgroup keeps the tensor cores busy meanwhile).  `two` marks
      // a stage whose second k8 slice lies inside K (a literal wherever it is known at compile time).
      // Weight slots: where a stage waits for its own MMAs (wait<0>) it hands its slot back right there; under wait<1>
      // the previous stage's slot is handed back once that stage's MMAs are done.
      auto stage = [&](int c, const float2* q, bool two) {
        mbar_wait(full + 8 * s, ph);
        // a stage is one k16 slice (bf16) or two k8 slices (TF32)
        constexpr int SLICES = MODE == MODE_BF16 ? 1 : 2;
        uint32_t ah[2][4], al[2][4];
        if constexpr (MODE == MODE_BF16) {
          const float x[8] = {q[0].x, q[0].y, q[1].x, q[1].y, q[2].x, q[2].y, q[3].x, q[3].y};
          frag_bf16(x, ah[0]);
        } else {
#pragma unroll
          for (int ks = 0; ks < 2; ++ks) {
            const float2 u = q[2 * ks], v = q[2 * ks + 1];
            const float x[4] = {u.x, v.x, u.y, v.y};
            frag_tf32(x, ah[ks], al[ks]);
          }
        }
        const uint32_t sb = smem_u32(smem + s * STAGE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < SLICES; ++ks) {
          if (ks == 1 && !two) break;
          const uint32_t acc0 = (c > 0 || ks > 0) ? 1u : 0u;
          const uint32_t base = sb + ks * 2 * lbo;
          if constexpr (WIDE) {
            mma_step<MODE, NMAX>(acc, ah[ks], al[ks], base, KC * N * 4, lbo, acc0);
          } else {
#pragma unroll
            for (int j = 0; j < NB; ++j) {
              if (j >= nb) break;
              mma_step<MODE, 16>(acc + 8 * j, ah[ks], al[ks], base + j * 256, KC * N * 4, lbo, acc0);
            }
          }
        }
        wgmma_commit();
        if constexpr (WIDE && MODE != MODE_BF16) {
          wgmma_wait<0>();                     // this stage's MMAs are done: hand its own slot back
          if (lane == 0) mbar_arrive(empty + 8 * s);
        } else {
          wgmma_wait<1>();                     // the previous stage's MMAs are done: hand its slot back
          if (prev >= 0 && lane == 0) mbar_arrive(empty + 8 * prev);
          prev = (int)s;
        }
        if (++s == NST) { s = 0; ph ^= 1; }
      };

      if (l == 0) {
        for (int c = 0; c < nst; ++c) {
          const bool two = c * KC + 8 < K;
          mbar_wait(afull + 8 * as, aph);
          const float* a = reinterpret_cast<const float*>(aring + as * A_STAGE_BYTES) + rloc * 8 + 2 * t;
          float2 q[4];
          q[0] = *reinterpret_cast<const float2*>(a);
          q[1] = *reinterpret_cast<const float2*>(a + 64);
          q[2] = q[3] = make_float2(0.f, 0.f);
          if (two) {
            q[2] = *reinterpret_cast<const float2*>(a + A_BOX_BYTES / 4);
            q[3] = *reinterpret_cast<const float2*>(a + A_BOX_BYTES / 4 + 64);
          }
          stage(c, q, two);
          // the slot is handed back once the stage's fragments are formed from the loaded values and its MMAs issued,
          // behind a proxy fence: the producer's next TMA write to it (async proxy) must not overtake these
          // generic-proxy reads.  (Handing it back before the MMAs, even behind the same fence, made two identical
          // bf16 forwards differ.)
          fence_proxy_async();
          __syncwarp();
          if (lane == 0) mbar_arrive(aempty + 8 * as);
          if (++as == A_NST) { as = 0; aph ^= 1; }
          if constexpr (kSmemAct) {
            if (Lr.residual && c < nb) residual_load(c);
          }
        }
        if constexpr (kSmemAct) {
          if (Lr.residual)
            for (int c = nst; c < nb; ++c) residual_load(c);   // layer 0 narrower than its output
        }
      } else if constexpr (kSmemAct) {
#pragma unroll
        for (int c = 0; c < NB; ++c) {
          const float* a = stg_box(2 * c) + ((warp & 3) * 16 + g) * 8 + 2 * t;
          const float2 q[4] = {*reinterpret_cast<const float2*>(a), *reinterpret_cast<const float2*>(a + 64),
                               *reinterpret_cast<const float2*>(a + 8 * OUT_ROWS),
                               *reinterpret_cast<const float2*>(a + 8 * OUT_ROWS + 64)};
          stage(c, q, true);
          if (Lr.residual) residual_load(c);
        }
      } else if constexpr (kChain) {
#pragma unroll
        for (int c = 0; c < NB; ++c) {
          if (c >= nst) break;
          const float2 q[4] = {make_float2(act[8 * c], act[8 * c + 1]), make_float2(act[8 * c + 2], act[8 * c + 3]),
                               make_float2(act[8 * c + 4], act[8 * c + 5]), make_float2(act[8 * c + 6], act[8 * c + 7])};
          stage(c, q, WIDE || c * KC + 8 < K);
        }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int j = 0; j < NB; ++j) fence_acc8(acc + 8 * j);
      if (prev >= 0 && lane == 0) mbar_arrive(empty + 8 * prev);

      // ---- epilogue (the operation order of simt_rows_gemm)
      const bool last = l + 1 == L;
      const bool head = last && p.head_w != nullptr;
      const bool keep_act = !last && p.layer[l + 1].sibling;   // the next layer reads this layer's input again
      const float rs0 = (Lr.row_scale && ok0) ? __ldg(Lr.row_scale + r0) : 1.f;
      const float rs1 = (Lr.row_scale && ok1) ? __ldg(Lr.row_scale + r1) : 1.f;
      float hp0[kChain ? 1 : 8], hp1[kChain ? 1 : 8];   // head partial sums of a single-layer (256-wide) chain
#pragma unroll
      for (int o = 0; o < (kChain ? 1 : 8); ++o) hp0[o] = hp1[o] = 0.f;
      if constexpr (kStage) {
        if (Lr.residual) {
          // the residual is in the staging buffer.  The elected lane waits and the barrier passes the news on: every
          // lane of the warpgroup spinning here made ptxas spill and serialize the MMAs (kSmemAct: so did a per-warp
          // barrier, with lane 0 or every lane of the warp waiting on it)
          if (elected) mbar_wait(rfull + 8 * wg, rph);
          rph ^= 1;
          named_bar_sync(2 + wg, 128);
        } else if (kSmemAct ? pred_stored : Lr.out != nullptr) {
          if (elected) bulk_wait_read<0>();  // the buffer's last stores have read it
          named_bar_sync(2 + wg, 128);
        }
      }
      // the bound is read from the layer even where it is known at compile time: the branch keeps the compiler from
      // hoisting the epilogue loads of every column block ahead of the first one, which would not fit in registers
      const int nb_epi = Lr.N / 16;
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        if (j >= nb_epi) break;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int col = 16 * j + 8 * h + 2 * t;
          float* d = acc + 8 * j + 4 * h;
          float2 v0 = make_float2(d[0], d[1]), v1 = make_float2(d[2], d[3]);
          if (Lr.bias) {
            const float2 b = *reinterpret_cast<const float2*>(sbias + l * NMAX + col);
            const float b0 = b.x, b1 = b.y;
            v0.x += b0; v0.y += b1; v1.x += b0; v1.y += b1;
          }
          if (Lr.relu) {
            v0.x = fmaxf(v0.x, 0.f); v0.y = fmaxf(v0.y, 0.f); v1.x = fmaxf(v1.x, 0.f); v1.y = fmaxf(v1.y, 0.f);
          }
          if (Lr.emul) {
            if (ok0) { const float2 e = __ldg(reinterpret_cast<const float2*>(Lr.emul + r0 * N + col)); v0.x *= e.x; v0.y *= e.y; }
            if (ok1) { const float2 e = __ldg(reinterpret_cast<const float2*>(Lr.emul + r1 * N + col)); v1.x *= e.x; v1.y *= e.y; }
          }
          if (Lr.relu_mask) {
            if (ok0) {
              const float2 m = __ldg(reinterpret_cast<const float2*>(Lr.relu_mask + r0 * N + col));
              v0.x = m.x > 0.f ? v0.x : 0.f; v0.y = m.y > 0.f ? v0.y : 0.f;
            }
            if (ok1) {
              const float2 m = __ldg(reinterpret_cast<const float2*>(Lr.relu_mask + r1 * N + col));
              v1.x = m.x > 0.f ? v1.x : 0.f; v1.y = m.y > 0.f ? v1.y : 0.f;
            }
          }
          if (Lr.row_scale) { v0.x *= rs0; v0.y *= rs0; v1.x *= rs1; v1.y *= rs1; }
          if constexpr (kStage) {
            float* so = stg_box(2 * j + h) + ((warp & 3) * 16 + g) * 8 + 2 * t;   // rows 16w+g, +8 at so + 64
            if (Lr.residual) {
              const float2 ra = *reinterpret_cast<const float2*>(so), rb = *reinterpret_cast<const float2*>(so + 64);
              v0.x = fmaf(Lr.res_scale, ra.x, v0.x); v0.y = fmaf(Lr.res_scale, ra.y, v0.y);
              v1.x = fmaf(Lr.res_scale, rb.x, v1.x); v1.y = fmaf(Lr.res_scale, rb.y, v1.y);
            }
            if (kSmemAct || Lr.out) {
              *reinterpret_cast<float2*>(so) = v0;
              *reinterpret_cast<float2*>(so + 64) = v1;
            }
          } else {
            if (Lr.residual) {
              if (ok0) {
                const float2 r = __ldg(reinterpret_cast<const float2*>(Lr.residual + r0 * Lr.ld_res + col));
                v0.x = fmaf(Lr.res_scale, r.x, v0.x); v0.y = fmaf(Lr.res_scale, r.y, v0.y);
              }
              if (ok1) {
                const float2 r = __ldg(reinterpret_cast<const float2*>(Lr.residual + r1 * Lr.ld_res + col));
                v1.x = fmaf(Lr.res_scale, r.x, v1.x); v1.y = fmaf(Lr.res_scale, r.y, v1.y);
              }
            }
            if (Lr.out) {
              if (ok0) *reinterpret_cast<float2*>(Lr.out + r0 * Lr.ld_out + col) = v0;
              if (ok1) *reinterpret_cast<float2*>(Lr.out + r1 * Lr.ld_out + col) = v1;
            }
          }
          if constexpr (kChain && !kSmemAct) {
            if (!keep_act) {
              act[8 * j + 4 * h] = v0.x; act[8 * j + 4 * h + 1] = v0.y;
              act[8 * j + 4 * h + 2] = v1.x; act[8 * j + 4 * h + 3] = v1.y;
            }
          }
          if (!kChain && head) {
#pragma unroll
            for (int o = 0; o < (kChain ? 1 : 8); ++o) {
              if (o >= p.head_n) break;
              const float2 w = __ldg(reinterpret_cast<const float2*>(p.head_w + (int64_t)o * N + col));
              hp0[o] = fmaf(w.y, v0.y, fmaf(w.x, v0.x, hp0[o]));
              hp1[o] = fmaf(w.y, v1.y, fmaf(w.x, v1.x, hp1[o]));
            }
          }
        }
      }
      if constexpr (kStage) {
        // (kSmemAct: the next residual loads are ordered per warp behind the next layer's reads)
        if (Lr.out || (!kSmemAct && Lr.residual)) {
          // this warpgroup's reads and writes of the buffer come before the async proxy's next access to it
          fence_proxy_async();
          named_bar_sync(2 + wg, 128);
          if (Lr.out && elected && row0 < p.V) {
            for (int b = 0; b < Lr.N / 8; ++b)
              tma_tile_2d_s2g(&p.omap[l], 8 * b, row0, smem_u32(stg_box(b)));
            bulk_commit();
            // in the CTA's last tile, every store is complete before the lane goes on (and so before it exits).  The
            // same wait after the tile loop made ptxas spill the bf16 full-width chain.
            if (tile + gridDim.x >= ntiles) bulk_wait<0>();
          }
        }
      }
      if (head) {
        auto head_store = [&](int o, float a0, float a1) {
          a0 += __shfl_xor_sync(0xffffffffu, a0, 1);
          a0 += __shfl_xor_sync(0xffffffffu, a0, 2);
          a1 += __shfl_xor_sync(0xffffffffu, a1, 1);
          a1 += __shfl_xor_sync(0xffffffffu, a1, 2);
          const float b = p.head_b ? __ldg(p.head_b + o) : 0.f;
          if (t == 0 && ok0) p.head_out[r0 * p.ld_head_out + o] = a0 + b;
          if (t == 0 && ok1) p.head_out[r1 * p.ld_head_out + o] = a1 + b;
        };
        if constexpr (kChain) {
          // the finished rows are in act: one output at a time keeps two partial sums and one weight pair live
          // (the same summation order as the single-layer form below)
#pragma unroll 1
          for (int o = 0; o < p.head_n; ++o) {
            float a0 = 0.f, a1 = 0.f;
#pragma unroll
            for (int j = 0; j < NB; ++j) {
              if (j >= nb) break;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const float2 w = __ldg(reinterpret_cast<const float2*>(p.head_w + (int64_t)o * N + 16 * j + 8 * h + 2 * t));
                if constexpr (kSmemAct) {
                  const float* so = stg_box(2 * j + h) + ((warp & 3) * 16 + g) * 8 + 2 * t;
                  const float2 u0 = *reinterpret_cast<const float2*>(so), u1 = *reinterpret_cast<const float2*>(so + 64);
                  a0 = fmaf(w.y, u0.y, fmaf(w.x, u0.x, a0));
                  a1 = fmaf(w.y, u1.y, fmaf(w.x, u1.x, a1));
                } else {
                  const float* v = act + 8 * j + 4 * h;
                  a0 = fmaf(w.y, v[1], fmaf(w.x, v[0], a0));
                  a1 = fmaf(w.y, v[3], fmaf(w.x, v[2], a1));
                }
              }
            }
            head_store(o, a0, a1);
          }
        } else {
#pragma unroll
          for (int o = 0; o < (kChain ? 1 : 8); ++o) {
            if (o >= p.head_n) break;
            head_store(o, hp0[o], hp1[o]);
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// to_basis, split over V:  partial[cta][k][c] = sum_{v in cta's range} Phi[v][k] * m[v] * x[v][c]
//   D = Phi^T (M = K_eig rows: warpgroup 0 rows 0..63, warpgroup 1 rows 64..127) times (m x) (N = C columns); the
//   reduction runs over v in stages of TB_ROWS = 32 rows (4 k8 slices).  Warp 8 loads a stage of Phi and of x with
//   2-D tiled TMA, 8 columns x 32 rows per box, each box laid out [row][8 floats] (columns >= K or C and rows >= V come
//   back as zeros); the A fragments are read from there, B = (m x)^T is written K-major (hi | lo) by all consumers.
//   Both reads and the B-image stores put a warp's 32 lanes on 32 banks: a warp builds one 8-channel x 4-row core
//   matrix of B per step from one box row run, and a fragment read of Phi covers 4 rows x 8 columns of one box.
//   One named barrier per stage: before it every consumer has built its part of stage c's B image and has waited for
//   its own MMAs of stage c - 1, so after it stage c's MMAs may start and stage c + 1 may overwrite the B slot of c - 1.
//   The MMA accumulator is folded into an fp32 sum in shared memory every 128 rows (TB_FOLD stages): short
//   accumulation chains keep the tensor core's accumulation below fp32 noise even for V = 200k.
//   The channel count C = 16 NBC is a compile-time parameter, so every MMA sits on a path ptxas can see is uniform.
//   C == 128: each k8 slice of a pass is one m64n128k8 MMA; otherwise NBC m64n16 MMAs.  Both warpgroups always
//   issue their MMAs (a warpgroup whose 64 eigen-rows all lie beyond K multiplies zero A fragments and stores nothing),
//   so no MMA sits on a path that depends on the warp index.
// ---------------------------------------------------------------------------------------------
constexpr int TB_ROWS = 32;                  // rows per stage
constexpr int TB_NST = 3;                    // raw staging ring depth
constexpr int TB_BOX = TB_ROWS * 8 * 4;      // one TMA box: 32 rows x 8 floats
constexpr int TB_RAW_HALF = 16 * TB_BOX;     // up to 128 columns
constexpr int TB_RAW = 2 * TB_RAW_HALF;      // Phi boxes | x boxes
constexpr int TB_BIMG = TB_ROWS * 128 * 4;   // one tf32 image of B: up to 128 channels x 32 v
constexpr int TB_BSTAGE = 2 * TB_BIMG;       // hi | lo
constexpr int TB_THREADS = 288;              // warps 0..7 consumers (two warpgroups), warp 8 TMA
constexpr int TB_SUMS = 64 * 256 * 4;        // fp32 fold sums: 64 per consumer thread, [i][thread] (conflict-free)
constexpr int TB_SMEM = TB_NST * TB_RAW + 2 * TB_BSTAGE + TB_SUMS + 256;
constexpr int TB_FOLD = 128 / TB_ROWS;       // stages per accumulation chain
static_assert(TB_SMEM <= 227 * 1024, "to_basis shared memory");

struct TcToBasisParams {
  CUtensorMap phi_map;   // basis: fp32 [V rows][K], 8 x 32 boxes
  CUtensorMap x_map;     // values: fp32 [V rows][C], row stride ld_values, 8 x 32 boxes
  const float* mass;     // (V) or null
  float* partial;        // (grid, K, C)
  int64_t V;
  int K, C;
  int64_t chunks_per_cta;   // 16-row chunks per CTA
  int64_t ldp;           // row stride of a partial (floats): partial[cta][k][ldp]
  const int32_t* cta_rows;   // optional device [2 * grid]: the row range [begin, end) CTA i reduces (mesh batches: a CTA
};                           //   never crosses a mesh boundary); null = uniform chunks_per_cta * 16 rows per CTA

template <int MODE, int NBC>
__global__ void __launch_bounds__(TB_THREADS, 1) to_basis_kernel(const __grid_constant__ TcToBasisParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* raw = smem;
  uint8_t* bimg = smem + TB_NST * TB_RAW;
  float* sums = reinterpret_cast<float*>(bimg + 2 * TB_BSTAGE);
  uint64_t* bars = reinterpret_cast<uint64_t*>(bimg + 2 * TB_BSTAGE + TB_SUMS);
  const uint32_t st_full = smem_u32(bars), st_empty = smem_u32(bars + TB_NST);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < TB_NST; ++i) { mbar_init(st_full + 8 * i, 1); mbar_init(st_empty + 8 * i, 8); }
    fence_barrier_init();
  }
  __syncthreads();

  int64_t rb, re;
  if (p.cta_rows) {
    rb = p.cta_rows[2 * blockIdx.x];
    re = p.cta_rows[2 * blockIdx.x + 1];
  } else {
    rb = (int64_t)blockIdx.x * p.chunks_per_cta * KC;
    re = rb + p.chunks_per_cta * KC;
    if (re > p.V) re = p.V;
  }
  const int64_t nst = re > rb ? (re - rb + TB_ROWS - 1) / TB_ROWS : 0;
  constexpr int C = 16 * NBC, XB = C / 8;   // x boxes per stage
  const int K = p.K;

  if (warp == 8) {
    if (lane == 0) {
      const int kbn = (K + 7) / 8;            // Phi boxes per stage
      const uint32_t bytes = (uint32_t)(kbn + XB) * TB_BOX;
      for (int64_t c = 0; c < nst; ++c) {
        const uint32_t s = c % TB_NST, ph = (c / TB_NST) & 1;
        mbar_wait(st_empty + 8 * s, ph ^ 1);
        const int v0 = (int)(rb + c * TB_ROWS);
        const uint32_t dst = smem_u32(raw + s * TB_RAW);
        mbar_arrive_expect_tx(st_full + 8 * s, bytes);
        for (int b = 0; b < kbn; ++b) tma_tile_2d_g2s(dst + b * TB_BOX, &p.phi_map, 8 * b, v0, st_full + 8 * s);
#pragma unroll
        for (int b = 0; b < XB; ++b)
          tma_tile_2d_g2s(dst + TB_RAW_HALF + b * TB_BOX, &p.x_map, 8 * b, v0, st_full + 8 * s);
      }
    }
    return;
  }

  const int g = lane >> 2, t = lane & 3;
  const int m0 = (warp >> 2) * 64 + (warp & 3) * 16 + g;   // eigen-index rows m0, m0 + 8
  const int abox = m0 >> 3;                                 // their Phi boxes abox, abox + 1 (column m0 & 7 == g)
  const uint32_t lbo = (uint32_t)C * 16;
  // B image: this thread writes row bv of every stage, channels 8 b + (lane & 7), at boff + 128 b = kmajor_off(bv,
  // 8 b + (lane & 7), C).  (boff written with kmajor_off costs ptxas up to 4 more registers in some instances.)
  const int bv = 4 * warp + (lane >> 3);
  const uint32_t boff = (uint32_t)warp * C * 16 + (lane & 7) * 16 + (lane >> 3) * 4;
  // the fold sums live in shared memory: the 64 accumulators, the A fragments of a stage and the addressing fit the
  // register budget, a second register array of 64 would not
  float acc[64];
  float* sum = sums + threadIdx.x;
#pragma unroll
  for (int i = 0; i < 64; ++i) sum[256 * i] = 0.f;

  for (int64_t c = 0; c < nst; ++c) {
    const uint32_t s = c % TB_NST, ph = (c / TB_NST) & 1;
    const int64_t v0 = rb + c * TB_ROWS;
    const int nv = (int)((re - v0) < TB_ROWS ? (re - v0) : TB_ROWS);   // rows >= nv are another range's: zeroed
    const int fold = (int)(c % TB_FOLD);
    // the mass value (global) is loaded before the wait, so its latency overlaps it; row bv >= nv reads a valid row
    float mv = 1.f;
    if (p.mass) mv = __ldg(p.mass + v0 + (bv < nv ? bv : nv - 1));
    mbar_wait(st_full + 8 * s, ph);
    const float* rphi = reinterpret_cast<const float*>(raw + s * TB_RAW);
    const float* rx = reinterpret_cast<const float*>(raw + s * TB_RAW + TB_RAW_HALF);
    uint8_t* bh = bimg + (c & 1) * TB_BSTAGE;   // stage c - 2's MMAs, its last readers, were waited for before the
    float xv[XB];                               //   previous stage's barrier
#pragma unroll
    for (int b = 0; b < XB; ++b) xv[b] = rx[b * (TB_BOX / 4) + 32 * warp + lane];   // box b, row bv, column lane & 7
#pragma unroll
    for (int b = 0; b < XB; ++b) {
      float x = 0.f;
      if (bv < nv) x = p.mass ? xv[b] * mv : xv[b];     // (values * massvec), geometry.py:583
      float hi, lo;
      split_tf32_fast(x, hi, lo);
      *reinterpret_cast<float*>(bh + boff + 128 * b) = hi;
      if (MODE == MODE_TF32X3) *reinterpret_cast<float*>(bh + TB_BIMG + boff + 128 * b) = lo;
    }
    // the A fragment registers are the same in every stage: the MMAs of stage c - 1, which read them, must be done
    // before they are rewritten (they ran while this stage's B image was built)
    wgmma_wait<0>();
    if (fold == 0 && c > 0) {              // fold the finished accumulation chain into the sum
#pragma unroll
      for (int j = 0; j < 8; ++j) fence_acc8(acc + 8 * j);
#pragma unroll
      for (int i = 0; i < 64; ++i) sum[256 * i] += acc[i];
    }
    uint32_t ah[4][4], al[4][4];           // A fragments, all formed before wgmma_fence
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      float x[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int vv = 8 * ks + t + 4 * (i >> 1), k = m0 + 8 * (i & 1);
        // read unconditionally and select: the box stays inside the staging slot, and a load under a lane-dependent
        // branch would put the MMA operands on a divergent path
        const float v = rphi[(abox + (i & 1)) * (TB_BOX / 4) + vv * 8 + g];
        x[i] = (vv < nv && k < K) ? v : 0.f;
      }
      frag_tf32(x, ah[ks], al[ks]);
    }
    fence_proxy_async();
    __syncwarp();
    if (lane == 0) mbar_arrive(st_empty + 8 * s);
    named_bar_sync(1, 256);                // the B image is complete; every warp's MMAs of stage c - 1 are done
    const uint32_t sb = smem_u32(bh);
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      fence_frag4(ah[ks]);
      if (MODE == MODE_TF32X3) fence_frag4(al[ks]);
    }
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint32_t acc0 = (fold > 0 || ks > 0) ? 1u : 0u;
      const uint32_t base = sb + ks * 2 * lbo;
      if constexpr (NBC == 8) {
        mma_step<MODE, 128>(acc, ah[ks], al[ks], base, TB_BIMG, lbo, acc0);
      } else {
#pragma unroll
        for (int j = 0; j < NBC; ++j) mma_step<MODE, 16>(acc + 8 * j, ah[ks], al[ks], base + j * 256, TB_BIMG, lbo, acc0);
      }
    }
    wgmma_commit();
  }
  wgmma_wait<0>();
#pragma unroll
  for (int j = 0; j < 8; ++j) fence_acc8(acc + 8 * j);
  if (nst > 0)
#pragma unroll
    for (int i = 0; i < 64; ++i) sum[256 * i] += acc[i];
  float* out = p.partial + (int64_t)blockIdx.x * K * p.ldp;
#pragma unroll
  for (int b = 0; b < 16; ++b) {
    const int col = 8 * b + 2 * t;
    if (col >= C) break;
    if (m0 < K) *reinterpret_cast<float2*>(out + (int64_t)m0 * p.ldp + col) = make_float2(sum[256 * (4 * b)], sum[256 * (4 * b + 1)]);
    if (m0 + 8 < K)
      *reinterpret_cast<float2*>(out + (int64_t)(m0 + 8) * p.ldp + col) = make_float2(sum[256 * (4 * b + 2)], sum[256 * (4 * b + 3)]);
  }
}

// Per-device table: SM count and capability, read on the first use of the device, and whether the >48 KB dynamic
// shared memory attributes were set on it, tried on the first use of the tensor-core engine there (function attributes
// are per device: a process that drives several GPUs needs them on each one).
constexpr int kMaxDev = 64;
struct DevState { int queried, sms, sm90, tc_tried, tc; };
DevState g_dev[kMaxDev];

template <typename F>
bool set_smem(F* f, int bytes) {
  return cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) == cudaSuccess;
}
// to_basis_kernel<MODE, NBC> for NBC = NBC0 .. 8 (C = 16 .. 128)
template <int MODE, int NBC0 = 1>
bool set_to_basis_smem() {
  if constexpr (NBC0 > 8) return true;
  else return set_smem(to_basis_kernel<MODE, NBC0>, TB_SMEM) && set_to_basis_smem<MODE, NBC0 + 1>();
}
template <int MODE, int NBC0 = 1>
void launch_to_basis(int nbc, int grid, const TcToBasisParams& p, cudaStream_t st) {
  if constexpr (NBC0 <= 8) {
    if (nbc == NBC0) to_basis_kernel<MODE, NBC0><<<grid, TB_THREADS, TB_SMEM, st>>>(p);
    else launch_to_basis<MODE, NBC0 + 1>(nbc, grid, p, st);
  }
}
template <int MODE>
bool set_chain_smem() {
  constexpr int s128 = ChainRing<MODE, 128>::SMEM, s256 = ChainRing<MODE, 256>::SMEM;
  bool ok = set_smem(rows_chain_kernel<MODE, 128, false>, s128) && set_smem(rows_chain_kernel<MODE, 128, true>, s128) &&
            set_smem(rows_chain_kernel<MODE, 256, false>, s256) && set_smem(rows_chain_kernel<MODE, 256, true>, s256);
  if constexpr (MODE != MODE_BF16)
    ok = ok && set_smem(rows_chain_kernel<MODE, 128, true, 3>, ChainRing<MODE, 128, 3>::SMEM);
  return ok;
}

// cuTensorMapEncodeTiled from the driver the runtime already loaded (no link dependency on libcuda); null if absent
PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder() {
  static const PFN_cuTensorMapEncodeTiled_v12000 fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &f, 12000, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess) {
      cudaGetLastError();
      f = nullptr;
    }
    return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(f);
  }();
  return fn;
}

}  // namespace

bool encode_tensor_map_f32(CUtensorMap* m, const float* base, int64_t rows, int width, int64_t ld, int box_cols,
                           int box_rows, bool swizzle128) {
  const PFN_cuTensorMapEncodeTiled_v12000 encode = tensor_map_encoder();
  if (!encode) return false;
  const cuuint64_t dims[2] = {(cuuint64_t)width, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  const cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows}, estr[2] = {1, 1};
  return encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static DevState* cur_dev_state() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDev) {
    cudaGetLastError();
    return nullptr;
  }
  DevState& d = g_dev[dev];
  if (!d.queried) {
    d.queried = 1;
    int major = 0, minor = 0;
    if (cudaDeviceGetAttribute(&d.sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) {
      cudaGetLastError();
      major = 0;
    }
    if (d.sms < 1) d.sms = 1;
    d.sm90 = major == 9 && minor == 0;
  }
  return &d;
}

int dn_sm_count() {
  const DevState* d = cur_dev_state();
  return d ? d->sms : 1;
}

bool tc_supported_device() {
  DevState* d = cur_dev_state();
  if (!d || !d->sm90) return false;
  if (!d->tc_tried) {
    d->tc_tried = 1;
    d->tc = tensor_map_encoder() != nullptr && set_chain_smem<MODE_TF32X3>() && set_chain_smem<MODE_TF32>() &&
            set_chain_smem<MODE_BF16>() && set_to_basis_smem<MODE_TF32X3>() && set_to_basis_smem<MODE_TF32>();
    if (!d->tc) cudaGetLastError();
  }
  return d->tc;
}

static bool aligned8(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 7) == 0; }
static bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

// shapes rows_chain_kernel takes (bf16: 16-wide K steps; tf32: 8-wide).  Layer 0's sources and every layer's out and
// residual are TMA tensor maps: base 16-byte aligned, row stride a multiple of 16 bytes.
static int chain_supported(const DnRowsSrc& src, const DnLayer* layers, int n_layers, bool bf16) {
  const int ks = bf16 ? 16 : 8;
  if (n_layers < 1 || n_layers > DN_MAX_LAYERS) return DN_ERR_UNSUPPORTED;
  int k0 = 0;
  for (int s = 0; s < src.nsrc; ++s) {
    if (src.width[s] % ks || src.ld[s] % 4 || src.ld[s] < src.width[s] || !aligned16(src.ptr[s]))
      return DN_ERR_UNSUPPORTED;
    k0 += src.width[s];
  }
  if (k0 != layers[0].K) return DN_ERR_UNSUPPORTED;
  for (int l = 0; l < n_layers; ++l) {
    const DnLayer& L = layers[l];
    const bool last = l + 1 == n_layers;
    if (L.K % ks || L.K < ks || L.N % 16 || L.N < 16 || L.N > (n_layers > 1 ? 128 : 256)) return DN_ERR_UNSUPPORTED;
    // a sibling reads the input of the layer before it, which must itself be a chain layer (not layer 0's sources)
    if (L.sibling && l < 2) return DN_ERR_UNSUPPORTED;
    if (l > 0 && (L.K != (L.sibling ? layers[l - 1].K : layers[l - 1].N) || L.tile_group)) return DN_ERR_UNSUPPORTED;
    if (L.emul && !aligned8(L.emul)) return DN_ERR_UNSUPPORTED;
    if (L.relu_mask_src && !aligned8(L.relu_mask_src)) return DN_ERR_UNSUPPORTED;
    // out and residual are TMA tensor maps too (the same rule as layer 0's sources)
    if (L.residual && (L.ld_res % 4 || !aligned16(L.residual))) return DN_ERR_UNSUPPORTED;
    if (L.out && (L.ld_out % 4 || !aligned16(L.out))) return DN_ERR_UNSUPPORTED;
    if (!last && L.head_w) return DN_ERR_UNSUPPORTED;
    if (last && !L.out && !L.head_w) return DN_ERR_UNSUPPORTED;
    if (L.head_w && (!L.head_out || L.head_n < 1 || L.head_n > 8 || !aligned8(L.head_w))) return DN_ERR_UNSUPPORTED;
  }
  return DN_OK;
}

int tc_chain_plan(const DnRowsSrc& src, DnLayer* layers, int n_layers, int passes) {
  int fmt;
  if (passes == DN_PASSES_BF16 && chain_supported(src, layers, n_layers, true) == DN_OK) fmt = 2;
  else if (chain_supported(src, layers, n_layers, false) == DN_OK) fmt = 0;
  else return DN_ERR_UNSUPPORTED;
  for (int l = 0; l < n_layers; ++l) layers[l].pack_fmt = fmt;
  return fmt;
}

int64_t tc_chain_ws_bytes(const DnLayer* layers, int n_layers, int n_meshes) {
  int64_t b = (n_meshes - 1) * packed_bytes(layers[0].K, layers[0].N);
  for (int l = 0; l < n_layers; ++l) b += packed_bytes(layers[l].K, layers[l].N);
  return b;
}

int tc_pack_layers(DnLayer* layers, int n_layers, void* ws, int64_t ws_bytes, const TcSpectral* sp, cudaStream_t st) {
  if (n_layers < 1 || n_layers > kMaxPackJobs || (sp && sp->n_meshes < 1)) return DN_ERR_INVALID_ARGUMENT;
  if (tc_chain_ws_bytes(layers, n_layers, sp ? sp->n_meshes : 1) > ws_bytes || !ws) return DN_ERR_WORKSPACE;
  PackJobs jobs;
  memset(&jobs, 0, sizeof(jobs));
  jobs.n = n_layers;
  char* wp = static_cast<char*>(ws);
  int blocks = 0;
  for (int l = 0; l < n_layers; ++l) {
    DnLayer& L = layers[l];
    PackJob& J = jobs.j[l];
    J.W = L.W; J.W2 = L.W2; J.n_split = L.n_split; J.ldw = L.ldw; J.w_trans = L.w_trans; J.K = L.K; J.N = L.N;
    J.fmt = L.pack_fmt;
    J.dst = reinterpret_cast<float*>(wp);
    J.blk0 = blocks;
    L.prepacked = J.dst;
    if (l == 0 && sp) {
      jobs.sp = *sp;
      jobs.sp_blocks = (L.K * L.N + 31) / 32;
      jobs.sp_stride = packed_bytes(L.K, L.N) / 4;
      blocks += jobs.sp_blocks * sp->n_meshes;
      wp += packed_bytes(L.K, L.N) * sp->n_meshes;
      if (sp->tile_mesh) { L.tile_group = sp->tile_mesh; L.group_stride = jobs.sp_stride; }
    } else {
      blocks += (L.K * L.N + 255) / 256;
      wp += packed_bytes(L.K, L.N);
    }
  }
  pack_weights_kernel<<<blocks, 256, 0, st>>>(jobs);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

// wide: every layer is exactly 128 wide, or the single layer is 256 wide (full-width MMAs); cwg: consumer warpgroups
template <int MODE>
static void launch_chain(const HcParams& p, int nmax, bool wide, int cwg, int grid, cudaStream_t st) {
  using R128 = ChainRing<MODE, 128>;
  using R256 = ChainRing<MODE, 256>;
  if constexpr (MODE != MODE_BF16) {
    if (cwg == 3) {
      using R3 = ChainRing<MODE, 128, 3>;
      rows_chain_kernel<MODE, 128, true, 3><<<grid, R3::THREADS, R3::SMEM, st>>>(p);
      return;
    }
  }
  if (nmax <= 128) {
    if (wide) rows_chain_kernel<MODE, 128, true><<<grid, R128::THREADS, R128::SMEM, st>>>(p);
    else rows_chain_kernel<MODE, 128, false><<<grid, R128::THREADS, R128::SMEM, st>>>(p);
  } else {
    if (wide) rows_chain_kernel<MODE, 256, true><<<grid, R256::THREADS, R256::SMEM, st>>>(p);
    else rows_chain_kernel<MODE, 256, false><<<grid, R256::THREADS, R256::SMEM, st>>>(p);
  }
}

int tc_rows_chain(const DnRowsSrc& src, const DnLayer* layers_in, int n_layers, int64_t V, int passes, void* ws,
                  int64_t ws_bytes, cudaStream_t st) {
  if (V <= 0) return DN_OK;
  if (n_layers < 1 || n_layers > DN_MAX_LAYERS) return DN_ERR_INVALID_ARGUMENT;
  DnLayer layers[DN_MAX_LAYERS];
  bool packed = true;
  for (int l = 0; l < n_layers; ++l) {
    layers[l] = layers_in[l];
    packed = packed && layers[l].prepacked != nullptr;
  }
  if (!packed) {
    int rc = tc_pack_layers(layers, n_layers, ws, ws_bytes, nullptr, st);
    if (rc) return rc;
  }
  // bf16 engine: bf16 MMAs when the shapes fit them (weights packed as bf16), single-pass TF32 otherwise
  const bool bf16 = passes == DN_PASSES_BF16 && layers[0].pack_fmt == 2;
  if (passes == DN_PASSES_BF16 && !bf16) passes = 1;
  if (V >= (1ll << 31) - 256) return DN_ERR_UNSUPPORTED;
  HcParams p;
  memset(&p, 0, sizeof(p));
  p.src = src;
  p.n_layers = n_layers;
  p.V = V;
  p.tile_group = layers[0].tile_group;
  p.group_stride = layers[0].group_stride;
  int nmax = 0, nmin = 1 << 30;
  bool sibling = false;
  for (int l = 0; l < n_layers; ++l) {
    const DnLayer& L = layers[l];
    HcLayer& T = p.layer[l];
    T.wpack = L.prepacked; T.bias = L.bias; T.emul = L.emul; T.relu_mask = L.relu_mask_src; T.row_scale = L.row_scale;
    T.residual = L.residual; T.ld_res = L.ld_res; T.res_scale = L.res_scale; T.out = L.out; T.ld_out = L.ld_out;
    T.K = L.K; T.N = L.N; T.relu = L.relu; T.sibling = L.sibling;
    if (L.N > nmax) nmax = L.N;
    if (L.N < nmin) nmin = L.N;
    sibling = sibling || L.sibling;
  }
  const bool wide = nmin == nmax && (nmax == 128 || nmax == 256);
  // Full-width TF32 chains of several layers at 128 without a sibling (which reads a layer's input after its epilogue)
  // or per-tile weight groups run on three consumer warpgroups over 192-row tiles when the 128-row tiles would not fit
  // in one wave on the SMs; everything else on two over 128-row tiles.  In one wave every CTA runs one tile either way,
  // and the 192-row tiles only put each tile's MMAs on fewer SMs: the training forward's MiniMLP at V = 7056 (56 tiles
  // of 128 rows, 37 of 192) made fwd_bwd slower on three.  (A build that also sent single-layer chains to three, before
  // this rule, was slower on fwd_bwd too; single-layer chains were not measured under the rule.)
  const int sms = dn_sm_count();
  const int cwg = !bf16 && wide && nmax == 128 && n_layers > 1 && !sibling && !p.tile_group && (V + 127) / 128 > sms
                      ? 3 : 2;
  const int tile_rows = 64 * cwg;
  // tensor maps (encoded on the host; a captured graph keeps them with the launch): fp32 [V rows][width], row stride
  // ld, 8-column boxes of a tile's rows; one per source of layer 0
  for (int s = 0; s < src.nsrc; ++s)
    if (!encode_tensor_map_f32(&p.amap[s], src.ptr[s], V, src.width[s], src.ld[s], 8, tile_rows, false))
      return DN_ERR_UNSUPPORTED;
  // the TF32 chains at NMAX <= 128 store each layer's out and load its residual through shared memory: one map each,
  // 8 x 64 boxes (residuals of the three-warpgroup chains: 8 x 16, one warp's rows)
  // (a column slice such as P or Q of [P|Q] is its own map: base at the slice, width N, the buffer's row stride)
  if (nmax <= 128 && !bf16)
    for (int l = 0; l < n_layers; ++l) {
      const DnLayer& L = layers[l];
      if (L.out && !encode_tensor_map_f32(&p.omap[l], L.out, V, L.N, L.ld_out, 8, OUT_ROWS, false))
        return DN_ERR_UNSUPPORTED;
      if (L.residual &&
          !encode_tensor_map_f32(&p.rmap[l], L.residual, V, L.N, L.ld_res, 8, cwg == 3 ? RES_ROWS : OUT_ROWS, false))
        return DN_ERR_UNSUPPORTED;
    }
  const DnLayer& Ll = layers[n_layers - 1];
  p.head_w = Ll.head_w; p.head_b = Ll.head_b; p.head_out = Ll.head_out; p.ld_head_out = Ll.ld_head_out; p.head_n = Ll.head_n;
  const int64_t ntiles = (V + tile_rows - 1) / tile_rows;
  const int grid = (int)(ntiles < sms ? ntiles : sms);
  if (bf16) launch_chain<MODE_BF16>(p, nmax, wide, cwg, grid, st);
  else if (passes == 3) launch_chain<MODE_TF32X3>(p, nmax, wide, cwg, grid, st);
  else launch_chain<MODE_TF32>(p, nmax, wide, cwg, grid, st);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

int tc_to_basis_supported(int K, int C) {
  if (K % 4 || K < 4 || K > 128) return DN_ERR_UNSUPPORTED;
  if (C % 16 || C < 16 || C > 128) return DN_ERR_UNSUPPORTED;
  return DN_OK;
}

int tc_to_basis_partial(const float* values, const float* basis, const float* massvec, int64_t V, int K, int C,
                        float* partial, int* P_out, int passes, cudaStream_t st, int64_t ld_values, int64_t ldp,
                        const int32_t* cta_rows, int n_ctas) {
  if (tc_to_basis_supported(K, C) != DN_OK) return DN_ERR_UNSUPPORTED;
  if (ld_values <= 0) ld_values = C;
  if (ldp <= 0) ldp = C;
  if ((reinterpret_cast<uintptr_t>(values) & 15) || (reinterpret_cast<uintptr_t>(basis) & 15) || (ld_values % 4) ||
      (ldp % 2) || (reinterpret_cast<uintptr_t>(partial) & 7))
    return DN_ERR_UNSUPPORTED;
  if (V >= (1ll << 31) - 256) return DN_ERR_UNSUPPORTED;   // TMA row coordinates are 32-bit
  TcToBasisParams p;
  memset(&p, 0, sizeof(p));
  // tensor maps (encoded on the host; a captured graph keeps them with the launch): fp32 [V rows][width], row stride
  // ld, 8 x TB_ROWS boxes; columns >= width and rows >= V are zero-filled
  const int64_t rows = V > 0 ? V : 1;
  if (!encode_tensor_map_f32(&p.phi_map, basis, rows, K, K, 8, TB_ROWS, false) ||
      !encode_tensor_map_f32(&p.x_map, values, rows, C, ld_values, 8, TB_ROWS, false))
    return DN_ERR_UNSUPPORTED;
  p.mass = massvec; p.partial = partial;
  p.ldp = ldp; p.cta_rows = cta_rows;
  p.V = V; p.K = K; p.C = C; p.chunks_per_cta = 0;
  int grid;
  if (cta_rows) {                       // batch of meshes: the caller planned the CTAs (dn_mesh_batch_plan)
    if (n_ctas < 1) return DN_ERR_INVALID_ARGUMENT;
    grid = n_ctas;
  } else {
    const int64_t total_chunks = (V + KC - 1) / KC;
    grid = dn_sm_count();
    if (total_chunks < grid) grid = (int)(total_chunks > 0 ? total_chunks : 1);
    p.chunks_per_cta = (total_chunks + grid - 1) / grid;
    if (p.chunks_per_cta < 1) p.chunks_per_cta = 1;
    grid = (int)((total_chunks + p.chunks_per_cta - 1) / p.chunks_per_cta);
    if (grid < 1) grid = 1;
  }
  if (passes == 3) launch_to_basis<MODE_TF32X3>(C / 16, grid, p, st);
  else launch_to_basis<MODE_TF32>(C / 16, grid, p, st);
  DN_LAUNCH_CHECK();
  *P_out = grid;
  return DN_OK;
}
