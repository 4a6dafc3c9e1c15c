// A mesh batch gathered from a device-resident dataset (dn_batch_gather, batch.MeshDataset.batch): one launch writes
// every array of the batch.  Grid: x runs over the CTAs of every part (part p owns x in [cta_begin[p],
// cta_begin[p + 1])), y over the batch's meshes; the CTAs of (part, mesh) stride over that mesh's units of the part.
// Two routines serve every array: a word copy with zero padding (per-row data, CSR values, eigenvalues) and an integer
// copy that adds the mesh's offset and pads with offset + count (column indices, element corners, row pointers).
#include "dn_internal.h"

namespace {

constexpr int kThreads = 256;
constexpr int kUnroll = 4;
constexpr int64_t kWordsPerCta = (int64_t)kThreads * kUnroll * 2;

struct GatherArgs {
  dn_gather_part part[DN_GATHER_MAX_PARTS];
  int32_t cta_begin[DN_GATHER_MAX_PARTS + 1];
  int32_t n_parts;
  int32_t n_ranges;
  const int64_t* table;
};

// dst[i] = i < n ? f(src[i]) : pad for i in [0, total), by `stride` threads starting at i0, kUnroll loads in flight
template <typename T, typename F>
__device__ __forceinline__ void gather_units(const T* __restrict__ src, T* __restrict__ dst, int64_t n, int64_t total,
                                             T pad, int64_t i0, int64_t stride, F f) {
  for (int64_t i = i0; i < total; i += kUnroll * stride) {
    T v[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const int64_t j = i + u * stride;
      v[u] = j < n ? f(__ldg(src + j)) : pad;
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const int64_t j = i + u * stride;
      if (j < total) dst[j] = v[u];
    }
  }
}

__global__ void __launch_bounds__(kThreads) batch_gather_kernel(const __grid_constant__ GatherArgs a) {
  int p = 0;
  while (p + 1 < a.n_parts && (int)blockIdx.x >= a.cta_begin[p + 1]) ++p;
  const dn_gather_part& P = a.part[p];
  const int64_t* r = a.table + ((int64_t)blockIdx.y * a.n_ranges + P.range) * 4;
  const int64_t w = P.width;
  const int64_t n_dst = r[3] * w;
  const int64_t n = (r[2] < r[3] ? r[2] : r[3]) * w;
  const int64_t stride = (int64_t)(a.cta_begin[p + 1] - a.cta_begin[p]) * kThreads;
  const int64_t i0 = (int64_t)(blockIdx.x - a.cta_begin[p]) * kThreads + threadIdx.x;
  if (P.op == DN_GATHER_COPY) {
    gather_units(static_cast<const uint32_t*>(P.src) + r[0] * w, static_cast<uint32_t*>(P.dst) + r[1] * w, n, n_dst,
                 0u, i0, stride, [](uint32_t x) { return x; });
    return;
  }
  const int64_t* o = a.table + ((int64_t)blockIdx.y * a.n_ranges + P.offset_range) * 4;
  const int64_t off = o[1];
  if (P.op == DN_GATHER_ADD_I32) {
    gather_units(static_cast<const int32_t*>(P.src) + r[0] * w, static_cast<int32_t*>(P.dst) + r[1] * w, n, n_dst,
                 (int32_t)(off + o[2]), i0, stride, [off](int32_t x) { return (int32_t)(x + off); });
  } else {
    gather_units(static_cast<const int64_t*>(P.src) + r[0] * w, static_cast<int64_t*>(P.dst) + r[1] * w, n, n_dst,
                 off + o[2], i0, stride, [off](int64_t x) { return x + off; });
  }
}

}  // namespace

int launch_batch_gather(const dn_gather_part* parts, int n_parts, const int64_t* table, int n_ranges, int n_meshes,
                        cudaStream_t st) {
  GatherArgs a;
  a.n_parts = n_parts;
  a.n_ranges = n_ranges;
  a.table = table;
  int64_t ctas = 0;
  for (int p = 0; p < n_parts; ++p) {
    a.part[p] = parts[p];
    a.cta_begin[p] = (int32_t)ctas;
    const int64_t words = parts[p].max_units * parts[p].width * (parts[p].op == DN_GATHER_ADD_I64 ? 2 : 1);
    int64_t c = (words + kWordsPerCta - 1) / kWordsPerCta;
    ctas += c < 1 ? 1 : (c > 4096 ? 4096 : c);
  }
  a.cta_begin[n_parts] = (int32_t)ctas;
  batch_gather_kernel<<<dim3((unsigned)ctas, (unsigned)n_meshes), kThreads, 0, st>>>(a);
  DN_LAUNCH_CHECK();
  return DN_OK;
}
