// The layout of a fixed-capacity batch slot planned on the device (dn_mesh_batch_plan_device, batch.BatchSlot.fill):
// from the batch's mesh ids and the dataset's per-mesh sizes, one CTA writes every table dn_mesh_batch_plan and
// batch.batch_tables build on the host, so a training step over any meshes can be captured in one CUDA graph.  One
// thread per batch mesh; row, entry and CTA starts are block scans.  The host planner's CTA count has one sequential
// rule (a running count forces one CTA per mesh near the 1024-CTA budget); when the parallel result shows that the
// rule fires, thread 0 replays the host loop.  Element kinds (faces, edges) are planned in the same launch: every mesh's
// elements start on a 128-element tile, and their vertex -> element CSR entries follow each other without gaps.
#include "dn_internal.h"

namespace {

constexpr int kThreads = 1024;       // one thread per batch mesh: at most 1024 meshes
constexpr int kMaxCtas = 1024;       // dn_mesh_batch_plan's to_basis CTA budget
enum { R_ROWS = 0, R_MESH = 1, R_PTR = 2, R_ENT = 3 };
enum { ST_OK = 0, ST_BAD_ID = 1, ST_OVER_CAPACITY = 2 };

struct PlanArgs {
  const int64_t* ids;
  // [n_dataset][size_cols]: rows, first row, gradient entries, first entry, then per element kind (count, first)
  const int64_t* sizes;
  int64_t n_dataset, V_cap, entry_cap, tail_rows;
  int n_meshes, sm_count, n_tb_ctas, n_ranges, size_cols, n_kinds, corner_range;
  dn_slot_plan out;
  dn_slot_elements kind[DN_SLOT_MAX_ELEMENT_KINDS];
};

// inclusive sum over the block's threads; *total gets the sum over all of them
__device__ int64_t block_scan(int64_t v, int64_t* warp_tot, int64_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  if (lane == 31) warp_tot[warp] = v;
  __syncthreads();
  if (warp == 0) {
    int64_t t = warp_tot[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t u = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t += u;
    }
    warp_tot[lane] = t;
  }
  __syncthreads();
  if (warp > 0) v += warp_tot[warp - 1];
  *total = warp_tot[31];
  __syncthreads();
  return v;
}

__device__ __forceinline__ void put_range(int64_t* e, int64_t src, int64_t dst, int64_t n, int64_t n_dst) {
  e[0] = src; e[1] = dst; e[2] = n; e[3] = n_dst;
}

__global__ void __launch_bounds__(kThreads) plan_kernel(const __grid_constant__ PlanArgs a) {
  __shared__ int64_t warp_tot[32];
  __shared__ int32_t s_row_begin[kThreads];
  __shared__ int32_t s_want[kThreads], s_chunks[kThreads], s_per[kThreads], s_cta_begin[kThreads + 1];
  __shared__ int s_first_bad, s_first_over, s_capped;
  const int b = threadIdx.x, B = a.n_meshes;
  if (b == 0) { s_first_bad = B; s_first_over = B; s_capped = 0; }
  __syncthreads();

  int64_t id = 0, n = 0, src_row = 0, ent = 0, src_ent = 0;
  bool id_ok = false;
  if (b < B) {
    id = a.ids[b];
    id_ok = id >= 0 && id < a.n_dataset;
    if (id_ok) {
      const int64_t* s = a.sizes + a.size_cols * id;
      n = s[0]; src_row = s[1]; ent = s[2]; src_ent = s[3];
    } else {
      atomicMin(&s_first_bad, b);
    }
  }
  int64_t padded = (n + 127) / 128 * 128, rows_total, ents_total;
  int64_t row_end = block_scan(padded, warp_tot, &rows_total);
  int64_t ent_end = block_scan(ent, warp_tot, &ents_total);
  if (b < B && (row_end > a.V_cap || ent_end > a.entry_cap)) atomicMin(&s_first_over, b);
  for (int q = 0; q < a.n_kinds; ++q) {
    const int64_t ne = id_ok ? a.sizes[a.size_cols * id + 4 + 2 * q] : 0;
    int64_t elems_total;
    const int64_t elem_end = block_scan((ne + 127) / 128 * 128, warp_tot, &elems_total);
    if (b < B && elem_end > a.kind[q].capacity) atomicMin(&s_first_over, b);
  }
  __syncthreads();
  // an invalid batch is planned with every mesh empty: nothing is read for it, every loss over it is 0 / 0
  const bool bad = s_first_bad < B || s_first_over < B;
  if (bad) id = n = src_row = ent = src_ent = padded = row_end = ent_end = rows_total = ents_total = 0;
  const int64_t row0 = row_end - padded, ent0 = ent_end - ent;
  if (b < B) s_row_begin[b] = (int32_t)row0;

  // to_basis CTAs, dn_mesh_batch_plan's rule: proportional to the mesh's 16-row chunks, at least 1, no empty CTAs
  const int64_t chunks = (n + 15) / 16;
  int64_t chunks_total;
  block_scan(chunks, warp_tot, &chunks_total);
  int64_t want = chunks_total > 0 ? (chunks * a.sm_count + chunks_total / 2) / chunks_total : 1;
  if (want < 1) want = 1;
  if (want > chunks && chunks > 0) want = chunks;
  int64_t per = chunks > 0 ? (chunks + want - 1) / want : 0;
  int64_t cnt = b < B ? (per > 0 ? (chunks + per - 1) / per : want) : 0;
  int64_t n_ctas;
  int64_t cta0 = block_scan(cnt, warp_tot, &n_ctas) - cnt;
  if (b < B && cta0 + want + (B - 1 - b) > kMaxCtas) s_capped = 1;
  if (b < B) { s_want[b] = (int32_t)want; s_chunks[b] = (int32_t)chunks; }
  __syncthreads();
  if (s_capped) {                    // the running count decides: the host loop, in mesh order
    if (b == 0) {
      int c = 0;
      for (int m = 0; m < B; ++m) {
        int64_t w = s_want[m];
        const int64_t ch = s_chunks[m];
        if (c + w + (B - 1 - m) > kMaxCtas) w = 1;
        const int64_t p = ch > 0 ? (ch + w - 1) / w : 0;
        if (p > 0) w = (ch + p - 1) / p;
        s_cta_begin[m] = c;
        s_per[m] = (int32_t)p;
        c += (int)w;
      }
      s_cta_begin[B] = c;
    }
    __syncthreads();
    if (b < B) { cta0 = s_cta_begin[b]; cnt = s_cta_begin[b + 1] - cta0; per = s_per[b]; }
    n_ctas = s_cta_begin[B];
  }

  const dn_slot_plan& o = a.out;
  if (b < B) {
    o.row_begin[b] = (int32_t)row0;
    o.mesh_cta_begin[b] = (int32_t)cta0;
    o.seg_begin[b] = (int32_t)row0;
    o.seg_rows[b] = (int32_t)n;
    const int64_t end = row0 + n;
    for (int64_t c = 0; c < cnt; ++c) {
      int64_t rb = row0 + c * per * 16, re = rb + per * 16;
      if (rb > end) rb = end;
      if (re > end) re = end;
      o.tb_rows[2 * (cta0 + c)] = (int32_t)rb;
      o.tb_rows[2 * (cta0 + c) + 1] = (int32_t)re;
    }
    // gather table: mesh b, then tail piece b (the rows past the batch's end, up to V_cap, in pieces of tail_rows:
    // padding of the last mesh, so no piece's grid is sized by the whole capacity)
    int64_t* e = a.out.table + (int64_t)b * a.n_ranges * 4;
    for (int r = 0; r < a.n_ranges; ++r) put_range(e + 4 * r, 0, 0, 0, 0);
    put_range(e + 4 * R_ROWS, src_row, row0, n, padded);
    put_range(e + 4 * R_MESH, id, b, bad ? 0 : 1, 1);
    put_range(e + 4 * R_PTR, src_row + id, row0, bad ? 0 : n + 1, padded + (b == B - 1));
    put_range(e + 4 * R_ENT, src_ent, ent0, ent, ent);
    int64_t* t = a.out.table + (int64_t)(B + b) * a.n_ranges * 4;
    const int64_t start = rows_total + b * a.tail_rows;
    int64_t len = a.V_cap - start;
    len = len < 0 ? 0 : (len > a.tail_rows ? a.tail_rows : len);
    for (int r = 0; r < a.n_ranges; ++r) put_range(t + 4 * r, 0, 0, 0, 0);
    put_range(t + 4 * R_ROWS, 0, start, 0, len);
    put_range(t + 4 * R_PTR, 0, start + 1, 0, len);        // empty rows: every pointer is the batch's entry count
    put_range(t + 4 * R_ENT, 0, ents_total, 0, 0);
    // element corners are offset by the mesh's first row and padded with it (the tail's with row 0): always a row
    if (a.n_kinds > 0) put_range(e + 4 * a.corner_range, 0, row0, 0, 0);
  }
  if (b == 0) {
    o.row_begin[B] = (int32_t)rows_total;
    o.mesh_cta_begin[B] = (int32_t)n_ctas;
    if (bad && o.status[0] == ST_OK) {               // sticky: the first invalid fill is kept until read
      const bool id_bad = s_first_bad < B;
      const int pos = id_bad ? s_first_bad : s_first_over;
      o.status[0] = id_bad ? ST_BAD_ID : ST_OVER_CAPACITY;
      o.status[1] = pos;
      o.status[2] = a.ids[pos];
    }
  }
  // CTAs past the batch's own: empty ranges, outside every mesh's [cta_begin[b], cta_begin[b + 1])
  for (int64_t c = n_ctas + b; c < a.n_tb_ctas; c += kThreads) {
    o.tb_rows[2 * c] = (int32_t)rows_total;
    o.tb_rows[2 * c + 1] = (int32_t)rows_total;
  }
  __syncthreads();
  // tiles: the mesh whose padded rows hold them (the tail: the last mesh); segments cover the batch's tiles only
  for (int64_t tile = b; tile < a.V_cap / 128; tile += kThreads) {
    const int64_t r = tile * 128;
    int lo = 0, hi = B - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) / 2;
      if (s_row_begin[mid] <= r) lo = mid; else hi = mid - 1;
    }
    o.tile_mesh[tile] = lo;
    o.tile_seg[tile] = r < rows_total ? lo : -1;
  }
  // element kinds: mesh b's elements at a 128-aligned begin, padded to its tile end; its CSR entries right after the
  // previous mesh's (so no vertex's entry range crosses a padding element); the tail pieces pad [total, capacity)
  for (int q = 0; q < a.n_kinds; ++q) {
    const dn_slot_elements& k = a.kind[q];
    int64_t ne = 0, src_el = 0;
    if (b < B && !bad) {
      const int64_t* s = a.sizes + a.size_cols * id + 4 + 2 * q;
      ne = s[0]; src_el = s[1];
    }
    const int64_t pe = (ne + 127) / 128 * 128, nc = ne * k.k;
    int64_t elems_total, corners_total;
    const int64_t e0 = block_scan(pe, warp_tot, &elems_total) - pe;
    const int64_t c0 = block_scan(nc, warp_tot, &corners_total) - nc;
    if (b < B) {
      s_row_begin[b] = (int32_t)e0;
      k.begin[b] = (int32_t)e0;
      k.count[b] = (int32_t)ne;
      int64_t* e = a.out.table + (int64_t)b * a.n_ranges * 4;
      put_range(e + 4 * k.range, src_el, e0, ne, pe);
      put_range(e + 4 * k.csr_range, src_el * k.k, c0, nc, nc);
      int64_t* t = a.out.table + (int64_t)(B + b) * a.n_ranges * 4;
      const int64_t start = elems_total + b * k.tail;
      int64_t len = k.capacity - start;
      len = len < 0 ? 0 : (len > k.tail ? k.tail : len);
      put_range(t + 4 * k.range, 0, start, 0, len);
      put_range(t + 4 * k.csr_range, 0, corners_total, 0, 0);
    }
    if (b == 0) k.begin[B] = (int32_t)elems_total;
    __syncthreads();
    for (int64_t tile = b; tile < k.capacity / 128; tile += kThreads) {
      const int64_t r = tile * 128;
      int lo = 0, hi = B - 1;
      while (lo < hi) {
        const int mid = (lo + hi + 1) / 2;
        if (s_row_begin[mid] <= r) lo = mid; else hi = mid - 1;
      }
      k.tile_seg[tile] = r < elems_total ? lo : -1;
    }
    __syncthreads();
  }
}

}  // namespace

int launch_mesh_batch_plan_device(const int64_t* ids, int n_meshes, const int64_t* sizes, int size_cols,
                                  int64_t n_dataset, int sm_count, int64_t V_cap, int64_t entry_cap, int n_tb_ctas,
                                  int64_t tail_rows, int n_ranges, const dn_slot_plan& out,
                                  const dn_slot_elements* kinds, int n_kinds, int corner_range, cudaStream_t st) {
  PlanArgs a = {};
  a.ids = ids; a.sizes = sizes; a.n_dataset = n_dataset;
  a.V_cap = V_cap; a.entry_cap = entry_cap; a.tail_rows = tail_rows;
  a.n_meshes = n_meshes; a.sm_count = sm_count; a.n_tb_ctas = n_tb_ctas; a.n_ranges = n_ranges;
  a.size_cols = size_cols; a.n_kinds = n_kinds; a.corner_range = corner_range;
  a.out = out;
  for (int q = 0; q < n_kinds; ++q) a.kind[q] = kinds[q];
  plan_kernel<<<1, kThreads, 0, st>>>(a);
  DN_LAUNCH_CHECK();
  return DN_OK;
}
