// C-ABI entry points (include/diffusion_net_b200.h).  Argument checking, workspace carving and
// the kernel sequence of each reference function; no torch types, no hidden synchronisation.
#include "dn_internal.h"
#include <stdio.h>
#include <stdlib.h>
#include <vector>
#include <string.h>

namespace {

struct Bump {
  char* base;
  int64_t size, off;
  Bump(void* p, int64_t n) : base(static_cast<char*>(p)), size(n), off(0) {}
  float* take(int64_t floats) {
    const int64_t bytes = (floats * 4 + 255) / 256 * 256;
    if (!base || off + bytes > size) return nullptr;
    float* r = reinterpret_cast<float*>(base + off);
    off += bytes;
    return r;
  }
  int64_t left_floats() const { return (size - off) / 4; }
};

constexpr int64_t kPartialFloats = 16ll << 20;  // 64 MiB split-V partial sums

// The engine of one C-ABI call: tensor cores (with their pass count) or the exact SIMT kernels throughout.
struct Engine {
  bool tc;
  int passes;
};

// A tensor-core engine on a device without the tensor-core kernels is an error (DN_ERR_NOT_SM100): there is no
// multi-backend dispatch.  Every entry point that dispatches resolves its engine once, before it enqueues any work.
int resolve(int engine, Engine* e) {
  e->tc = engine == DN_ENGINE_TC3X || engine == DN_ENGINE_TC1X || engine == DN_ENGINE_BF16;
  e->passes = engine == DN_ENGINE_TC1X ? 1 : (engine == DN_ENGINE_BF16 ? DN_PASSES_BF16 : 3);
  return e->tc && !tc_supported_device() ? DN_ERR_NOT_SM100 : DN_OK;
}

// A tensor-core engine was requested but this contraction is outside the wgmma kernels' envelope and runs the exact
// fp32 SIMT kernel instead (same result class or better, slower).  Said once per shape on stderr; DN_STRICT_TC=1 turns
// it into DN_ERR_UNSUPPORTED so that a deployment never runs the slow path unnoticed.
int note_simt_fallback(const char* what, int K, int N) {
  static int strict = -1;
  if (strict < 0) { const char* e = getenv("DN_STRICT_TC"); strict = (e && atoi(e)) ? 1 : 0; }
  static int seen[64][2];
  static int nseen = 0;
  bool first = true;
  for (int i = 0; i < nseen; ++i) if (seen[i][0] == K && seen[i][1] == N) first = false;
  if (first && nseen < 64) {
    seen[nseen][0] = K; seen[nseen][1] = N; ++nseen;
    fprintf(stderr, "diffusion_net_b200: %s with K=%d, N=%d is outside the tensor-core kernels' envelope; running the exact "
                    "fp32 SIMT kernel%s\n", what, K, N, strict ? " is refused (DN_STRICT_TC=1)" : "");
  }
  return strict ? DN_ERR_UNSUPPORTED : DN_OK;
}

inline DnLayer make_layer(const float* W, int64_t ldw, int w_trans, const float* bias, int relu, int K, int N,
                          float* out, int64_t ld_out) {
  DnLayer L;
  memset(&L, 0, sizeof(L));
  L.W = W; L.ldw = ldw; L.w_trans = w_trans; L.bias = bias; L.relu = relu; L.K = K; L.N = N;
  L.out = out; L.ld_out = ld_out; L.res_scale = 1.f;
  return L;
}

inline DnRowsSrc one_src(const float* p, int width, int64_t ld) {
  DnRowsSrc s;
  memset(&s, 0, sizeof(s));
  s.ptr[0] = p; s.width[0] = width; s.ld[0] = ld; s.nsrc = 1;
  return s;
}

// One layer on the exact SIMT kernel.  simt_rows_gemm takes every layer but a w_trans one with a second weight block
// (grad_x = dP A_re + dQ A_im over the sources dP | dQ): that runs as two passes, the second adding the first's output
// as its residual, which is exact only for a layer without bias or activation.
int simt_layer(const DnRowsSrc& src, const DnLayer& L, int64_t V, cudaStream_t st) {
  if (!L.w_trans || !L.W2) return simt_rows_gemm(src, L, V, st);
  if (src.nsrc != 2 || src.width[0] != L.n_split || L.bias || L.relu || L.emul || L.relu_mask_src || L.row_scale)
    return DN_ERR_UNSUPPORTED;
  DnLayer L0 = L;
  L0.W2 = nullptr; L0.n_split = 0; L0.K = L.n_split;
  int rc = simt_rows_gemm(one_src(src.ptr[0], src.width[0], src.ld[0]), L0, V, st);
  if (rc) return rc;
  DnLayer L1 = L0;
  L1.W = L.W2; L1.K = L.K - L.n_split; L1.residual = L.out; L1.ld_res = L.ld_out; L1.res_scale = 1.f;
  return simt_rows_gemm(one_src(src.ptr[1], src.width[1], src.ld[1]), L1, V, st);
}

// The one way dense layers run.  The chain is one fused tensor-core launch when rows_chain_kernel takes it whole (a
// chain whose weights the caller packed, the caller planned).  Otherwise it runs layer by layer, each on the tensor-core
// kernel when its shape allows and on the exact SIMT kernel otherwise; layers without `out` then write two V x N
// ping-pong buffers carved from ws.  The rest of ws is where the tensor-core kernel packs weights.
int run_chain(const DnRowsSrc& src, DnLayer* layers, int n_layers, int64_t V, Engine e, Bump ws, cudaStream_t st) {
  if (e.tc && (layers[0].prepacked || tc_chain_plan(src, layers, n_layers, e.passes) >= 0))
    return tc_rows_chain(src, layers, n_layers, V, e.passes, ws.base + ws.off, ws.size - ws.off, st);
  // not fusable as a whole (e.g. a 256-wide layer inside a chain)
  float* tmp[2] = {nullptr, nullptr};
  int maxn = 0;
  bool need_tmp = false;
  for (int l = 0; l < n_layers; ++l) {
    if (layers[l].N > maxn) maxn = layers[l].N;
    need_tmp = need_tmp || !layers[l].out;
  }
  if (need_tmp) {
    tmp[0] = ws.take(V * maxn);
    tmp[1] = ws.take(V * maxn);
    if (!tmp[0] || !tmp[1]) return DN_ERR_WORKSPACE;
  }
  DnRowsSrc cur = src;
  for (int l = 0; l < n_layers; ++l) {
    DnLayer L = layers[l];
    // a sibling reads the same input as the layer before it: its own output must not overwrite that input
    if (L.sibling && (l == 0 || !L.out)) return DN_ERR_UNSUPPORTED;
    L.sibling = 0;
    if (!L.out) { L.out = tmp[l & 1]; L.ld_out = L.N; }
    int rc;
    // (a single layer was planned above)
    if (e.tc && n_layers > 1 && tc_chain_plan(cur, &L, 1, e.passes) >= 0)
      rc = tc_rows_chain(cur, &L, 1, V, e.passes, ws.base + ws.off, ws.size - ws.off, st);
    else if (e.tc && (rc = note_simt_fallback("a dense layer", L.K, L.N)))
      return rc;
    else
      rc = simt_layer(cur, L, V, st);
    if (rc) return rc;
    if (!(l + 1 < n_layers && layers[l + 1].sibling)) cur = one_src(L.out, L.N, L.ld_out);
  }
  return DN_OK;
}

// partial[p][k][c] = sum over the rows of split p of basis[v][k] * (mass[v] * values[v][c]), p < *P.  `batch`
// (optional) is a mesh batch's CTA plan: CTA p reduces rows tb_rows[2p] .. tb_rows[2p + 1], on tensor cores only.
int to_basis_partials(const float* values, const float* basis, const float* massvec, int64_t V, int K, int C,
                      float* partial, int64_t partial_floats, int* P, Engine e, cudaStream_t st,
                      const dn_mesh_batch* batch = nullptr) {
  const int32_t* rows = batch ? batch->tb_rows : nullptr;
  const int ctas = batch ? batch->n_tb_ctas : dn_sm_count();
  if (e.tc && (int64_t)ctas * K * C <= partial_floats) {
    if (tc_to_basis_supported(K, C) == DN_OK)
      return tc_to_basis_partial(values, basis, massvec, V, K, C, partial, P, e.passes, st, 0, 0, rows, ctas);
    // wider than one accumulator set (C_width = 256): 128-column slices, each its own launch into the shared partials
    if (C > 128 && C % 128 == 0 && tc_to_basis_supported(K, 128) == DN_OK) {
      for (int c0 = 0; c0 < C; c0 += 128) {
        const int rc = tc_to_basis_partial(values + c0, basis, massvec, V, K, 128, partial + c0, P, e.passes, st, C, C,
                                           rows, ctas);
        if (rc) return rc;
      }
      return DN_OK;
    }
  }
  if (batch) return DN_ERR_UNSUPPORTED;   // mesh batches have no SIMT route
  if (e.tc) { const int rc = note_simt_fallback("to_basis", K, C); if (rc) return rc; }
  return simt_atb_partial_st(basis, K, K, values, C, C, massvec, V, partial, partial_floats, P, st);
}

// out[i][j] (ld_out) (+)= sum_v A[v][i] * B[v][j]   (weight gradients: A = dz, B = layer input).
// Tensor cores (the split-V to_basis kernel, reference geometry.py:572-583 has the same contraction) when both
// operands are contiguous and at most 128 wide; the exact SIMT kernel otherwise.
int atb(const float* A, int64_t lda, int I, const float* B, int64_t ldb, int J, int64_t V, float* out, int64_t ld_out,
        int accumulate, float* part, int64_t part_floats, Engine e, cudaStream_t st) {
  if (e.tc && lda == I && ldb == J && tc_to_basis_supported(I, J) == DN_OK &&
      (int64_t)dn_sm_count() * I * J <= part_floats) {
    int P = 0;
    int rc = tc_to_basis_partial(B, A, nullptr, V, I, J, part, &P, e.passes, st);
    if (rc == DN_OK) return launch_reduce_partials(part, P, nullptr, 1, I, J, out, ld_out, accumulate, st);
    if (rc != DN_ERR_UNSUPPORTED) return rc;
  }
  if (e.tc) { const int rc = note_simt_fallback("a weight gradient", I, J); if (rc) return rc; }
  return simt_atb(A, lda, I, B, ldb, J, nullptr, V, out, ld_out, accumulate, part, part_floats, st);
}

// Plan and scratch of a spectral diffusion over a mesh batch (dn_learned_time_diffusion_{fwd,bwd}_batched): grouped
// to_basis partials -> one pack launch forming every mesh's multiplier -> the from_basis chain picking its matrix per
// tile.  The envelope is dn_block_fwd_batched's (tensor-core engine, V a multiple of 128, a planned batch, a from_basis
// layer the fused chain takes); everything is checked and carved before any work is enqueued.
struct BatchedSpectral {
  Engine e;
  DnRowsSrc src;       // evecs
  DnLayer L;           // from_basis, packed once per mesh by tc_pack_layers
  float* partial;      // [n_tb_ctas][K][C]
  int64_t pf;
  float* packed;
  int64_t packed_bytes;
  float* sums;         // [n_meshes][K][C]
};

int batched_spectral_plan(const dn_mesh_batch* batch, const float* evecs, int64_t V, int K, int C, int engine,
                          float* out, Bump& ws, BatchedSpectral* b) {
  int rc = resolve(engine, &b->e);
  if (rc) return rc;
  if (!b->e.tc || (V % 128) || batch->n_meshes < 1 || !batch->tile_mesh || !batch->tb_rows || !batch->mesh_cta_begin ||
      batch->n_tb_ctas < 1)
    return DN_ERR_UNSUPPORTED;
  const bool tb = tc_to_basis_supported(K, C) == DN_OK ||
                  (C > 128 && C % 128 == 0 && tc_to_basis_supported(K, 128) == DN_OK);
  b->src = one_src(evecs, K, K);
  b->L = make_layer(nullptr, C, 1, nullptr, 0, K, C, out, C);
  if (!tb || tc_chain_plan(b->src, &b->L, 1, b->e.passes) < 0) return DN_ERR_UNSUPPORTED;
  b->pf = (int64_t)batch->n_tb_ctas * K * C;
  b->packed_bytes = tc_chain_ws_bytes(&b->L, 1, batch->n_meshes);
  b->partial = ws.take(b->pf);
  b->packed = ws.take(b->packed_bytes / 4);
  b->sums = ws.take((int64_t)batch->n_meshes * K * C);
  return (b->partial && b->packed && b->sums) ? DN_OK : DN_ERR_WORKSPACE;
}

}  // namespace

long long g_dn_launches = 0;

extern "C" {

int dn_abi_version(void) { return DN_ABI_VERSION; }

int64_t dn_kernel_launch_count(void) { return (int64_t)g_dn_launches; }

const char* dn_error_string(int code) {
  switch (code) {
    case DN_OK: return "ok";
    case DN_ERR_INVALID_ARGUMENT: return "diffusion_net_b200: invalid argument";
    case DN_ERR_UNSUPPORTED: return "diffusion_net_b200: unsupported shape/engine";
    case DN_ERR_WORKSPACE: return "diffusion_net_b200: workspace too small (see dn_workspace_bytes)";
    case DN_ERR_NOT_SM100: return "diffusion_net_b200: tensor-core engine needs an sm_90 (H100) GPU";
    default: break;
  }
  if (code > 0) return cudaGetErrorString(static_cast<cudaError_t>(code));
  return "diffusion_net_b200: unknown error";
}

int dn_device_query(int device, int* sm_count, int* cc, int64_t* smem_optin_bytes) {
  cudaDeviceProp p;
  DN_CUDA_TRY(cudaGetDeviceProperties(&p, device));
  if (sm_count) *sm_count = p.multiProcessorCount;
  if (cc) *cc = p.major * 10 + p.minor;
  if (smem_optin_bytes) *smem_optin_bytes = (int64_t)p.sharedMemPerBlockOptin;
  return DN_OK;
}

int64_t dn_workspace_bytes(int64_t V, int K, int C) {
  if (V < 0 || K < 0 || C <= 0) return -1;
  const int64_t vc = ((V + 127) / 128 * 128) * (int64_t)C * 4;
  return kPartialFloats * 4 + 14 * (vc + 256) + (8ll << 20) + (int64_t)K * C * 16;
}

int dn_csr_from_coo(const int64_t* rows, const int64_t* cols, const float* vx, const float* vy, int64_t nnz,
                    int64_t V, int32_t* rowptr, int32_t* colidx, float* vals, dn_stream_t stream) {
  if (nnz < 0 || V < 0 || !rowptr || (nnz > 0 && (!rows || !cols || !vx || !colidx || !vals)))
    return DN_ERR_INVALID_ARGUMENT;
  if (nnz >= (1ll << 31) || V >= (1ll << 31)) return DN_ERR_UNSUPPORTED;
  return launch_csr_from_coo(rows, cols, vx, vy, nnz, V, rowptr, colidx, vals, (cudaStream_t)stream);
}

int64_t dn_patch_build(int64_t V, const int32_t* rowptr, const int32_t* colidx, int max_targets, int max_src,
                       int32_t* tgt_ptr, int32_t* tgt, int32_t* src_ptr, int32_t* src_rows, int32_t* ent_ptr,
                       uint8_t* lcol, int32_t* perm, int32_t* max_src_out) {
  if (V < 0 || !rowptr || max_targets < 1 || max_src < 1 || max_src > 256 || !tgt_ptr || !tgt || !src_ptr ||
      !ent_ptr || !max_src_out || (V > 0 && rowptr[V] > 0 && (!colidx || !src_rows || !lcol || !perm)))
    return DN_ERR_INVALID_ARGUMENT;
  if (V >= (1ll << 31) - 1) return DN_ERR_UNSUPPORTED;
  // state: 0 free, 1 queued by the patch being grown, 2 assigned
  std::vector<int32_t> stamp((size_t)V, -1), lidx((size_t)V, 0), seeds, q;
  std::vector<uint8_t> state((size_t)V, 0);
  size_t seed_head = 0;
  int64_t scan = 0, np = 0, nt = 0, nsr = 0, ne = 0;
  int32_t worst = 0;
  tgt_ptr[0] = 0; src_ptr[0] = 0; ent_ptr[0] = 0;
  while (nt < V) {
    int32_t s = -1;
    while (seed_head < seeds.size()) {                       // prefer a vertex next to an earlier patch
      const int32_t c = seeds[seed_head++];
      if (state[c] == 0) { s = c; break; }
    }
    if (s < 0) {
      while (state[scan] != 0) ++scan;
      s = (int32_t)scan;
    }
    q.clear();
    q.push_back(s);
    state[s] = 1;
    size_t qh = 0;
    int nsrc = 0, ntg = 0;
    while (qh < q.size() && ntg < max_targets) {
      const int32_t v = q[qh++];
      const int32_t rs = rowptr[v], re = rowptr[v + 1];
      if (re - rs > max_src) return DN_ERR_UNSUPPORTED;
      int newc = 0;
      for (int32_t e = rs; e < re; ++e) newc += (stamp[colidx[e]] != (int32_t)np);
      if (nsrc + newc > max_src) {                           // does not fit here: a later patch takes it
        state[v] = 0;
        seeds.push_back(v);
        continue;
      }
      state[v] = 2;
      tgt[nt++] = v;
      ++ntg;
      for (int32_t e = rs; e < re; ++e) {
        const int32_t c = colidx[e];
        if (stamp[c] != (int32_t)np) {
          stamp[c] = (int32_t)np;
          lidx[c] = nsrc++;
          src_rows[nsr++] = c;
        }
        lcol[ne] = (uint8_t)lidx[c];
        perm[ne] = e;
        ++ne;
      }
      ent_ptr[nt] = (int32_t)ne;
      for (int32_t e = rs; e < re; ++e) {
        const int32_t c = colidx[e];
        if (c < V && state[c] == 0) { state[c] = 1; q.push_back(c); }
      }
    }
    for (; qh < q.size(); ++qh) {                            // frontier we did not get to: seeds of the next patches
      const int32_t v = q[qh];
      if (state[v] == 1) { state[v] = 0; seeds.push_back(v); }
    }
    if (nsrc > worst) worst = nsrc;
    ++np;
    tgt_ptr[np] = (int32_t)nt;
    src_ptr[np] = (int32_t)nsr;
  }
  *max_src_out = worst;
  return np;
}

int dn_csr_transpose(const dn_csr* in, int64_t V, int32_t* rowptr_out, int32_t* colidx_out, float* vals_out,
                     void* workspace, int64_t ws_bytes, dn_stream_t stream) {
  if (!in || V < 0 || in->nnz < 0 || !rowptr_out || (in->nnz > 0 && (!in->rowptr || !in->colidx || !in->vals ||
                                                                        !colidx_out || !vals_out)))
    return DN_ERR_INVALID_ARGUMENT;
  if (in->nnz >= (1ll << 31) || V >= (1ll << 31) - 1) return DN_ERR_UNSUPPORTED;
  if (in->nnz > 0 && (!workspace || ws_bytes < (int64_t)sizeof(int32_t) * V)) return DN_ERR_WORKSPACE;
  return launch_csr_transpose(in, V, rowptr_out, colidx_out, vals_out, (int32_t*)workspace, (cudaStream_t)stream);
}

int dn_build_grad(const float* verts, const float* frames, const float* edge_tangent, const int64_t* edges, int64_t E,
                  int64_t V, int32_t* rowptr_out, int32_t* colidx_out, float* vals_out, void* workspace, int64_t ws_bytes,
                  dn_stream_t stream) {
  if (V < 0 || E < 0 || !rowptr_out || (V > 0 && (!colidx_out || !vals_out)) || (E > 0 && !edges) ||
      (E > 0 && !edge_tangent && (!verts || !frames)))
    return DN_ERR_INVALID_ARGUMENT;
  if (E + V >= (1ll << 31) || V >= (1ll << 31) - 1) return DN_ERR_UNSUPPORTED;
  if (V > 0 && (!workspace || ws_bytes < (int64_t)sizeof(int32_t) * V)) return DN_ERR_WORKSPACE;
  return launch_build_grad(verts, frames, edge_tangent, edges, E, V, rowptr_out, colidx_out, vals_out, (int32_t*)workspace,
                           (cudaStream_t)stream);
}

int dn_mesh_laplacian(const double* verts, const int64_t* faces, int64_t F, int64_t V, double eps, int32_t* rowptr_out,
                      int32_t* colidx_out, double* L_vals_out, double* mass_out, double* A_vals_out, double* A_diag_out,
                      double* bound_out, int32_t* nan_out, void* workspace, int64_t ws_bytes, dn_stream_t stream) {
  if (V < 0 || F < 0 || !rowptr_out || !bound_out || !nan_out || (F > 0 && (!faces || !verts)) ||
      (V > 0 && (!colidx_out || !L_vals_out || !mass_out)))
    return DN_ERR_INVALID_ARGUMENT;
  if (6 * F + V >= (1ll << 31) || V >= (1ll << 31) - 1) return DN_ERR_UNSUPPORTED;
  if (V > 0 && (!workspace || ws_bytes < mesh_laplacian_ws_bytes(F, V))) return DN_ERR_WORKSPACE;
  return launch_mesh_laplacian(verts, faces, F, V, eps, rowptr_out, colidx_out, L_vals_out, mass_out, A_vals_out,
                               A_diag_out, bound_out, nan_out, workspace, (cudaStream_t)stream);
}

int dn_vertex_frames(const double* verts, const int64_t* faces, int64_t F, int64_t V, const double* normals_in,
                     double* normals_out, double* frames_out, int32_t* n_bad_out, void* workspace, int64_t ws_bytes,
                     dn_stream_t stream) {
  if (V < 0 || F < 0 || !n_bad_out || (V > 0 && !frames_out) ||
      (!normals_in && V > 0 && (!normals_out || (F > 0 && (!faces || !verts)))))
    return DN_ERR_INVALID_ARGUMENT;
  if (3 * F >= (1ll << 31) || V >= (1ll << 31) - 1) return DN_ERR_UNSUPPORTED;
  if (!normals_in && V > 0 && (!workspace || ws_bytes < vertex_frames_ws_bytes(F, V))) return DN_ERR_WORKSPACE;
  return launch_vertex_frames(verts, faces, F, V, normals_in, normals_out, frames_out, n_bad_out, workspace,
                              (cudaStream_t)stream);
}

int dn_eig_filter(const int32_t* rowptr, const int32_t* colidx, const double* A_vals, const double* A_diag, int64_t V,
                  int n, const double* Y, const double* Y_prev, int64_t ld, double alpha, double beta, double gamma,
                  double* Y_out, dn_stream_t stream) {
  if (V < 0 || n < 0 || ld < n || (V > 0 && n > 0 && (!rowptr || !colidx || !A_vals || !A_diag || !Y || !Y_out)) ||
      (Y_out && (Y_out == Y || Y_out == Y_prev)))
    return DN_ERR_INVALID_ARGUMENT;
  return launch_eig_filter(rowptr, colidx, A_vals, A_diag, V, n, Y, Y_prev, ld, alpha, beta, gamma, Y_out,
                           (cudaStream_t)stream);
}

int dn_eig_gram(const double* X, int64_t ldx, const double* Y, int64_t ldy, int64_t V, int m, int n, double* out,
                void* workspace, int64_t ws_bytes, dn_stream_t stream) {
  if (V < 0 || m < 0 || n < 0 || ldx < m || ldy < n || (m > 0 && n > 0 && (!out || (V > 0 && (!X || !Y)))))
    return DN_ERR_INVALID_ARGUMENT;
  if (m > 0 && n > 0 && V > 0 && (!workspace || ws_bytes < eig_gram_ws_bytes(V, m, n))) return DN_ERR_WORKSPACE;
  return launch_eig_gram(X, ldx, Y, ldy, V, m, n, out, (double*)workspace, (cudaStream_t)stream);
}

int dn_eig_rotate(const double* X, int64_t ldx, const double* C, int64_t ldc, int64_t V, int kd, int n, double beta,
                  double* Z, int64_t ldz, dn_stream_t stream) {
  if (V < 0 || kd < 0 || n < 0 || ldx < kd || ldc < n || ldz < n || (V > 0 && n > 0 && (!Z || (kd > 0 && (!X || !C)))) ||
      (Z && Z == X))
    return DN_ERR_INVALID_ARGUMENT;
  return launch_eig_rotate(X, ldx, C, ldc, V, kd, n, beta, Z, ldz, (cudaStream_t)stream);
}

int dn_eig_residual_norms(const double* W, int64_t ldw, const double* Q, int64_t ldq, const double* theta, int64_t V,
                          int n, double* out, void* workspace, int64_t ws_bytes, dn_stream_t stream) {
  if (V < 0 || n < 0 || ldw < n || ldq < n || (n > 0 && (!out || !theta || (V > 0 && (!W || !Q)))))
    return DN_ERR_INVALID_ARGUMENT;
  if (n > 0 && V > 0 && (!workspace || ws_bytes < eig_resid_ws_bytes(V, n))) return DN_ERR_WORKSPACE;
  return launch_eig_residual_norms(W, ldw, Q, ldq, theta, V, n, out, (double*)workspace, (cudaStream_t)stream);
}

int dn_eig_finalize(const double* Y, int64_t ldy, const int32_t* cols, int k, const double* mass, int64_t V, double* out,
                    void* workspace, int64_t ws_bytes, dn_stream_t stream) {
  if (V < 0 || k < 0 || (V > 0 && k > 0 && (!Y || !cols || !mass || !out)))
    return DN_ERR_INVALID_ARGUMENT;
  if (V > 0 && k > 0 && (!workspace || ws_bytes < 8ll * k)) return DN_ERR_WORKSPACE;
  return launch_eig_finalize(Y, ldy, cols, k, mass, V, out, (double*)workspace, (cudaStream_t)stream);
}

int dn_mesh_laplacian_batched(const double* verts, const int64_t* faces, int64_t F, int64_t V, int n_meshes,
                              const int32_t* row_begin, double eps, int32_t* rowptr_out, int32_t* colidx_out,
                              double* L_vals_out, double* mass_out, double* A_vals_out, double* A_diag_out,
                              double* bound_out, int32_t* nan_out, void* workspace, int64_t ws_bytes, dn_stream_t stream) {
  if (V < 0 || F < 0 || n_meshes < 0 || !rowptr_out || (n_meshes > 0 && (!row_begin || !bound_out || !nan_out)) ||
      (F > 0 && (!faces || !verts)) || (V > 0 && (n_meshes == 0 || !colidx_out || !L_vals_out || !mass_out)))
    return DN_ERR_INVALID_ARGUMENT;
  if (6 * F + V >= (1ll << 31) || V >= (1ll << 31) - 1) return DN_ERR_UNSUPPORTED;
  if (V > 0 && (!workspace || ws_bytes < mesh_laplacian_ws_bytes(F, V))) return DN_ERR_WORKSPACE;
  return launch_mesh_laplacian_batched(verts, faces, F, V, n_meshes, row_begin, eps, rowptr_out, colidx_out, L_vals_out,
                                       mass_out, A_vals_out, A_diag_out, bound_out, nan_out, workspace,
                                       (cudaStream_t)stream);
}

static bool eig_batch_ok(const dn_eig_batch* bt) {
  return bt && bt->n_meshes >= 0 && bt->n_tiles >= 0 && bt->n_slices >= 0 && bt->n_slices <= 65535 &&
         (bt->n_meshes == 0 || (bt->n_meshes <= 65535 && bt->row_begin && bt->tile_begin && bt->slice_begin)) &&
         (bt->n_tiles == 0 || bt->tile_mesh) && (bt->n_slices == 0 || bt->slice_mesh);
}

int dn_eig_filter_batched(const int32_t* rowptr, const int32_t* colidx, const double* A_vals, const double* A_diag,
                          const dn_eig_batch* batch, int n, const double* Y, const double* Y_prev, int64_t ld,
                          const double* alpha, const double* beta, const double* gamma, const int32_t* active,
                          double* Y_out, dn_stream_t stream) {
  if (!eig_batch_ok(batch) || n < 0 || ld < n ||
      (batch->n_tiles > 0 && n > 0 && (!rowptr || !colidx || !A_vals || !A_diag || !Y || !Y_out || !alpha || !beta || !gamma)) ||
      (Y_out && (Y_out == Y || Y_out == Y_prev)))
    return DN_ERR_INVALID_ARGUMENT;
  if ((int64_t)batch->n_tiles * 8 >= (1ll << 31)) return DN_ERR_UNSUPPORTED;
  return launch_eig_filter_batched(rowptr, colidx, A_vals, A_diag, batch, n, Y, Y_prev, ld, alpha, beta, gamma, active,
                                   Y_out, (cudaStream_t)stream);
}

int dn_eig_gram_batched(const double* X, int64_t ldx, const double* Y, int64_t ldy, const dn_eig_batch* batch, int m, int n,
                        const int32_t* active, double* out, void* workspace, int64_t ws_bytes, dn_stream_t stream) {
  if (!eig_batch_ok(batch) || m < 0 || n < 0 || ldx < m || ldy < n ||
      (m > 0 && n > 0 && batch->n_meshes > 0 && (!out || (batch->n_tiles > 0 && (!X || !Y)))))
    return DN_ERR_INVALID_ARGUMENT;
  if (m > 0 && n > 0 && batch->n_slices > 0 && (!workspace || ws_bytes < eig_gram_batched_ws_bytes(batch->n_slices, m, n)))
    return DN_ERR_WORKSPACE;
  return launch_eig_gram_batched(X, ldx, Y, ldy, batch, m, n, active, out, (double*)workspace, (cudaStream_t)stream);
}

int dn_eig_rotate_batched(const double* X, int64_t ldx, const double* C, const dn_eig_batch* batch, int kd, int n,
                          double beta, const int32_t* active, double* Z, int64_t ldz, dn_stream_t stream) {
  if (!eig_batch_ok(batch) || kd < 0 || n < 0 || ldx < kd || ldz < n ||
      (batch->n_tiles > 0 && n > 0 && (!Z || (kd > 0 && (!X || !C)))) || (Z && Z == X))
    return DN_ERR_INVALID_ARGUMENT;
  if (batch->n_tiles > 65535) return DN_ERR_UNSUPPORTED;
  return launch_eig_rotate_batched(X, ldx, C, batch, kd, n, beta, active, Z, ldz, (cudaStream_t)stream);
}

int dn_eig_residual_norms_batched(const double* W, int64_t ldw, const double* Q, int64_t ldq, const double* theta,
                                  const dn_eig_batch* batch, int n, const int32_t* active, double* out, void* workspace,
                                  int64_t ws_bytes, dn_stream_t stream) {
  if (!eig_batch_ok(batch) || n < 0 || ldw < n || ldq < n ||
      (n > 0 && batch->n_meshes > 0 && (!out || !theta || (batch->n_tiles > 0 && (!W || !Q)))))
    return DN_ERR_INVALID_ARGUMENT;
  if (n > 0 && batch->n_slices > 0 && (!workspace || ws_bytes < eig_resid_batched_ws_bytes(batch->n_slices, n)))
    return DN_ERR_WORKSPACE;
  return launch_eig_residual_norms_batched(W, ldw, Q, ldq, theta, batch, n, active, out, (double*)workspace,
                                           (cudaStream_t)stream);
}

int dn_eig_finalize_batched(const double* Y, int64_t ldy, const int32_t* cols, int k, const double* mass,
                            const dn_eig_batch* batch, double* out, void* workspace, int64_t ws_bytes, dn_stream_t stream) {
  if (!eig_batch_ok(batch) || k < 0 || (batch->n_tiles > 0 && k > 0 && (!Y || !cols || !mass || !out)))
    return DN_ERR_INVALID_ARGUMENT;
  if (batch->n_tiles > 0 && k > 0 && (!workspace || ws_bytes < 8ll * batch->n_meshes * k)) return DN_ERR_WORKSPACE;
  return launch_eig_finalize_batched(Y, ldy, cols, k, mass, batch, out, (double*)workspace, (cudaStream_t)stream);
}

int64_t dn_implicit_diffusion_workspace_bytes(int64_t V, int C) {
  if (V < 0 || C <= 0) return -1;
  return implicit_ws_bytes(V, C);
}

static int implicit_check(const dn_csr* L, const float* mass, const float* time, const float* rhs, int64_t V, int C,
                          double rtol, int max_iter, const float* out, const double* status, const void* workspace,
                          int64_t ws_bytes) {
  if (!L || V < 0 || C <= 0 || L->nnz < 0 || !(rtol >= 0.0) || max_iter < 1 || !time || !status ||
      (V > 0 && (!L->rowptr || !mass || !rhs || !out || (L->nnz > 0 && (!L->colidx || !L->vals)))))
    return DN_ERR_INVALID_ARGUMENT;
  if (C > 256 || L->nnz >= (1ll << 31) || V >= (1ll << 31) - 1) return DN_ERR_UNSUPPORTED;
  if (!workspace || ws_bytes < implicit_ws_bytes(V, C)) return DN_ERR_WORKSPACE;
  return DN_OK;
}

int dn_implicit_diffusion_fwd(const dn_csr* L, const float* x, const float* mass, float* time, int64_t V, int C,
                              double rtol, int max_iter, float* x_diffuse, double* status, void* workspace,
                              int64_t ws_bytes, dn_stream_t stream) {
  const int rc = implicit_check(L, mass, time, x, V, C, rtol, max_iter, x_diffuse, status, workspace, ws_bytes);
  if (rc != DN_OK) return rc;
  return launch_implicit_diffusion(L, mass, time, x, nullptr, V, C, rtol, max_iter, 0, x_diffuse, nullptr, status,
                                   workspace, (cudaStream_t)stream);
}

int dn_implicit_diffusion_bwd(const dn_csr* L, const float* grad_out, const float* mass, const float* time,
                              const float* x_diffuse, int64_t V, int C, double rtol, int max_iter, float* grad_x,
                              float* grad_time, double* status, void* workspace, int64_t ws_bytes, dn_stream_t stream) {
  const int rc = implicit_check(L, mass, time, grad_out, V, C, rtol, max_iter, grad_x, status, workspace, ws_bytes);
  if (rc != DN_OK) return rc;
  if (!grad_time || (V > 0 && !x_diffuse)) return DN_ERR_INVALID_ARGUMENT;
  return launch_implicit_diffusion(L, mass, const_cast<float*>(time), grad_out, x_diffuse, V, C, rtol, max_iter, 1,
                                   grad_x, grad_time, status, workspace, (cudaStream_t)stream);
}

int64_t dn_implicit_diffusion_workspace_bytes_batched(int64_t V, int C, int n_meshes) {
  if (V < 0 || C <= 0 || n_meshes < 1) return -1;
  return implicit_batched_ws_bytes(V, C, n_meshes);
}

static int implicit_batched_check(const dn_csr* L, const float* mass, const float* time, const float* rhs,
                                  const dn_mesh_batch* batch, const int32_t* mesh_rows, int64_t V, int C, double rtol,
                                  int max_iter, const float* out, const double* status, const void* workspace,
                                  int64_t ws_bytes) {
  if (!L || !batch || batch->n_meshes < 1 || !batch->tile_mesh || !mesh_rows || V <= 0 || V % 128 != 0 || C <= 0 ||
      L->nnz < 0 || !(rtol >= 0.0) || max_iter < 1 || !time || !status || !L->rowptr || !mass || !rhs || !out ||
      (L->nnz > 0 && (!L->colidx || !L->vals)))
    return DN_ERR_INVALID_ARGUMENT;
  if (C > 256 || L->nnz >= (1ll << 31) || V >= (1ll << 31) - 1 || (int64_t)batch->n_meshes * C >= (1ll << 31))
    return DN_ERR_UNSUPPORTED;
  if (!workspace || ws_bytes < implicit_batched_ws_bytes(V, C, batch->n_meshes)) return DN_ERR_WORKSPACE;
  return DN_OK;
}

int dn_implicit_diffusion_fwd_batched(const dn_csr* L, const float* x, const float* mass, float* time,
                                      const dn_mesh_batch* batch, const int32_t* mesh_rows, int64_t V, int C,
                                      double rtol, int max_iter, float* x_diffuse, double* status, void* workspace,
                                      int64_t ws_bytes, dn_stream_t stream) {
  const int rc = implicit_batched_check(L, mass, time, x, batch, mesh_rows, V, C, rtol, max_iter, x_diffuse, status,
                                        workspace, ws_bytes);
  if (rc != DN_OK) return rc;
  return launch_implicit_diffusion_batched(L, mass, time, x, nullptr, batch, mesh_rows, V, C, rtol, max_iter, 0,
                                           x_diffuse, nullptr, status, workspace, (cudaStream_t)stream);
}

int dn_implicit_diffusion_bwd_batched(const dn_csr* L, const float* grad_out, const float* mass, const float* time,
                                      const float* x_diffuse, const dn_mesh_batch* batch, const int32_t* mesh_rows,
                                      int64_t V, int C, double rtol, int max_iter, float* grad_x, float* grad_time,
                                      double* status, void* workspace, int64_t ws_bytes, dn_stream_t stream) {
  const int rc = implicit_batched_check(L, mass, time, grad_out, batch, mesh_rows, V, C, rtol, max_iter, grad_x,
                                        status, workspace, ws_bytes);
  if (rc != DN_OK) return rc;
  if (!grad_time || !x_diffuse) return DN_ERR_INVALID_ARGUMENT;
  return launch_implicit_diffusion_batched(L, mass, const_cast<float*>(time), grad_out, x_diffuse, batch, mesh_rows, V,
                                           C, rtol, max_iter, 1, grad_x, grad_time, status, workspace,
                                           (cudaStream_t)stream);
}

int dn_compute_hks(const float* evals, const float* evecs, const float* scales, int64_t V, int K, int S, float* out,
                   dn_stream_t stream) {
  if (V < 0 || K <= 0 || S < 0 || ((V > 0 && S > 0) && (!evals || !evecs || !scales || !out)))
    return DN_ERR_INVALID_ARGUMENT;
  return launch_compute_hks(evals, evecs, scales, V, K, S, out, (cudaStream_t)stream);
}

int dn_to_basis(const float* values, const float* basis, const float* massvec, int64_t V, int K, int C, float* out,
                void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream) {
  if (!values || !basis || !out || V < 0 || K <= 0 || C <= 0) return DN_ERR_INVALID_ARGUMENT;
  Engine e;
  int rc = resolve(engine, &e);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Bump ws(workspace, ws_bytes);
  const int64_t pf = ws.left_floats() < kPartialFloats ? ws.left_floats() : kPartialFloats;
  float* partial = ws.take(pf);
  if (!partial) return DN_ERR_WORKSPACE;
  int P = 0;
  if ((rc = to_basis_partials(values, basis, massvec, V, K, C, partial, pf, &P, e, st))) return rc;
  return launch_reduce_partials(partial, P, nullptr, 1, K, C, out, C, 0, st);
}

int dn_from_basis(const float* values, const float* basis, const float* row_scale, int64_t V, int K, int C,
                  float* out, void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream) {
  if (!values || !basis || !out || V < 0 || K <= 0 || C <= 0) return DN_ERR_INVALID_ARGUMENT;
  Engine e;
  const int rc = resolve(engine, &e);
  if (rc) return rc;
  DnRowsSrc src = one_src(basis, K, K);
  DnLayer L = make_layer(values, C, /*w_trans=*/1, nullptr, 0, K, C, out, C);
  L.row_scale = row_scale;
  return run_chain(src, &L, 1, V, e, Bump(workspace, ws_bytes), (cudaStream_t)stream);
}

int dn_learned_time_diffusion_fwd(const float* x, const float* mass, const float* evals, const float* evecs,
                                  float* time, int64_t V, int K, int C, float* x_diffuse, float* x_spec_out,
                                  void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream) {
  if (!x || !mass || !evals || !evecs || !time || !x_diffuse || V < 0 || K <= 0 || C <= 0)
    return DN_ERR_INVALID_ARGUMENT;
  Engine e;
  int rc = resolve(engine, &e);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Bump ws(workspace, ws_bytes);
  float* S = ws.take((int64_t)K * C);
  const int64_t pf = ws.left_floats() / 2 < kPartialFloats ? ws.left_floats() / 2 : kPartialFloats;
  float* partial = ws.take(pf);
  if (!S || !partial) return DN_ERR_WORKSPACE;
  int P = 0;
  if ((rc = to_basis_partials(x, evecs, mass, V, K, C, partial, pf, &P, e, st))) return rc;
  rc = launch_spectral_scale(partial, P, evals, time, K, C, x_spec_out, S, /*clamp_writeback=*/1, st);
  if (rc) return rc;
  DnRowsSrc src = one_src(evecs, K, K);
  DnLayer L = make_layer(S, C, 1, nullptr, 0, K, C, x_diffuse, C);
  return run_chain(src, &L, 1, V, e, ws, st);
}

int dn_learned_time_diffusion_bwd(const float* grad_out, const float* mass, const float* evals, const float* evecs,
                                  const float* time, const float* x_spec, int64_t V, int K, int C, float* grad_x,
                                  float* grad_time, void* workspace, int64_t ws_bytes, int engine,
                                  dn_stream_t stream) {
  if (!grad_out || !mass || !evals || !evecs || !time || !x_spec || !grad_x || !grad_time)
    return DN_ERR_INVALID_ARGUMENT;
  Engine e;
  int rc = resolve(engine, &e);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Bump ws(workspace, ws_bytes);
  float* dS = ws.take((int64_t)K * C);
  const int64_t pf = ws.left_floats() / 2 < kPartialFloats ? ws.left_floats() / 2 : kPartialFloats;
  float* partial = ws.take(pf);
  if (!dS || !partial) return DN_ERR_WORKSPACE;
  int P = 0;
  if ((rc = to_basis_partials(grad_out, evecs, nullptr, V, K, C, partial, pf, &P, e, st))) return rc;
  if (P > 4) {
    // spectral_bwd walks the partials serially per channel: with the ~132 split-V partials of the tensor-core kernel that
    // took 4.5 ms (V = 7k); sum them first (coalesced, parallel) and hand it one
    float* red = ws.take((int64_t)K * C);
    if (!red) return DN_ERR_WORKSPACE;
    if ((rc = launch_reduce_partials(partial, P, nullptr, 1, K, C, red, C, 0, st))) return rc;
    rc = launch_spectral_bwd(red, 1, evals, time, x_spec, K, C, dS, grad_time, st);
  } else {
    rc = launch_spectral_bwd(partial, P, evals, time, x_spec, K, C, dS, grad_time, st);
  }
  if (rc) return rc;
  DnRowsSrc src = one_src(evecs, K, K);
  DnLayer L = make_layer(dS, C, 1, nullptr, 0, K, C, grad_x, C);
  L.row_scale = mass;
  return run_chain(src, &L, 1, V, e, ws, st);
}

int dn_learned_time_diffusion_fwd_batched(const float* x, const float* mass, const float* evals, const float* evecs,
                                          float* time, const dn_mesh_batch* batch, int64_t V, int K, int C,
                                          float* x_diffuse, float* x_spec_out, void* workspace, int64_t ws_bytes,
                                          int engine, dn_stream_t stream) {
  if (!x || !mass || !evals || !evecs || !time || !batch || !x_diffuse || V < 0 || K <= 0 || C <= 0)
    return DN_ERR_INVALID_ARGUMENT;
  Bump ws(workspace, ws_bytes);
  BatchedSpectral b;
  int rc = batched_spectral_plan(batch, evecs, V, K, C, engine, x_diffuse, ws, &b);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int P = 0;
  if ((rc = to_basis_partials(x, evecs, mass, V, K, C, b.partial, b.pf, &P, b.e, st, batch))) return rc;
  // S_b = exp(-lambda_b t) * (Phi_b^T M_b x_b), packed per mesh; the unscaled sums go to x_spec_out, the clamp to time
  const TcSpectral sp = {b.partial, P, evals, time, batch->n_meshes, batch->mesh_cta_begin, batch->tile_mesh,
                         x_spec_out, /*no_clamp_writeback=*/0};
  if ((rc = tc_pack_layers(&b.L, 1, b.packed, b.packed_bytes, &sp, st))) return rc;
  return run_chain(b.src, &b.L, 1, V, b.e, ws, st);
}

int dn_learned_time_diffusion_bwd_batched(const float* grad_out, const float* mass, const float* evals,
                                          const float* evecs, const float* time, const float* x_spec,
                                          const dn_mesh_batch* batch, int64_t V, int K, int C, float* grad_x,
                                          float* grad_time, void* workspace, int64_t ws_bytes, int engine,
                                          dn_stream_t stream) {
  if (!grad_out || !mass || !evals || !evecs || !time || !x_spec || !batch || !grad_x || !grad_time || V < 0 ||
      K <= 0 || C <= 0)
    return DN_ERR_INVALID_ARGUMENT;
  Bump ws(workspace, ws_bytes);
  BatchedSpectral b;
  int rc = batched_spectral_plan(batch, evecs, V, K, C, engine, grad_x, ws, &b);
  if (rc) return rc;
  b.L.row_scale = mass;
  cudaStream_t st = (cudaStream_t)stream;
  int P = 0;
  if ((rc = to_basis_partials(grad_out, evecs, nullptr, V, K, C, b.partial, b.pf, &P, b.e, st, batch))) return rc;
  // G_b = Phi_b^T g_b to b.sums and dS_b = exp(-lambda_b t) * G_b packed per mesh; time is only read
  const TcSpectral sp = {b.partial, P, evals, const_cast<float*>(time), batch->n_meshes, batch->mesh_cta_begin,
                         batch->tile_mesh, b.sums, /*no_clamp_writeback=*/1};
  if ((rc = tc_pack_layers(&b.L, 1, b.packed, b.packed_bytes, &sp, st))) return rc;
  if ((rc = run_chain(b.src, &b.L, 1, V, b.e, ws, st))) return rc;                // grad_x = M Phi_b dS_b
  return launch_spectral_time_grad_batched(b.sums, x_spec, evals, time, batch->n_meshes, K, C, grad_time, st);
}

int dn_to_basis_batched(const float* values, const float* basis, const float* mass, const dn_mesh_batch* batch,
                        int64_t V, int K, int C, float* out, void* workspace, int64_t ws_bytes, int engine,
                        dn_stream_t stream) {
  if (!values || !basis || !batch || !out || V < 0 || K <= 0 || C <= 0) return DN_ERR_INVALID_ARGUMENT;
  Bump ws(workspace, ws_bytes);
  BatchedSpectral b;
  // the batch envelope and scratch of the spectral diffusion; its from_basis chain (checked on `values`, a V x C array
  // like its output) is not run here
  int rc = batched_spectral_plan(batch, basis, V, K, C, engine, const_cast<float*>(values), ws, &b);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int P = 0;
  if ((rc = to_basis_partials(values, basis, mass, V, K, C, b.partial, b.pf, &P, b.e, st, batch))) return rc;
  return launch_reduce_partials(b.partial, P, batch->mesh_cta_begin, batch->n_meshes, K, C, out, C, 0, st);
}

int dn_from_basis_batched(const float* values, const float* basis, const float* row_scale, const dn_mesh_batch* batch,
                          int64_t V, int K, int C, float* out, void* workspace, int64_t ws_bytes, int engine,
                          dn_stream_t stream) {
  if (!values || !basis || !batch || !out || V < 0 || K <= 0 || C <= 0) return DN_ERR_INVALID_ARGUMENT;
  Bump ws(workspace, ws_bytes);
  BatchedSpectral b;
  int rc = batched_spectral_plan(batch, basis, V, K, C, engine, out, ws, &b);
  if (rc) return rc;
  b.L.row_scale = row_scale;
  cudaStream_t st = (cudaStream_t)stream;
  // every mesh's G_b packed as it is, in one launch; the chain then picks G_b per 128-row tile
  TcSpectral sp;
  memset(&sp, 0, sizeof(sp));
  sp.partial = values;
  sp.P = batch->n_meshes;
  sp.n_meshes = batch->n_meshes;
  sp.tile_mesh = batch->tile_mesh;
  sp.no_clamp_writeback = 1;
  sp.plain = 1;
  if ((rc = tc_pack_layers(&b.L, 1, b.packed, b.packed_bytes, &sp, st))) return rc;
  return run_chain(b.src, &b.L, 1, V, b.e, ws, st);
}

int dn_grad_spmm(const dn_csr* grad, const float* x, int64_t V, int C, float* out, dn_stream_t stream) {
  if (!grad || !grad->rowptr || !x || !out || V < 0 || C <= 0) return DN_ERR_INVALID_ARGUMENT;
  return launch_grad_spmm_pair(grad, x, V, C, out, (cudaStream_t)stream);
}

int dn_spatial_gradient_features_fwd(const float* vectors, const float* A_re, const float* A_im,
                                     int with_gradient_rotations, int64_t V, int C, float* out, void* workspace,
                                     int64_t ws_bytes, int engine, dn_stream_t stream) {
  if (!vectors || !A_re || (with_gradient_rotations && !A_im) || !out || V < 0 || C <= 0)
    return DN_ERR_INVALID_ARGUMENT;
  cudaStream_t st = (cudaStream_t)stream;
  Bump ws(workspace, ws_bytes);
  float* g01 = ws.take(V * 2 * C);
  float* b01 = ws.take(V * 2 * C);
  if (!g01 || !b01) return DN_ERR_WORKSPACE;
  int rc = launch_deinterleave_vc2(vectors, V, C, g01, st);
  if (rc) return rc;
  // Bre = g0 A_re^T - g1 A_im^T ; Bim = g1 A_re^T + g0 A_im^T   (layers.py:122-123)
  DnRowsSrc s0 = one_src(g01, C, 2 * C), s1 = one_src(g01 + C, C, 2 * C);
  if (with_gradient_rotations) {
    DnLayer T = make_layer(A_im, C, 0, nullptr, 0, C, C, b01, 2 * C);           // b0 = g1 A_im^T
    if ((rc = simt_rows_gemm(s1, T, V, st))) return rc;
    DnLayer L = make_layer(A_re, C, 0, nullptr, 0, C, C, b01, 2 * C);           // b0 = g0 A_re^T - b0
    L.residual = b01; L.ld_res = 2 * C; L.res_scale = -1.f;
    if ((rc = simt_rows_gemm(s0, L, V, st))) return rc;
    DnLayer M = make_layer(A_re, C, 0, nullptr, 0, C, C, b01 + C, 2 * C);       // b1 = g1 A_re^T
    if ((rc = simt_rows_gemm(s1, M, V, st))) return rc;
    DnLayer N2 = make_layer(A_im, C, 0, nullptr, 0, C, C, b01 + C, 2 * C);      // b1 = g0 A_im^T + b1
    N2.residual = b01 + C; N2.ld_res = 2 * C;
    if ((rc = simt_rows_gemm(s0, N2, V, st))) return rc;
  } else {
    DnLayer L = make_layer(A_re, C, 0, nullptr, 0, C, C, b01, 2 * C);           // layers.py:125-126
    if ((rc = simt_rows_gemm(s0, L, V, st))) return rc;
    L.out = b01 + C;
    if ((rc = simt_rows_gemm(s1, L, V, st))) return rc;
  }
  (void)engine;
  return launch_complex_dots_tanh(g01, b01, V, C, out, st);
}

int dn_gradient_features_fwd(const dn_csr* grad, const float* x_diffuse, const float* A_re, const float* A_im,
                             int with_gradient_rotations, int64_t V, int C, float* features, float* pq_out,
                             void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream) {
  if (!grad || !grad->rowptr || !x_diffuse || !A_re || (with_gradient_rotations && !A_im) || !features || V < 0 ||
      C <= 0)
    return DN_ERR_INVALID_ARGUMENT;
  Engine e;
  int rc = resolve(engine, &e);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Bump ws(workspace, ws_bytes);
  const int npq = with_gradient_rotations ? 2 * C : C;
  float* pq = pq_out ? pq_out : ws.take(V * npq);
  if (!pq) return DN_ERR_WORKSPACE;
  DnRowsSrc src = one_src(x_diffuse, C, C);
  DnLayer L = make_layer(A_re, C, 0, nullptr, 0, C, npq, pq, npq);   // [P|Q] = xd [A_re;A_im]^T
  if (with_gradient_rotations) { L.W2 = A_im; L.n_split = C; }
  if ((rc = run_chain(src, &L, 1, V, e, ws, st))) return rc;
  return launch_spmm_features(grad, x_diffuse, pq, with_gradient_rotations, V, C, features, st);
}

int dn_gradient_features_bwd(const dn_csr* grad, const dn_csr* grad_t, const float* grad_features,
                             const float* x_diffuse, const float* pq, const float* features, const float* A_re,
                             const float* A_im, int with_gradient_rotations, int64_t V, int C, float* grad_x,
                             float* grad_A_re, float* grad_A_im, void* workspace, int64_t ws_bytes, int engine,
                             dn_stream_t stream) {
  if (!grad || !grad_t || !grad_features || !x_diffuse || !pq || !features || !A_re || !grad_x || !grad_A_re ||
      (with_gradient_rotations && (!A_im || !grad_A_im)))
    return DN_ERR_INVALID_ARGUMENT;
  Engine e;
  int rc = resolve(engine, &e);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Bump ws(workspace, ws_bytes);
  const int rot = with_gradient_rotations;
  float* U = ws.take(V * 4 * C);
  float* dxd = ws.take(V * C);
  float* dP = ws.take(V * C);                      // dP, dQ as two contiguous (V, C) matrices: they are the chain
  float* dQ = rot ? ws.take(V * C) : nullptr;      // kernel's two sources and the weight-gradient kernel's operands
  float* part = ws.take(kPartialFloats / 4);
  if (!U || !dxd || !dP || (rot && !dQ) || !part) return DN_ERR_WORKSPACE;
  if ((rc = launch_features_bwd_local(grad, x_diffuse, pq, features, grad_features, rot, V, C, U, st))) return rc;
  if ((rc = launch_features_bwd_transpose(grad_t, U, rot, V, C, dxd, dP, dQ, C, st))) return rc;
  // grad_x = dxd + dP A_re (+ dQ A_im): one layer over the sources (dP | dQ) with [A_re ; A_im] stacked along K
  DnRowsSrc s = one_src(dP, C, C);
  if (rot) { s.ptr[1] = dQ; s.width[1] = C; s.ld[1] = C; s.nsrc = 2; }
  DnLayer L = make_layer(A_re, C, /*w_trans=*/1, nullptr, 0, rot ? 2 * C : C, C, grad_x, C);
  if (rot) { L.W2 = A_im; L.n_split = C; }
  L.residual = dxd; L.ld_res = C;
  if ((rc = run_chain(s, &L, 1, V, e, ws, st))) return rc;
  // grad_A_re[n][k] += sum_v dP[v][n] xd[v][k]   (and grad_A_im from dQ)
  if ((rc = atb(dP, C, C, x_diffuse, C, C, V, grad_A_re, C, 1, part, kPartialFloats / 4, e, st))) return rc;
  if (rot)
    if ((rc = atb(dQ, C, C, x_diffuse, C, C, V, grad_A_im, C, 1, part, kPartialFloats / 4, e, st))) return rc;
  return DN_OK;
}

int dn_mini_mlp_fwd(const float* const* src_host, const int* src_width_host, int nsrc,
                    const float* const* weight_host, const float* const* bias_host, const int* dims_host,
                    int n_layers, const float* const* drop_mask_host, const float* residual, int64_t V,
                    float* const* hidden_out_host, float* out, void* workspace, int64_t ws_bytes, int engine,
                    dn_stream_t stream) {
  if (!src_host || !src_width_host || nsrc < 1 || nsrc > DN_MAX_SRC || !weight_host || !dims_host || n_layers < 1 ||
      !out || V < 0)
    return DN_ERR_INVALID_ARGUMENT;
  DnRowsSrc src;
  memset(&src, 0, sizeof(src));
  int k0 = 0;
  for (int s = 0; s < nsrc; ++s) {
    if (!src_host[s] || src_width_host[s] <= 0) return DN_ERR_INVALID_ARGUMENT;
    src.ptr[s] = src_host[s]; src.width[s] = src_width_host[s]; src.ld[s] = src_width_host[s];
    k0 += src_width_host[s];
  }
  src.nsrc = nsrc;
  if (k0 != dims_host[0]) return DN_ERR_INVALID_ARGUMENT;
  // a MiniMLP deeper than one fused chain (DN_MAX_LAYERS) runs layer by layer in run_chain
  std::vector<DnLayer> layers(n_layers);
  for (int l = 0; l < n_layers; ++l) {
    if (!weight_host[l] || dims_host[l + 1] <= 0) return DN_ERR_INVALID_ARGUMENT;
    const bool last = (l + 1 == n_layers);
    float* o = last ? out : (hidden_out_host ? hidden_out_host[l] : nullptr);
    layers[l] = make_layer(weight_host[l], dims_host[l], 0, bias_host ? bias_host[l] : nullptr, last ? 0 : 1,
                           dims_host[l], dims_host[l + 1], o, dims_host[l + 1]);
    if (!last && drop_mask_host) layers[l].emul = drop_mask_host[l];
    if (last && residual) { layers[l].residual = residual; layers[l].ld_res = dims_host[l + 1]; }
  }
  Engine e;
  const int rc = resolve(engine, &e);
  if (rc) return rc;
  return run_chain(src, layers.data(), n_layers, V, e, Bump(workspace, ws_bytes), (cudaStream_t)stream);
}

int dn_mini_mlp_bwd(const float* grad_out, const float* const* src_host, const int* src_width_host, int nsrc,
                    const float* const* weight_host, const int* dims_host, int n_layers,
                    const float* const* hidden_host, const float* const* drop_mask_host, int64_t V,
                    float* const* grad_src_host, float* const* grad_weight_host, float* const* grad_bias_host,
                    void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream) {
  if (!grad_out || !src_host || !src_width_host || nsrc < 1 || nsrc > DN_MAX_SRC || !weight_host || !dims_host ||
      n_layers < 1 || (n_layers > 1 && !hidden_host) || !grad_src_host ||
      !grad_weight_host)
    return DN_ERR_INVALID_ARGUMENT;
  Engine e;
  int rc = resolve(engine, &e);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int maxn = 0;
  for (int l = 0; l <= n_layers; ++l) maxn = dims_host[l] > maxn ? dims_host[l] : maxn;
  Bump ws(workspace, ws_bytes);
  float* d0 = ws.take(V * maxn);
  float* d1 = ws.take(V * maxn);
  float* part = ws.take(kPartialFloats / 2);
  if (!d0 || !d1 || !part) return DN_ERR_WORKSPACE;
  const float* dz = grad_out;   // gradient w.r.t. the pre-activation of layer l
  for (int l = n_layers - 1; l >= 0; --l) {
    const int nout = dims_host[l + 1], nin = dims_host[l];
    // weight / bias gradients:  grad_W[n][k] += sum_v dz[v][n] * h_{l-1}[v][k]
    if (l > 0) {
      if ((rc = atb(dz, nout, nout, hidden_host[l - 1], nin, nin, V, grad_weight_host[l], nin, 1, part,
                    kPartialFloats / 2, e, st)))
        return rc;
    } else {
      int off = 0;
      for (int s = 0; s < nsrc; ++s) {
        if ((rc = atb(dz, nout, nout, src_host[s], src_width_host[s], src_width_host[s], V, grad_weight_host[0] + off,
                      nin, 1, part, kPartialFloats / 2, e, st)))
          return rc;
        off += src_width_host[s];
      }
    }
    if (grad_bias_host && grad_bias_host[l])
      if ((rc = simt_colsum(dz, nout, nout, V, grad_bias_host[l], 1, part, kPartialFloats / 2, st))) return rc;
    // input gradient:  dz_{l-1} = (dz_l W_l) * 1[h_{l-1} > 0] (* dropout mask)
    DnRowsSrc s = one_src(dz, nout, nout);
    if (l > 0) {
      float* o = (dz == d0) ? d1 : d0;
      DnLayer L = make_layer(weight_host[l], nin, /*w_trans=*/1, nullptr, 0, nout, nin, o, nin);
      L.relu_mask_src = hidden_host[l - 1];
      if (drop_mask_host && drop_mask_host[l - 1]) L.emul = drop_mask_host[l - 1];
      if ((rc = run_chain(s, &L, 1, V, e, ws, st))) return rc;
      dz = o;
    } else {
      int off = 0;
      for (int q = 0; q < nsrc; ++q) {
        if (grad_src_host[q]) {
          DnLayer L = make_layer(weight_host[0] + off, nin, 1, nullptr, 0, nout, src_width_host[q], grad_src_host[q],
                                 src_width_host[q]);
          if ((rc = run_chain(s, &L, 1, V, e, ws, st))) return rc;
        }
        off += src_width_host[q];
      }
    }
  }
  return DN_OK;
}

static int block_fwd_impl(const float* x_in, const float* mass, const float* evals, const float* evecs,
                          const dn_csr* grad, const dn_block_params* p, int64_t V, int K, int C, float* out,
                          void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream, cudaEvent_t* ev,
                          const dn_mesh_batch* batch = nullptr, const dn_head* head = nullptr) {
  // ev (optional, DN_PROFILE_STAGES + 1 events): recorded on the launching stream between the stages
  auto mark = [&](int i) { if (ev) cudaEventRecord(ev[i], (cudaStream_t)stream); };
  if (!x_in || !mass || !evals || !evecs || !p || !p->diffusion_time || (!out && !head) || V < 0 || K <= 0 || C <= 0)
    return DN_ERR_INVALID_ARGUMENT;
  if (head && (!head->weight || !head->out || head->n_out < 1 || head->n_out > 8 || head->ld_out < head->n_out))
    return DN_ERR_INVALID_ARGUMENT;
  if (p->with_gradient_features && (!grad || !grad->rowptr || !p->A_re || (p->with_gradient_rotations && !p->A_im)))
    return DN_ERR_INVALID_ARGUMENT;
  if (p->n_mlp_layers < 1 || !p->mlp_weight_host || !p->mlp_dims_host)
    return DN_ERR_INVALID_ARGUMENT;
  cudaStream_t st = (cudaStream_t)stream;
  Bump ws(workspace, ws_bytes);
  const int rot = p->with_gradient_rotations;
  const int npq = rot ? 2 * C : C;
  float* S = ws.take((int64_t)K * C);
  float* xd = ws.take(V * C);
  float* pq = p->with_gradient_features ? ws.take(V * npq) : nullptr;
  float* feat = p->with_gradient_features ? ws.take(V * C) : nullptr;
  const int64_t pf = kPartialFloats;
  float* partial = ws.take(pf);
  if (!S || !xd || !partial || (p->with_gradient_features && (!pq || !feat))) return DN_ERR_WORKSPACE;
  int rc, P = 0;

  // every dense layer of the block: [0] from_basis, [1] (a5, commuted) [P|Q] = x_diffuse [A_re;A_im]^T,
  // [2..] cat -> MiniMLP -> + x_in  [layers.py:229-239]
  const int nm = p->n_mlp_layers;
  Engine e;
  if ((rc = resolve(engine, &e))) return rc;
  // a MiniMLP deeper than one fused chain (DN_MAX_LAYERS) is not a tensor-core chain: run_chain runs it layer by layer
  std::vector<DnLayer> L(3 + nm);
  L[0] = make_layer(S, C, 1, nullptr, 0, K, C, xd, C);
  int nfront = 1;
  // gradient features, commuted route: [P|Q] = x_diffuse [A_re; A_im]^T as a dense layer in front of one CSR gather of
  // x, P and Q that forms tanh(gX * Bre + gY * Bim) (layers.py:117-130)
  if (p->with_gradient_features) {
    if (rot && (npq > 256 || (e.tc && npq > 128))) {
      // [P|Q] wider than one tensor-core layer (C_width = 256), or wider than a layer inside a chain (C_width = 128):
      // P and Q are separate layers writing the two halves.  At C_width = 128 they join from_basis in one chain, Q
      // as P's sibling (both read x_diffuse from the registers from_basis left it in)
      L[1] = make_layer(p->A_re, C, 0, nullptr, 0, C, C, pq, npq);
      L[2] = make_layer(p->A_im, C, 0, nullptr, 0, C, C, pq + C, npq);
      L[2].sibling = 1;
      nfront = 3;
    } else {
      L[1] = make_layer(p->A_re, C, 0, nullptr, 0, C, npq, pq, npq);
      if (rot) { L[1].W2 = p->A_im; L[1].n_split = C; }
      nfront = 2;
    }
  }
  const int nsrc = p->with_gradient_features ? 3 : 2;
  if (p->mlp_dims_host[0] != nsrc * C) return DN_ERR_INVALID_ARGUMENT;
  for (int l = 0; l < nm; ++l) {
    const bool last = (l + 1 == nm);
    if (!p->mlp_weight_host[l] || p->mlp_dims_host[l + 1] <= 0) return DN_ERR_INVALID_ARGUMENT;
    L[nfront + l] = make_layer(p->mlp_weight_host[l], p->mlp_dims_host[l], 0,
                               p->mlp_bias_host ? p->mlp_bias_host[l] : nullptr, last ? 0 : 1, p->mlp_dims_host[l],
                               p->mlp_dims_host[l + 1], last ? out : nullptr, p->mlp_dims_host[l + 1]);
    if (last) {
      L[nfront + l].residual = x_in; L[nfront + l].ld_res = C;
      if (head) {        // DiffusionNet.last_lin in this layer's epilogue; the block output itself is not stored
        DnLayer& Lh = L[nfront + l];
        Lh.head_w = head->weight; Lh.head_b = head->bias; Lh.head_out = head->out; Lh.ld_head_out = head->ld_out;
        Lh.head_n = head->n_out;
        if (!out) Lh.out = nullptr;
      }
    }
  }
  if (p->mlp_dims_host[nm] != C) return DN_ERR_INVALID_ARGUMENT;
  DnRowsSrc src_fb = one_src(evecs, K, K);
  DnRowsSrc src_pq = one_src(xd, C, C);
  DnRowsSrc src_mlp;
  memset(&src_mlp, 0, sizeof(src_mlp));
  const float* srcs[3] = {x_in, xd, feat};
  for (int q = 0; q < nsrc; ++q) { src_mlp.ptr[q] = srcs[q]; src_mlp.width[q] = C; src_mlp.ld[q] = C; }
  src_mlp.nsrc = nsrc;
  // which chains run on tensor cores: from_basis and [P|Q] (or P, Q) as one fused chain when it fits, else each layer
  // on its own (Q then reads x_diffuse from HBM like P); the MiniMLP chain
  const bool front_fused = e.tc && nfront > 1 && tc_chain_plan(src_fb, &L[0], nfront, e.passes) >= 0;
  if (!front_fused && nfront == 3) L[2].sibling = 0;
  bool tc_front = front_fused;
  if (e.tc && !front_fused) {
    tc_front = tc_chain_plan(src_fb, &L[0], 1, e.passes) >= 0;
    for (int l = 1; l < nfront; ++l) tc_front = tc_front && tc_chain_plan(src_pq, &L[l], 1, e.passes) >= 0;
  }
  const bool tc_mlp = e.tc && tc_chain_plan(src_mlp, &L[nfront], nm, e.passes) >= 0;
  if (head && !tc_mlp) return DN_ERR_UNSUPPORTED;
  // a batch forms every mesh's spectral multiplier in the pack launch of the tensor-core front chain
  if (batch && (!tc_front || (V % 128) || batch->n_meshes < 1 || !batch->tile_mesh || !batch->tb_rows ||
                !batch->mesh_cta_begin || batch->n_tb_ctas < 1))
    return DN_ERR_UNSUPPORTED;
  // (nothing has been launched up to here: an unsupported head / batch returns before any work is enqueued)
  mark(0);
  // (a1) spectral diffusion: to_basis -> exp(-lambda t) -> from_basis   [layers.py:56-67]
  if ((rc = to_basis_partials(x_in, evecs, mass, V, K, C, partial, pf, &P, e, st, batch))) return rc;
  mark(1);
  if (!tc_front)
    if ((rc = launch_spectral_scale(partial, P, evals, p->diffusion_time, K, C, nullptr, S, 1, st))) return rc;
  mark(2);
  // one launch packs (hi/lo split + wgmma layout) every weight the tensor-core kernels will stream.  On the front chain
  // the spectral multiplier S = exp(-lambda t) * (reduced partial sums), layer 0's weight, is formed there (no separate
  // scale kernel, S never round-trips HBM), one per mesh of a batch.
  if (tc_front || tc_mlp) {
    DnLayer* first = tc_front ? &L[0] : &L[nfront];
    const int cnt = (tc_front ? nfront : 0) + (tc_mlp ? nm : 0);
    const TcSpectral sp = {partial, P, evals, p->diffusion_time, batch ? batch->n_meshes : 1,
                           batch ? batch->mesh_cta_begin : nullptr, batch ? batch->tile_mesh : nullptr};
    const int64_t pb = tc_chain_ws_bytes(first, cnt, tc_front ? sp.n_meshes : 1);
    float* pk = ws.take(pb / 4);
    if (!pk) return DN_ERR_WORKSPACE;
    if ((rc = tc_pack_layers(first, cnt, pk, pb, tc_front ? &sp : nullptr, st))) return rc;
  }
  mark(3);
  const int n_fused = front_fused ? nfront : 1;
  if ((rc = run_chain(src_fb, &L[0], n_fused, V, e, ws, st))) return rc;
  for (int l = n_fused; l < nfront; ++l)
    if ((rc = run_chain(src_pq, &L[l], 1, V, e, ws, st))) return rc;
  mark(4);
  // (a4+a5) sparse tangent gradient + complex inner product + tanh   [layers.py:216-226,128-130]
  if (p->with_gradient_features) {
    if ((rc = launch_spmm_features(grad, xd, pq, rot, V, C, feat, st))) return rc;
  }
  mark(5);
  rc = run_chain(src_mlp, &L[nfront], nm, V, e, ws, st);
  mark(6);
  return rc;
}

int dn_block_fwd(const float* x_in, const float* mass, const float* evals, const float* evecs, const dn_csr* grad,
                 const dn_block_params* p, int64_t V, int K, int C, float* out, void* workspace, int64_t ws_bytes,
                 int engine, dn_stream_t stream) {
  return block_fwd_impl(x_in, mass, evals, evecs, grad, p, V, K, C, out, workspace, ws_bytes, engine, stream, nullptr);
}

int dn_block_fwd_batched(const float* x_in, const float* mass, const float* evals, const float* evecs, const dn_csr* grad,
                         const dn_block_params* p, const dn_mesh_batch* batch, int64_t V, int K, int C, float* out,
                         void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream) {
  if (!batch) return DN_ERR_INVALID_ARGUMENT;
  return block_fwd_impl(x_in, mass, evals, evecs, grad, p, V, K, C, out, workspace, ws_bytes, engine, stream, nullptr, batch);
}

int dn_block_fwd_ex(const float* x_in, const float* mass, const float* evals, const float* evecs, const dn_csr* grad,
                    const dn_block_params* p, const dn_mesh_batch* batch, const dn_head* head, int64_t V, int K, int C,
                    float* out, void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream) {
  return block_fwd_impl(x_in, mass, evals, evecs, grad, p, V, K, C, out, workspace, ws_bytes, engine, stream, nullptr, batch, head);
}

int dn_mesh_batch_plan(int n_meshes, const int32_t* n_rows_host, int sm_count, int32_t* row_begin_host,
                       int32_t* tile_mesh_host, int32_t* tb_rows_host, int32_t* mesh_cta_begin_host) {
  if (n_meshes < 1 || !n_rows_host || !row_begin_host || !tile_mesh_host || !tb_rows_host || !mesh_cta_begin_host)
    return DN_ERR_INVALID_ARGUMENT;
  if (sm_count < 1) sm_count = 132;
  int64_t row = 0, chunks_total = 0;
  for (int b = 0; b < n_meshes; ++b) {
    if (n_rows_host[b] < 0) return DN_ERR_INVALID_ARGUMENT;
    row_begin_host[b] = (int32_t)row;
    const int64_t padded = ((int64_t)n_rows_host[b] + 127) / 128 * 128;
    for (int64_t t = row / 128; t < (row + padded) / 128; ++t) tile_mesh_host[t] = b;
    row += padded;
    if (row >= (1ll << 31) - 256) return DN_ERR_UNSUPPORTED;
    chunks_total += ((int64_t)n_rows_host[b] + 15) / 16;
  }
  row_begin_host[n_meshes] = (int32_t)row;
  // CTAs per mesh proportional to its 16-row chunks (>= 1), about sm_count in total, at most 1024
  int n_ctas = 0;
  for (int b = 0; b < n_meshes; ++b) {
    const int64_t chunks = ((int64_t)n_rows_host[b] + 15) / 16;
    int64_t want = chunks_total > 0 ? (chunks * sm_count + chunks_total / 2) / chunks_total : 1;
    if (want < 1) want = 1;
    if (want > chunks && chunks > 0) want = chunks;
    if (n_ctas + want + (n_meshes - 1 - b) > 1024) want = 1;
    if (n_ctas + want > 1024) return DN_ERR_UNSUPPORTED;
    mesh_cta_begin_host[b] = n_ctas;
    const int64_t per = chunks > 0 ? (chunks + want - 1) / want : 0;
    if (per > 0) want = (chunks + per - 1) / per;              // no empty CTAs
    for (int64_t c = 0; c < want; ++c) {
      int64_t rb = row_begin_host[b] + c * per * 16;
      int64_t re = rb + per * 16;
      const int64_t end = (int64_t)row_begin_host[b] + n_rows_host[b];
      if (rb > end) rb = end;
      if (re > end) re = end;
      tb_rows_host[2 * n_ctas] = (int32_t)rb;
      tb_rows_host[2 * n_ctas + 1] = (int32_t)re;
      ++n_ctas;
    }
  }
  mesh_cta_begin_host[n_meshes] = n_ctas;
  return n_ctas;
}

int dn_batch_gather(const dn_gather_part* parts_host, int n_parts, const int64_t* table, int n_ranges, int n_meshes,
                    dn_stream_t stream) {
  if (!parts_host || n_parts < 1 || n_parts > DN_GATHER_MAX_PARTS || !table || n_ranges < 1 || n_meshes < 1 ||
      n_meshes > 65535)
    return DN_ERR_INVALID_ARGUMENT;
  for (int p = 0; p < n_parts; ++p) {
    const dn_gather_part& q = parts_host[p];
    if (!q.src || !q.dst || q.width < 1 || q.range < 0 || q.range >= n_ranges || q.max_units < 0) return DN_ERR_INVALID_ARGUMENT;
    if (q.op != DN_GATHER_COPY && q.op != DN_GATHER_ADD_I32 && q.op != DN_GATHER_ADD_I64) return DN_ERR_INVALID_ARGUMENT;
    if (q.op != DN_GATHER_COPY && (q.offset_range < 0 || q.offset_range >= n_ranges)) return DN_ERR_INVALID_ARGUMENT;
  }
  return launch_batch_gather(parts_host, n_parts, table, n_ranges, n_meshes, (cudaStream_t)stream);
}

int dn_mesh_batch_plan_device(const int64_t* ids, int n_meshes, const int64_t* dataset_sizes, int64_t n_dataset,
                              int sm_count, int64_t V_cap, int64_t entry_cap, int n_tb_ctas, int64_t tail_rows,
                              int n_ranges, const dn_slot_plan* out_host, dn_stream_t stream) {
  return dn_mesh_batch_plan_device_elements(ids, n_meshes, dataset_sizes, 4, n_dataset, sm_count, V_cap, entry_cap,
                                            n_tb_ctas, tail_rows, n_ranges, out_host, nullptr, 0, 0, stream);
}

int dn_mesh_batch_plan_device_elements(const int64_t* ids, int n_meshes, const int64_t* dataset_sizes, int size_cols,
                                       int64_t n_dataset, int sm_count, int64_t V_cap, int64_t entry_cap,
                                       int n_tb_ctas, int64_t tail_rows, int n_ranges, const dn_slot_plan* out_host,
                                       const dn_slot_elements* elements_host, int n_kinds, int corner_range,
                                       dn_stream_t stream) {
  if (n_kinds < 0 || n_kinds > DN_SLOT_MAX_ELEMENT_KINDS || (n_kinds > 0 && !elements_host) ||
      size_cols < 4 + 2 * n_kinds)
    return DN_ERR_INVALID_ARGUMENT;
  if (n_kinds > 0) {                   // corner_range, every range and csr_range: distinct, past the four fixed ones
    int used[2 * DN_SLOT_MAX_ELEMENT_KINDS + 1] = {corner_range};
    int n_used = 1;
    for (int q = 0; q < n_kinds; ++q) {
      const dn_slot_elements& k = elements_host[q];
      if (k.capacity < 128 || k.capacity % 128 || k.k < 1 || k.capacity * k.k >= (1ll << 31) || k.tail < 1 ||
          k.tail * n_meshes < k.capacity || !k.begin || !k.count || !k.tile_seg)
        return DN_ERR_INVALID_ARGUMENT;
      used[n_used++] = k.range;
      used[n_used++] = k.csr_range;
    }
    for (int i = 0; i < n_used; ++i) {
      if (used[i] < 4 || used[i] >= n_ranges) return DN_ERR_INVALID_ARGUMENT;
      for (int j = 0; j < i; ++j)
        if (used[i] == used[j]) return DN_ERR_INVALID_ARGUMENT;
    }
  }
  if (sm_count < 1) sm_count = 132;
  const int64_t min_ctas = sm_count + (int64_t)n_meshes < 1024 ? sm_count + (int64_t)n_meshes : 1024;
  if (!ids || !dataset_sizes || !out_host || n_meshes < 1 || n_meshes > 1024 || n_dataset < 1 || V_cap < 128 ||
      V_cap % 128 || V_cap >= (1ll << 31) - 256 || entry_cap < 0 || entry_cap >= (1ll << 31) || n_tb_ctas < min_ctas ||
      n_tb_ctas > 1024 || tail_rows < 1 || tail_rows * n_meshes < V_cap || n_ranges < 4)
    return DN_ERR_INVALID_ARGUMENT;
  const dn_slot_plan& o = *out_host;
  if (!o.row_begin || !o.tile_mesh || !o.tb_rows || !o.mesh_cta_begin || !o.seg_begin || !o.seg_rows || !o.tile_seg ||
      !o.table || !o.status)
    return DN_ERR_INVALID_ARGUMENT;
  return launch_mesh_batch_plan_device(ids, n_meshes, dataset_sizes, size_cols, n_dataset, sm_count, V_cap, entry_cap,
                                       n_tb_ctas, tail_rows, n_ranges, o, elements_host, n_kinds, corner_range,
                                       (cudaStream_t)stream);
}

int dn_block_fwd_profile(const float* x_in, const float* mass, const float* evals, const float* evecs,
                         const dn_csr* grad, const dn_block_params* p, int64_t V, int K, int C, float* out,
                         void* workspace, int64_t ws_bytes, int engine, dn_stream_t stream, float* stage_ms_host) {
  if (!stage_ms_host) return DN_ERR_INVALID_ARGUMENT;
  cudaEvent_t ev[DN_PROFILE_STAGES + 1];
  for (int i = 0; i <= DN_PROFILE_STAGES; ++i) DN_CUDA_TRY(cudaEventCreate(&ev[i]));
  int rc = block_fwd_impl(x_in, mass, evals, evecs, grad, p, V, K, C, out, workspace, ws_bytes, engine, stream, ev);
  if (rc == DN_OK) {
    rc = (int)cudaEventSynchronize(ev[DN_PROFILE_STAGES]);
    for (int i = 0; i < DN_PROFILE_STAGES && rc == DN_OK; ++i)
      rc = (int)cudaEventElapsedTime(&stage_ms_host[i], ev[i], ev[i + 1]);
  }
  for (int i = 0; i <= DN_PROFILE_STAGES; ++i) cudaEventDestroy(ev[i]);
  return rc;
}

}  // extern "C"

// ---- fused classification head ----
namespace {
int linear_nll_check(const float* x, const float* weight, const int64_t* labels, int64_t R, int C, int n_class,
                     int engine, Engine* e) {
  if (!x || !weight || !labels || R < 1 || n_class < 1 || C < 1) return DN_ERR_INVALID_ARGUMENT;
  if (C % 16 != 0 || C > 256 || R >= (1ll << 31) || (int64_t)n_class * C >= (1ll << 31)) return DN_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(weight)) & 15) return DN_ERR_UNSUPPORTED;
  const int rc = resolve(engine, e);
  if (rc != DN_OK) return rc;
  return e->tc ? DN_OK : DN_ERR_UNSUPPORTED;   // tensor cores only: the SIMT engine composes mlp + log_softmax instead
}

int smoothing_check(float s, int n_class) {
  if (!(s >= 0.f && s <= 1.f) || (s > 0.f && n_class < 2)) return DN_ERR_INVALID_ARGUMENT;
  return DN_OK;
}

int global_mean_check(const float* x, const float* mass, int64_t V, int C, const int32_t* begin, const int32_t* rows,
                      const int32_t* tile_seg, int n_seg) {
  if (!x || !mass || !begin || !rows || !tile_seg || V < 1 || n_seg < 1 || C < 1) return DN_ERR_INVALID_ARGUMENT;
  if (C % 4 != 0 || C > 256 || V >= (1ll << 31) || (reinterpret_cast<uintptr_t>(x) & 15)) return DN_ERR_UNSUPPORTED;
  return DN_OK;
}
}  // namespace

extern "C" {

int64_t dn_linear_nll_workspace_bytes(int64_t R, int C, int n_class) {
  if (R < 1 || C < 1 || n_class < 1) return 0;
  return head_ws_bytes(R, C, n_class);
}

int dn_linear_nll_fwd(const float* x, const float* weight, const float* bias, const int64_t* labels, int64_t R, int C,
                      int n_class, int64_t ignore_index, float* nll, int64_t* argmax, float* lse, int engine,
                      dn_stream_t stream) {
  Engine e;
  int rc = linear_nll_check(x, weight, labels, R, C, n_class, engine, &e);
  if (rc != DN_OK) return rc;
  if (!nll || !argmax || !lse) return DN_ERR_INVALID_ARGUMENT;
  return launch_linear_nll_fwd(x, weight, bias, labels, R, C, n_class, ignore_index, 0.f, nll, argmax, lse, e.passes,
                               (cudaStream_t)stream);
}

int dn_linear_nll_ls_fwd(const float* x, const float* weight, const float* bias, const int64_t* labels, int64_t R,
                         int C, int n_class, int64_t ignore_index, float* nll, int64_t* argmax, float* lse, int engine,
                         dn_stream_t stream, float label_smoothing) {
  Engine e;
  int rc = linear_nll_check(x, weight, labels, R, C, n_class, engine, &e);
  if (rc == DN_OK) rc = smoothing_check(label_smoothing, n_class);
  if (rc != DN_OK) return rc;
  if (!nll || !argmax || !lse) return DN_ERR_INVALID_ARGUMENT;
  return launch_linear_nll_fwd(x, weight, bias, labels, R, C, n_class, ignore_index, label_smoothing, nll, argmax, lse,
                               e.passes, (cudaStream_t)stream);
}

int dn_linear_nll_bwd(const float* x, const float* weight, const float* bias, const int64_t* labels, const float* lse,
                      const float* grad_nll, int64_t R, int C, int n_class, int64_t ignore_index, float* grad_x,
                      float* grad_weight, float* grad_bias, void* workspace, int64_t ws_bytes, int engine,
                      dn_stream_t stream) {
  Engine e;
  int rc = linear_nll_check(x, weight, labels, R, C, n_class, engine, &e);
  if (rc != DN_OK) return rc;
  if (!lse || !grad_nll || !grad_x || !grad_weight || (bias && !grad_bias)) return DN_ERR_INVALID_ARGUMENT;
  if (!workspace || ws_bytes < head_ws_bytes(R, C, n_class)) return DN_ERR_WORKSPACE;
  return launch_linear_nll_bwd(x, weight, bias, labels, lse, grad_nll, R, C, n_class, ignore_index, 0.f, grad_x,
                               grad_weight, bias ? grad_bias : nullptr, workspace, e.passes, (cudaStream_t)stream);
}

int dn_linear_nll_ls_bwd(const float* x, const float* weight, const float* bias, const int64_t* labels,
                         const float* lse, const float* grad_nll, int64_t R, int C, int n_class, int64_t ignore_index,
                         float* grad_x, float* grad_weight, float* grad_bias, void* workspace, int64_t ws_bytes,
                         int engine, dn_stream_t stream, float label_smoothing) {
  Engine e;
  int rc = linear_nll_check(x, weight, labels, R, C, n_class, engine, &e);
  if (rc == DN_OK) rc = smoothing_check(label_smoothing, n_class);
  if (rc != DN_OK) return rc;
  if (!lse || !grad_nll || !grad_x || !grad_weight || (bias && !grad_bias)) return DN_ERR_INVALID_ARGUMENT;
  if (!workspace || ws_bytes < head_ws_bytes(R, C, n_class)) return DN_ERR_WORKSPACE;
  return launch_linear_nll_bwd(x, weight, bias, labels, lse, grad_nll, R, C, n_class, ignore_index, label_smoothing,
                               grad_x, grad_weight, bias ? grad_bias : nullptr, workspace, e.passes,
                               (cudaStream_t)stream);
}

int dn_element_mean_fwd(const float* x, int64_t V, int C, const int64_t* elems, int64_t E, int k, float* out,
                        dn_stream_t stream) {
  if (V < 1 || C < 1 || E < 0 || k < 1 || (E > 0 && (!x || !elems || !out))) return DN_ERR_INVALID_ARGUMENT;
  if (E == 0) return DN_OK;
  return launch_element_mean_fwd(x, C, elems, E, k, out, (cudaStream_t)stream);
}

int dn_element_mean_bwd(const float* grad_out, int64_t E, int C, const int32_t* rowptr, const int32_t* entries,
                        int64_t V, int k, float* grad_x, dn_stream_t stream) {
  if (V < 1 || C < 1 || E < 0 || k < 1 || !rowptr || !grad_x || (E > 0 && (!grad_out || !entries)))
    return DN_ERR_INVALID_ARGUMENT;
  if (E * k >= (1ll << 31)) return DN_ERR_UNSUPPORTED;
  return launch_element_mean_bwd(grad_out, C, rowptr, entries, V, k, grad_x, (cudaStream_t)stream);
}

int64_t dn_global_mean_workspace_bytes(int64_t V, int C) {
  if (V < 1 || C < 1) return 0;
  return pool_ws_bytes(V, C);
}

int dn_global_mean_fwd(const float* x, const float* mass, int64_t V, int C, const int32_t* seg_begin,
                       const int32_t* seg_rows, const int32_t* tile_seg, int n_seg, float* pooled, float* mass_sum,
                       void* workspace, int64_t ws_bytes, dn_stream_t stream) {
  const int rc = global_mean_check(x, mass, V, C, seg_begin, seg_rows, tile_seg, n_seg);
  if (rc != DN_OK) return rc;
  if (!pooled || !mass_sum) return DN_ERR_INVALID_ARGUMENT;
  if (reinterpret_cast<uintptr_t>(pooled) & 15) return DN_ERR_UNSUPPORTED;
  if (!workspace || ws_bytes < pool_ws_bytes(V, C)) return DN_ERR_WORKSPACE;
  if (reinterpret_cast<uintptr_t>(workspace) & 15) return DN_ERR_UNSUPPORTED;
  return launch_global_mean_fwd(x, mass, V, C, seg_begin, seg_rows, tile_seg, n_seg, pooled, mass_sum, workspace,
                                (cudaStream_t)stream);
}

int dn_global_mean_bwd(const float* grad_pooled, const float* mass, const float* mass_sum, int64_t V, int C,
                       const int32_t* seg_begin, const int32_t* seg_rows, const int32_t* tile_seg, int n_seg,
                       float* grad_x, dn_stream_t stream) {
  const int rc = global_mean_check(grad_pooled, mass, V, C, seg_begin, seg_rows, tile_seg, n_seg);
  if (rc != DN_OK) return rc;
  if (!mass_sum || !grad_x) return DN_ERR_INVALID_ARGUMENT;
  if (reinterpret_cast<uintptr_t>(grad_x) & 15) return DN_ERR_UNSUPPORTED;
  return launch_global_mean_bwd(grad_pooled, mass, mass_sum, V, C, seg_begin, seg_rows, tile_seg, n_seg, grad_x,
                                (cudaStream_t)stream);
}

}  // extern "C"
