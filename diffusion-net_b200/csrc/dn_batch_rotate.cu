// Per-mesh rotations of the (V, 3) rows of a mesh batch or batch slot (dn_rotate_rows, batch.rotate_rows and the
// rotations= argument of MeshDataset.pack / BatchSlot.pack): the reference's random_rotate_points applied to every
// mesh of a batch in one launch.  The mesh of a row is read from the layout's tile table, so a host-planned batch and
// a device-planned slot are served alike.
#include "dn_internal.h"

namespace {

constexpr int kThreads = 256;

// out[v] = x[v] @ R[tile_mesh[v / 128]] for (V, 3) rows, each output one fmaf chain x0 R0j, + x1 R1j, + x2 R2j; a row
// whose tile names no mesh of R is NaN.  x and out may be the same array (each thread reads its row before writing it).
__global__ void __launch_bounds__(kThreads) rotate_rows_kernel(const float* x, int64_t V, const float* __restrict__ R,
                                                               int n_meshes, const int32_t* __restrict__ tile_mesh,
                                                               float* out) {
  const int64_t v = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (v >= V) return;
  const int b = tile_mesh[v >> 7];
  const float x0 = x[3 * v], x1 = x[3 * v + 1], x2 = x[3 * v + 2];
  float y[3];
  if (b < 0 || b >= n_meshes) {
    y[0] = y[1] = y[2] = NAN;
  } else {
    const float* r = R + (int64_t)b * 9;
#pragma unroll
    for (int j = 0; j < 3; ++j) y[j] = fmaf(x2, __ldg(r + 6 + j), fmaf(x1, __ldg(r + 3 + j), x0 * __ldg(r + j)));
  }
  out[3 * v] = y[0];
  out[3 * v + 1] = y[1];
  out[3 * v + 2] = y[2];
}

}  // namespace

extern "C" int dn_rotate_rows(const float* x, int64_t V, const float* R, int n_meshes, const int32_t* tile_mesh,
                              float* out, dn_stream_t stream) {
  if (!x || !R || !tile_mesh || !out || V < 128 || V % 128 || n_meshes < 1) return DN_ERR_INVALID_ARGUMENT;
  const int64_t blocks = (V + kThreads - 1) / kThreads;
  rotate_rows_kernel<<<(unsigned)blocks, kThreads, 0, (cudaStream_t)stream>>>(x, V, R, n_meshes, tile_mesh, out);
  DN_LAUNCH_CHECK();
  return DN_OK;
}

