// Stage 0's anchor mesh: octree refinement of the decoded logit grid and dual marching cubes.
//
// Grids are cubic, n points per side, fp32 or uint8, x slowest: element (x, y, z) at (x * n + y) * n + z.
//
// Octree refinement (third_party/TripoSG/triposg/inference_utils.py:318-460, flash_extract_geometry):
//   near_surface    extract_near_surface_volume_fn (:203-297) + `|logit| < 0.95` (:403)
//   dilate3         the ones-Conv3d(3, padding=1) dilation (:361-362,410-416): out = any of the 27 neighbours > 0
//   mark_upsampled  next_index[2x, 2y, 2z] = 1 (:414)
//   compact_points  torch.where(next_index > 0) and `idx * resolution + bbox_min` in fp32 (:417-421)
//   fill / scatter  torch.full(-10000) and next_logits[nidx] = logits (:401,457)
// Compactions (points, DMC vertices and faces) are count -> scan -> emit passes (scan.cuh), so every output is in grid order
// and two runs give identical arrays.
#include <cuda_runtime.h>
#include <cstdint>
#include "common.cuh"
#include "dmc_table.cuh"
#include "scan.cuh"
#include "../../include/actionmesh_b200.h"

namespace amb {
namespace {

// ---- octree refinement -------------------------------------------------------------------------------------------------

__device__ __forceinline__ float sign_of(float v) { return v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f); }  // torch.sign

__global__ void near_surface_kernel(const float* __restrict__ g, int n, uint8_t* __restrict__ out) {
  const long long total = (long long)n * n * n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(i % n), y = (int)((i / n) % n), x = (int)(i / ((long long)n * n));
    const float v = g[i];
    const float s = sign_of(v);
    bool differs = false;
    // the 6 face neighbours, replicate padding at the border; an invalid (<= -9000) neighbour counts as v itself
    const int nb[6][3] = {{x + 1, y, z}, {x - 1, y, z}, {x, y + 1, z}, {x, y - 1, z}, {x, y, z + 1}, {x, y, z - 1}};
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const int a = min(max(nb[k][0], 0), n - 1), b = min(max(nb[k][1], 0), n - 1), c = min(max(nb[k][2], 0), n - 1);
      float w = g[((long long)a * n + b) * n + c];
      if (!(w > -9000.f)) w = v;
      differs |= sign_of(w) != s;
    }
    out[i] = (uint8_t)(((differs && v > -9000.f) || fabsf(v) < 0.95f) ? 1 : 0);
  }
}

__global__ void dilate3_kernel(const uint8_t* __restrict__ in, int n, uint8_t* __restrict__ out) {
  const long long total = (long long)n * n * n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(i % n), y = (int)((i / n) % n), x = (int)(i / ((long long)n * n));
    uint8_t any = 0;
    for (int a = max(x - 1, 0); a <= min(x + 1, n - 1) && !any; ++a)
      for (int b = max(y - 1, 0); b <= min(y + 1, n - 1) && !any; ++b)
        for (int c = max(z - 1, 0); c <= min(z + 1, n - 1); ++c)
          if (in[((long long)a * n + b) * n + c]) { any = 1; break; }
    out[i] = any;
  }
}

__global__ void mark_upsampled_kernel(const uint8_t* __restrict__ coarse, int n, uint8_t* __restrict__ fine) {
  const int m = 2 * n - 1;
  const long long total = (long long)n * n * n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(i % n), y = (int)((i / n) % n), x = (int)(i / ((long long)n * n));
    fine[((long long)(2 * x) * m + 2 * y) * m + 2 * z] = coarse[i] ? 1 : 0;
  }
}

struct CompactPoints {
  const uint8_t* mask;
  int n;
  float rx, ry, rz, ox, oy, oz;  // fp32 resolution and bbox_min
  float* xyz;                    // (P, 3)
  int32_t* index;                // (P) linear grid index
  __device__ int count(long long i) const { return mask[i] ? 1 : 0; }
  __device__ void emit(long long i, int off) const {
    if (!mask[i]) return;
    const int z = (int)(i % n), y = (int)((i / n) % n), x = (int)(i / ((long long)n * n));
    // torch: (int64 idx -> fp32) * fp32 resolution, then + fp32 bbox_min, each op rounded on its own
    xyz[3LL * off + 0] = __fadd_rn(__fmul_rn((float)x, rx), ox);
    xyz[3LL * off + 1] = __fadd_rn(__fmul_rn((float)y, ry), oy);
    xyz[3LL * off + 2] = __fadd_rn(__fmul_rn((float)z, rz), oz);
    index[off] = (int32_t)i;
  }
};

__global__ void fill_kernel(float* __restrict__ g, long long total, float value) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    g[i] = value;
}

__global__ void replace_kernel(float* __restrict__ g, long long total, float from, float to) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    if (g[i] == from) g[i] = to;
}

__global__ void scatter_kernel(const float* __restrict__ values, int64_t ld, const int32_t* __restrict__ index, int count,
                               float* __restrict__ g) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x)
    g[index[i]] = values[i * ld];
}

// ---- dual marching cubes ------------------------------------------------------------------------------------------------
// Cells are indexed like points of an (n-1)^3 grid.  case = bit c set when corner c is inside (logit > 0); a cell with a
// non-finite corner gets case 0 (no patches).  A sign-changing edge makes every cell around it a case other than 0 or 255,
// so case 0 next to a crossing edge means "invalid cell".

__device__ __forceinline__ bool inside(float v) { return v > 0.f; }

__global__ void dmc_case_kernel(const float* __restrict__ g, int n, uint8_t* __restrict__ cases) {
  const int m = n - 1;
  const long long total = (long long)m * m * m;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(i % m), y = (int)((i / m) % m), x = (int)(i / ((long long)m * m));
    int c = 0;
    bool ok = true;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float v = g[((long long)(x + (k & 1)) * n + y + ((k >> 1) & 1)) * n + z + ((k >> 2) & 1)];
      ok &= isfinite(v);
      c |= inside(v) ? (1 << k) : 0;
    }
    cases[i] = ok ? (uint8_t)c : (uint8_t)0;
  }
}

struct DmcVertices {
  const float* g;
  const uint8_t* cases;
  int n;
  int32_t* voff;   // (n-1)^3 first vertex of each cell
  float* verts;    // (V, 3) in grid-index units
  __device__ int count(long long i) const { return kDmcPatchCount[cases[i]]; }
  __device__ void emit(long long i, int off) const {
    const int cs = cases[i];
    voff[i] = off;
    const int np = kDmcPatchCount[cs];
    if (!np) return;
    const int m = n - 1;
    const int z = (int)(i % m), y = (int)((i / m) % m), x = (int)(i / ((long long)m * m));
    float val[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) val[k] = g[((long long)(x + (k & 1)) * n + y + ((k >> 1) & 1)) * n + z + ((k >> 2) & 1)];
    for (int p = 0; p < np; ++p) {
      float s[3] = {0.f, 0.f, 0.f};
      int cnt = 0;
      for (int e = 0; e < 12; ++e) {
        if (kDmcPatchOfEdge[cs][e] != p) continue;
        const int axis = e >> 2, u = e & 1, v = (e >> 1) & 1;
        const int o0 = axis == 0 ? 1 : 0, o1 = axis == 2 ? 1 : 2;   // the other two axes in increasing order
        int off0[3] = {0, 0, 0};
        off0[o0] = u;
        off0[o1] = v;
        const int c0 = off0[0] | (off0[1] << 1) | (off0[2] << 2);
        const int c1 = c0 | (1 << axis);
        const float t = __fdiv_rn(val[c0], __fsub_rn(val[c0], val[c1]));   // linear interpolation of the crossing
        s[axis] = __fadd_rn(s[axis], t);
        s[o0] = __fadd_rn(s[o0], (float)u);
        s[o1] = __fadd_rn(s[o1], (float)v);
        ++cnt;
      }
      const float fc = (float)cnt;
      verts[3LL * (off + p) + 0] = __fadd_rn(__fdiv_rn(s[0], fc), (float)x);
      verts[3LL * (off + p) + 1] = __fadd_rn(__fdiv_rn(s[1], fc), (float)y);
      verts[3LL * (off + p) + 2] = __fadd_rn(__fdiv_rn(s[2], fc), (float)z);
    }
  }
};

// One quad per sign-changing grid edge p -> p + e_axis whose 4 surrounding cells exist and are valid.  The cells are visited
// counter-clockwise around +axis (normal +axis); the quad is reversed when p is outside, so the normal points from inside
// (logit > 0) to outside.  Split: (q0, q1, q2), (q0, q2, q3).
struct DmcFaces {
  const float* g;
  const uint8_t* cases;
  const int32_t* voff;
  int n;
  int32_t* faces;  // (F, 3)

  __device__ bool quad(long long i, int axis, int q[4]) const {
    const int z = (int)(i % n), y = (int)((i / n) % n), x = (int)(i / ((long long)n * n));
    const int p[3] = {x, y, z};
    if (p[axis] >= n - 1) return false;
    const int b = (axis + 1) % 3, c = (axis + 2) % 3;
    if (p[b] < 1 || p[b] > n - 2 || p[c] < 1 || p[c] > n - 2) return false;
    const float v0 = g[i];
    const long long step = axis == 0 ? (long long)n * n : (axis == 1 ? n : 1);
    const float v1 = g[i + step];
    if (!isfinite(v0) || !isfinite(v1) || inside(v0) == inside(v1)) return false;
    const int m = n - 1;
    const int db[4] = {-1, 0, 0, -1}, dc[4] = {-1, -1, 0, 0};
    for (int k = 0; k < 4; ++k) {
      int cc[3] = {p[0], p[1], p[2]};
      cc[b] += db[k];
      cc[c] += dc[k];
      const long long cell = ((long long)cc[0] * m + cc[1]) * m + cc[2];
      const int cs = cases[cell];
      if (cs == 0) return false;
      int bits[3] = {0, 0, 0};
      bits[b] = -db[k];
      bits[c] = -dc[k];
      const int o0 = axis == 0 ? 1 : 0, o1 = axis == 2 ? 1 : 2;
      const int e = 4 * axis + bits[o0] + 2 * bits[o1];
      q[k] = voff[cell] + kDmcPatchOfEdge[cs][e];
    }
    if (!inside(v0)) {
      const int t = q[1];
      q[1] = q[3];
      q[3] = t;
    }
    return true;
  }
  __device__ int count(long long i) const {
    int q[4], s = 0;
    for (int a = 0; a < 3; ++a) s += quad(i, a, q) ? 2 : 0;
    return s;
  }
  __device__ void emit(long long i, int off) const {
    int q[4];
    for (int a = 0; a < 3; ++a) {
      if (!quad(i, a, q)) continue;
      int32_t* f = faces + 3LL * off;
      f[0] = q[0]; f[1] = q[1]; f[2] = q[2];
      f[3] = q[0]; f[4] = q[2]; f[5] = q[3];
      off += 2;
    }
  }
};

}  // namespace
}  // namespace amb

using namespace amb;

extern "C" {

int amb_octree_near_surface(const float* grid, int n, uint8_t* mask, amb_stream_t stream) {
  AMB_CHECK_ARG(grid && mask && n >= 2, "octree_near_surface: bad arguments");
  const long long total = (long long)n * n * n;
  near_surface_kernel<<<blocks_for(total, 256), 256, 0, (cudaStream_t)stream>>>(grid, n, mask);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_octree_dilate(const uint8_t* in, int n, uint8_t* out, amb_stream_t stream) {
  AMB_CHECK_ARG(in && out && in != out && n >= 1, "octree_dilate: bad arguments");
  const long long total = (long long)n * n * n;
  dilate3_kernel<<<blocks_for(total, 256), 256, 0, (cudaStream_t)stream>>>(in, n, out);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_octree_mark_upsampled(const uint8_t* coarse, int n, uint8_t* fine, amb_stream_t stream) {
  AMB_CHECK_ARG(coarse && fine && n >= 1, "octree_mark_upsampled: bad arguments");
  const long long m = 2LL * n - 1;
  AMB_CHECK_CUDA(cudaMemsetAsync(fine, 0, m * m * m, (cudaStream_t)stream));
  const long long total = (long long)n * n * n;
  mark_upsampled_kernel<<<blocks_for(total, 256), 256, 0, (cudaStream_t)stream>>>(coarse, n, fine);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_scan_scratch_ints(int64_t n_items, int64_t* out_ints) {
  AMB_CHECK_ARG(out_ints && n_items >= 0, "scan_scratch_ints: bad arguments");
  *out_ints = scan_tiles(n_items) + 1;
  return AMB_OK;
}

int amb_octree_count_points(const uint8_t* mask, int n, int32_t* scratch, amb_stream_t stream) {
  AMB_CHECK_ARG(mask && scratch && n >= 1, "octree_count_points: bad arguments");
  AMB_CHECK_ARG((long long)n * n * n < (1LL << 31), "octree_count_points: grid of %d^3 is too large", n);
  CompactPoints f{mask, n, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, nullptr, nullptr};
  return scan_count((long long)n * n * n, f, scratch, (cudaStream_t)stream);
}

int amb_octree_emit_points(const uint8_t* mask, int n, const int32_t* scratch, const float* resolution3_host,
                           const float* bbox_min3_host, float* xyz, int32_t* index, amb_stream_t stream) {
  AMB_CHECK_ARG(mask && scratch && resolution3_host && bbox_min3_host && xyz && index && n >= 1,
                "octree_emit_points: null pointer");
  CompactPoints f{mask, n, resolution3_host[0], resolution3_host[1], resolution3_host[2], bbox_min3_host[0],
                  bbox_min3_host[1], bbox_min3_host[2], xyz, index};
  return scan_emit((long long)n * n * n, f, scratch, (cudaStream_t)stream);
}

int amb_grid_fill(float* grid, int64_t count, float value, amb_stream_t stream) {
  AMB_CHECK_ARG(grid && count >= 0, "grid_fill: bad arguments");
  if (!count) return AMB_OK;
  fill_kernel<<<blocks_for(count, 256), 256, 0, (cudaStream_t)stream>>>(grid, count, value);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_grid_replace(float* grid, int64_t count, float from, float to, amb_stream_t stream) {
  AMB_CHECK_ARG(grid && count >= 0, "grid_replace: bad arguments");
  if (!count) return AMB_OK;
  replace_kernel<<<blocks_for(count, 256), 256, 0, (cudaStream_t)stream>>>(grid, count, from, to);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_grid_scatter(const float* values, int64_t ld, const int32_t* index, int count, float* grid, amb_stream_t stream) {
  AMB_CHECK_ARG(values && index && grid && ld >= 1 && count >= 0, "grid_scatter: bad arguments");
  if (!count) return AMB_OK;
  scatter_kernel<<<blocks_for(count, 256), 256, 0, (cudaStream_t)stream>>>(values, ld, index, count, grid);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_dmc_count(const float* grid, int n, uint8_t* cases, int32_t* vertex_scratch, int32_t* face_scratch,
                  amb_stream_t stream) {
  AMB_CHECK_ARG(grid && cases && vertex_scratch && face_scratch, "dmc_count: null pointer");
  AMB_CHECK_ARG(n >= 2 && (long long)n * n * n < (1LL << 31), "dmc_count: grid side %d out of range", n);
  cudaStream_t st = (cudaStream_t)stream;
  const long long m = n - 1;
  dmc_case_kernel<<<blocks_for(m * m * m, 256), 256, 0, st>>>(grid, n, cases);
  AMB_CHECK_CUDA(cudaGetLastError());
  DmcVertices fv{grid, cases, n, nullptr, nullptr};
  int rc = scan_count(m * m * m, fv, vertex_scratch, st);
  if (rc) return rc;
  DmcFaces ff{grid, cases, nullptr, n, nullptr};
  return scan_count((long long)n * n * n, ff, face_scratch, st);
}

int amb_dmc_emit(const float* grid, int n, const uint8_t* cases, const int32_t* vertex_scratch, const int32_t* face_scratch,
                 int32_t* vertex_offsets, float* vertices, int32_t* faces, amb_stream_t stream) {
  AMB_CHECK_ARG(grid && cases && vertex_scratch && face_scratch && vertex_offsets && vertices && faces, "dmc_emit: null pointer");
  AMB_CHECK_ARG(n >= 2 && (long long)n * n * n < (1LL << 31), "dmc_emit: grid side %d out of range", n);
  cudaStream_t st = (cudaStream_t)stream;
  const long long m = n - 1;
  DmcVertices fv{grid, cases, n, vertex_offsets, vertices};
  int rc = scan_emit(m * m * m, fv, vertex_scratch, st);
  if (rc) return rc;
  DmcFaces ff{grid, cases, vertex_offsets, n, faces};
  return scan_emit((long long)n * n * n, ff, face_scratch, st);
}

}  // extern "C"
