// Joint rotations of an existing glTF skeleton fitted to a fixed-topology vertex animation (DESIGN.md §21).
// actionmesh_b200/rig.py drives the kernels and tests/rig_ref.py restates them in numpy float64 with the same operation
// order.  Every fp64 product, sum, quotient and square root is an explicit round-to-nearest intrinsic (fp64.cuh), every sum
// runs in a fixed order, and atomics are used only for a maximum: two runs give identical bits.
//
// Joints are numbered in a topological order (parent[j] < j, -1 for a root), so the subtree of joint j is [j, end_j) when
// the order is depth-first.  Transforms are 12 doubles (fp64.cuh): L row-major, then t.
//   rotations (T, J, 9) local R_j^t;  translations (T, J, 3) local translations (only the roots' change);  scale (J, 3);
//   above (J, 12) the fixed world transform above each root joint;  binds (NB, 12) bind matrices, bind_joint (NB) their
//   joints;  world (T, J, 12) G_j^t;  skin (T, NB, 12) K_b^t = G_{bind_joint[b]}^t B_b.
//   Vertex i: points (V, 3) the position its binds act on, rest (V, 3), vertices (T, V, 3), slots (V, 8) of (bind, weight),
//   used slots first (weight > 0); a vertex whose slot 0 is unused is static and shows rest[i].
//
//  forward       G_j = P_j (T(tau_j) R_j S_j), P_j = G_parent or above[j], in joint order; then K_b = G_{j_b} B_b.
//  rotation      joint j: forward, then per frame H_w = sum_i d_i e_i^T over j's vertex list (256-item tiles, tiles in
//                order) with d = a - m f, e = (v - c) - m f, a / c / m the subtree's / the others' blended positions / the
//                subtree's weight, f the translation of P_j T(tau_j); R_j = Horn(R_j^T (L^T (H_w L))), L the linear part of P_j.
//  translation   root j: forward, then tau_j += A^-1 (sum m (v - v^) / sum m^2) over j's vertex list (kept when sum m^2 == 0).
//  error         forward, then sum_i |v^_i - v_i|^2 per frame, their sum, and the maximum |v^_i - v_i|^2.
#include <cuda_runtime.h>
#include <cstdint>
#include "common.cuh"
#include "fp64.cuh"
#include "../../include/actionmesh_b200.h"

namespace amb {
namespace {

constexpr int RG_MAX_JOINTS = 1024;
constexpr int RG_MAX_BINDS = 1 << 20;
constexpr int RG_SLOTS = 8;
constexpr int RG_NMOM = 9;          // the largest moment count of a pass: H_w
constexpr int RG_FK_THREADS = 128;

struct Rig {
  const int32_t* parent;
  int J;
  const double* scale;
  const double* above;
  const double* binds;
  const int32_t* bind_joint;
  int NB;
  double* world;
  double* skin;
};

// out = A o B: linear ((A_a0 B_0b + A_a1 B_1b) + A_a2 B_2b), translation apply_xf(A, t_B)
__device__ __forceinline__ void compose(const double* __restrict__ A, const double* __restrict__ B, double* __restrict__ out) {
  double o[12];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b)
      o[3 * a + b] = dadd(dadd(dmul(A[3 * a], B[b]), dmul(A[3 * a + 1], B[3 + b])), dmul(A[3 * a + 2], B[6 + b]));
  const V3 t = apply_xf(A, {B[9], B[10], B[11]});
  o[9] = t.x;
  o[10] = t.y;
  o[11] = t.z;
#pragma unroll
  for (int k = 0; k < 12; ++k) out[k] = o[k];
}

// P_j: the parent's world transform, or the fixed transform above a root
__device__ __forceinline__ const double* parent_xf(const Rig& r, int t, int j) {
  const int p = r.parent[j];
  return p >= 0 ? r.world + ((int64_t)t * r.J + p) * 12 : r.above + (int64_t)j * 12;
}

// One block per frame: thread 0 walks the joints in order (local = [R diag(s) | tau], R_ab s_b rounded once), then the
// block computes every K_b.
__global__ void __launch_bounds__(RG_FK_THREADS) rig_forward_kernel(Rig r, const double* __restrict__ rotations,
                                                                   const double* __restrict__ translations) {
  const int t = blockIdx.x;
  if (threadIdx.x == 0) {
    for (int j = 0; j < r.J; ++j) {
      const double* R = rotations + ((int64_t)t * r.J + j) * 9;
      const double* tau = translations + ((int64_t)t * r.J + j) * 3;
      const double* s = r.scale + 3 * j;
      double local[12];
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) local[3 * a + b] = dmul(R[3 * a + b], s[b]);
      local[9] = tau[0];
      local[10] = tau[1];
      local[11] = tau[2];
      compose(parent_xf(r, t, j), local, r.world + ((int64_t)t * r.J + j) * 12);
    }
  }
  __syncthreads();
  for (int b = threadIdx.x; b < r.NB; b += blockDim.x)
    compose(r.world + ((int64_t)t * r.J + r.bind_joint[b]) * 12, r.binds + (int64_t)b * 12,
            r.skin + ((int64_t)t * r.NB + b) * 12);
}

// Over the used slots of vertex i in slot order, from 0: sub = sum of w u over the slots whose joint is in [j0, j1), rest =
// the sum over the others, m = the sum of the weights in [j0, j1), all = the sum over every slot.
struct Blend {
  V3 sub, rest, all;
  double m;
};

__device__ __forceinline__ Blend blend_split(const Rig& r, const double* __restrict__ skin_t, const int32_t* __restrict__ bind,
                                             const double* __restrict__ weight, int64_t i, V3 p, int j0, int j1) {
  Blend o = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, 0.0};
#pragma unroll
  for (int k = 0; k < RG_SLOTS; ++k) {
    const double w = weight[RG_SLOTS * i + k];
    if (w > 0.0) {
      const int b = bind[RG_SLOTS * i + k];
      const int jb = r.bind_joint[b];
      const V3 u = apply_xf(skin_t + 12 * (int64_t)b, p);
      const V3 wu = {dmul(w, u.x), dmul(w, u.y), dmul(w, u.z)};
      o.all = {dadd(o.all.x, wu.x), dadd(o.all.y, wu.y), dadd(o.all.z, wu.z)};
      if (jb >= j0 && jb < j1) {
        o.sub = {dadd(o.sub.x, wu.x), dadd(o.sub.y, wu.y), dadd(o.sub.z, wu.z)};
        o.m = dadd(o.m, w);
      } else {
        o.rest = {dadd(o.rest.x, wu.x), dadd(o.rest.y, wu.y), dadd(o.rest.z, wu.z)};
      }
    }
  }
  return o;
}

// grid (tiles of the list, T): partials[(t * tiles + tile) * 9 + 3 l + n] = the tile's sum of d_l e_n.
__global__ void __launch_bounds__(FP64_THREADS) rig_rotation_partial_kernel(Rig r, const double* __restrict__ translations,
                                                                           const double* __restrict__ points,
                                                                           const double* __restrict__ verts, int64_t V,
                                                                           const int32_t* __restrict__ bind,
                                                                           const double* __restrict__ weight,
                                                                           const int32_t* __restrict__ list, int64_t n,
                                                                           int joint, int end, double* __restrict__ partials) {
  __shared__ double red[FP64_THREADS / 32][RG_NMOM];
  const int t = blockIdx.y;
  const int64_t idx = (int64_t)blockIdx.x * FP64_THREADS + threadIdx.x;
  double c[RG_NMOM];
#pragma unroll
  for (int k = 0; k < RG_NMOM; ++k) c[k] = 0.0;
  if (idx < n) {
    const int64_t i = list[idx];
    const double* tau = translations + ((int64_t)t * r.J + joint) * 3;
    const V3 f = apply_xf(parent_xf(r, t, joint), {tau[0], tau[1], tau[2]});
    const Blend b = blend_split(r, r.skin + (int64_t)t * r.NB * 12, bind, weight, i, load3(points, i), joint, end);
    const V3 v = load3(verts, (int64_t)t * V + i);
    const double d[3] = {dsub(b.sub.x, dmul(b.m, f.x)), dsub(b.sub.y, dmul(b.m, f.y)), dsub(b.sub.z, dmul(b.m, f.z))};
    const double e[3] = {dsub(dsub(v.x, b.rest.x), dmul(b.m, f.x)), dsub(dsub(v.y, b.rest.y), dmul(b.m, f.y)),
                         dsub(dsub(v.z, b.rest.z), dmul(b.m, f.z))};
#pragma unroll
    for (int l = 0; l < 3; ++l)
#pragma unroll
      for (int m = 0; m < 3; ++m) c[3 * l + m] = dmul(d[l], e[m]);
  }
  block_sum<RG_NMOM>(c, red, partials + ((int64_t)t * gridDim.x + blockIdx.x) * RG_NMOM);
}

// One thread per frame: H_w = the tiles' partials in tile order; X = H_w L, Y = L^T X, H = R^T Y (each entry a 3-term sum in
// index order); R_j = Horn(H).
__global__ void rig_rotation_solve_kernel(Rig r, const double* __restrict__ partials, int T, int tiles, int joint,
                                          double* __restrict__ rotations) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  double Hw[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) Hw[k] = 0.0;
  const double* pt = partials + (int64_t)t * tiles * RG_NMOM;
  for (int s = 0; s < tiles; ++s)
#pragma unroll
    for (int k = 0; k < 9; ++k) Hw[k] = dadd(Hw[k], pt[(int64_t)s * RG_NMOM + k]);
  const double* L = parent_xf(r, t, joint);
  double* R = rotations + ((int64_t)t * r.J + joint) * 9;
  double X[9], Y[9], H[3][3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b)
      X[3 * a + b] = dadd(dadd(dmul(Hw[3 * a], L[b]), dmul(Hw[3 * a + 1], L[3 + b])), dmul(Hw[3 * a + 2], L[6 + b]));
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b)
      Y[3 * a + b] = dadd(dadd(dmul(L[a], X[b]), dmul(L[3 + a], X[3 + b])), dmul(L[6 + a], X[6 + b]));
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) H[a][b] = dadd(dadd(dmul(R[a], Y[b]), dmul(R[3 + a], Y[3 + b])), dmul(R[6 + a], Y[6 + b]));
  double Rn[9];
  horn_rotation(H, Rn);
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = Rn[k];
}

// grid (tiles of the list, T): partials[(t * tiles + tile) * 9 + k] = the tile's sums of m^2, m r_x, m r_y, m r_z
// (r = v - v^), slots 4..8 zero.
__global__ void __launch_bounds__(FP64_THREADS) rig_translation_partial_kernel(Rig r, const double* __restrict__ points,
                                                                              const double* __restrict__ verts, int64_t V,
                                                                              const int32_t* __restrict__ bind,
                                                                              const double* __restrict__ weight,
                                                                              const int32_t* __restrict__ list, int64_t n,
                                                                              int joint, int end,
                                                                              double* __restrict__ partials) {
  __shared__ double red[FP64_THREADS / 32][4];
  const int t = blockIdx.y;
  const int64_t idx = (int64_t)blockIdx.x * FP64_THREADS + threadIdx.x;
  double c[4] = {0.0, 0.0, 0.0, 0.0};
  if (idx < n) {
    const int64_t i = list[idx];
    const Blend b = blend_split(r, r.skin + (int64_t)t * r.NB * 12, bind, weight, i, load3(points, i), joint, end);
    const V3 res = sub3(load3(verts, (int64_t)t * V + i), b.all);
    c[0] = dmul(b.m, b.m);
    c[1] = dmul(b.m, res.x);
    c[2] = dmul(b.m, res.y);
    c[3] = dmul(b.m, res.z);
  }
  block_sum<4>(c, red, partials + ((int64_t)t * gridDim.x + blockIdx.x) * RG_NMOM);
}

// One thread per frame: sums in tile order; delta = (sum m r) / (sum m^2); tau_a += ((Ai_a0 delta_0 + Ai_a1 delta_1) +
// Ai_a2 delta_2).  Kept when sum m^2 == 0.
__global__ void rig_translation_solve_kernel(Rig r, const double* __restrict__ partials, int T, int tiles, int joint,
                                             const double* __restrict__ above_inv, double* __restrict__ translations) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  double m[4] = {0.0, 0.0, 0.0, 0.0};
  const double* pt = partials + (int64_t)t * tiles * RG_NMOM;
  for (int s = 0; s < tiles; ++s)
#pragma unroll
    for (int k = 0; k < 4; ++k) m[k] = dadd(m[k], pt[(int64_t)s * RG_NMOM + k]);
  if (!(m[0] > 0.0)) return;
  const double dl[3] = {ddiv(m[1], m[0]), ddiv(m[2], m[0]), ddiv(m[3], m[0])};
  const double* Ai = above_inv + (int64_t)joint * 9;
  double* tau = translations + ((int64_t)t * r.J + joint) * 3;
#pragma unroll
  for (int a = 0; a < 3; ++a)
    tau[a] = dadd(tau[a], dadd(dadd(dmul(Ai[3 * a], dl[0]), dmul(Ai[3 * a + 1], dl[1])), dmul(Ai[3 * a + 2], dl[2])));
}

__global__ void __launch_bounds__(FP64_THREADS) rig_error_partial_kernel(Rig r, const double* __restrict__ rest,
                                                                        const double* __restrict__ points,
                                                                        const double* __restrict__ verts, int64_t V,
                                                                        const int32_t* __restrict__ bind,
                                                                        const double* __restrict__ weight,
                                                                        double* __restrict__ partials,
                                                                        unsigned long long* __restrict__ max_bits) {
  __shared__ double red[FP64_THREADS / 32][1];
  const int t = blockIdx.y;
  const int64_t i = (int64_t)blockIdx.x * FP64_THREADS + threadIdx.x;
  double d2 = 0.0;
  if (i < V) {
    const V3 vh = weight[RG_SLOTS * i] > 0.0
                      ? blend_split(r, r.skin + (int64_t)t * r.NB * 12, bind, weight, i, load3(points, i), 0, 0).all
                      : load3(rest, i);
    d2 = norm2(sub3(vh, load3(verts, (int64_t)t * V + i)));
  }
  error_tile(d2, red, partials + (int64_t)t * gridDim.x + blockIdx.x, max_bits);
}

}  // namespace
}  // namespace amb

using namespace amb;

#define RG_CHECK_RIG(fn, parent, J, scale, above, rotations, translations, binds, bind_joint, NB, frames, world, skin)     \
  AMB_CHECK_ARG((parent) && (scale) && (above) && (rotations) && (translations) && (binds) && (bind_joint) && (world) &&  \
                    (skin),                                                                                            \
                fn ": null pointer");                                                                                  \
  AMB_CHECK_ARG((J) >= 1 && (J) <= RG_MAX_JOINTS && (NB) >= 1 && (NB) <= RG_MAX_BINDS && (frames) >= 1 &&                \
                    (frames) <= 65535,                                                                                 \
                fn ": bad sizes (joints %d, binds %d, frames %d)", (int)(J), (int)(NB), (int)(frames))

#define RG_CHECK_VERTS(fn, V)                                                                                           \
  AMB_CHECK_ARG((V) >= 1 && (V) < (1ll << 31) - FP64_THREADS, fn ": bad vertex count %lld", (long long)(V))

static Rig make_rig(const int32_t* parent, int J, const double* scale, const double* above, const double* binds,
                    const int32_t* bind_joint, int NB, double* world, double* skin) {
  return Rig{parent, J, scale, above, binds, bind_joint, NB, world, skin};
}

static int launch_forward(const Rig& r, const double* rotations, const double* translations, int frames, cudaStream_t s) {
  rig_forward_kernel<<<frames, RG_FK_THREADS, 0, s>>>(r, rotations, translations);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

extern "C" int amb_rig_scratch_doubles(int frames, int64_t n_vertices, int64_t* out_doubles) {
  AMB_CHECK_ARG(out_doubles, "rig_scratch_doubles: null pointer");
  AMB_CHECK_ARG(frames >= 1 && frames <= 65535, "rig_scratch_doubles: bad frame count %d", frames);
  RG_CHECK_VERTS("rig_scratch_doubles", n_vertices);
  *out_doubles = (int64_t)frames * tiles_of(n_vertices) * RG_NMOM;
  return AMB_OK;
}

extern "C" int amb_rig_forward(const int32_t* parent, int n_joints, const double* scale, const double* above,
                               const double* rotations, const double* translations, const double* binds,
                               const int32_t* bind_joint, int n_binds, int frames, double* world, double* skin,
                               amb_stream_t stream) {
  RG_CHECK_RIG("rig_forward", parent, n_joints, scale, above, rotations, translations, binds, bind_joint, n_binds, frames,
               world, skin);
  return launch_forward(make_rig(parent, n_joints, scale, above, binds, bind_joint, n_binds, world, skin), rotations,
                        translations, frames, (cudaStream_t)stream);
}

extern "C" int amb_rig_rotation_update(const int32_t* parent, int n_joints, const double* scale, const double* above,
                                       double* rotations, const double* translations, const double* binds,
                                       const int32_t* bind_joint, int n_binds, int frames, double* world, double* skin,
                                       const double* points, const double* vertices, int64_t n_vertices,
                                       const int32_t* slot_bind, const double* slot_weight, const int32_t* list,
                                       int64_t n_list, int joint, int subtree_end, double* scratch, amb_stream_t stream) {
  RG_CHECK_RIG("rig_rotation_update", parent, n_joints, scale, above, rotations, translations, binds, bind_joint, n_binds,
               frames, world, skin);
  RG_CHECK_VERTS("rig_rotation_update", n_vertices);
  AMB_CHECK_ARG(points && vertices && slot_bind && slot_weight && scratch && (list || n_list == 0),
                "rig_rotation_update: null pointer");
  AMB_CHECK_ARG(joint >= 0 && joint < subtree_end && subtree_end <= n_joints && n_list >= 0 && n_list <= n_vertices,
                "rig_rotation_update: bad joint %d, subtree end %d or list length %lld (joints %d, vertices %lld)", joint,
                subtree_end, (long long)n_list, n_joints, (long long)n_vertices);
  if (n_list == 0) return AMB_OK;  // a subtree that influences no vertex keeps its rotation
  cudaStream_t s = (cudaStream_t)stream;
  const Rig r = make_rig(parent, n_joints, scale, above, binds, bind_joint, n_binds, world, skin);
  if (int rc = launch_forward(r, rotations, translations, frames, s)) return rc;
  const int tiles = tiles_of(n_list);
  rig_rotation_partial_kernel<<<dim3(tiles, frames), FP64_THREADS, 0, s>>>(r, translations, points, vertices, n_vertices,
                                                                           slot_bind, slot_weight, list, n_list, joint,
                                                                           subtree_end, scratch);
  AMB_CHECK_CUDA(cudaGetLastError());
  rig_rotation_solve_kernel<<<(frames + 63) / 64, 64, 0, s>>>(r, scratch, frames, tiles, joint, rotations);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

extern "C" int amb_rig_translation_update(const int32_t* parent, int n_joints, const double* scale, const double* above,
                                          const double* above_inv, const double* rotations, double* translations,
                                          const double* binds, const int32_t* bind_joint, int n_binds, int frames,
                                          double* world, double* skin, const double* points, const double* vertices,
                                          int64_t n_vertices, const int32_t* slot_bind, const double* slot_weight,
                                          const int32_t* list, int64_t n_list, int joint, int subtree_end, double* scratch,
                                          amb_stream_t stream) {
  RG_CHECK_RIG("rig_translation_update", parent, n_joints, scale, above, rotations, translations, binds, bind_joint,
               n_binds, frames, world, skin);
  RG_CHECK_VERTS("rig_translation_update", n_vertices);
  AMB_CHECK_ARG(above_inv && points && vertices && slot_bind && slot_weight && scratch && (list || n_list == 0),
                "rig_translation_update: null pointer");
  AMB_CHECK_ARG(joint >= 0 && joint < subtree_end && subtree_end <= n_joints && n_list >= 0 && n_list <= n_vertices,
                "rig_translation_update: bad joint %d, subtree end %d or list length %lld (joints %d, vertices %lld)",
                joint, subtree_end, (long long)n_list, n_joints, (long long)n_vertices);
  if (n_list == 0) return AMB_OK;  // sum m^2 == 0: the translation is kept
  cudaStream_t s = (cudaStream_t)stream;
  const Rig r = make_rig(parent, n_joints, scale, above, binds, bind_joint, n_binds, world, skin);
  if (int rc = launch_forward(r, rotations, translations, frames, s)) return rc;
  const int tiles = tiles_of(n_list);
  rig_translation_partial_kernel<<<dim3(tiles, frames), FP64_THREADS, 0, s>>>(r, points, vertices, n_vertices, slot_bind,
                                                                              slot_weight, list, n_list, joint, subtree_end,
                                                                              scratch);
  AMB_CHECK_CUDA(cudaGetLastError());
  rig_translation_solve_kernel<<<(frames + 63) / 64, 64, 0, s>>>(r, scratch, frames, tiles, joint, above_inv, translations);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

extern "C" int amb_rig_error(const int32_t* parent, int n_joints, const double* scale, const double* above,
                             const double* rotations, const double* translations, const double* binds,
                             const int32_t* bind_joint, int n_binds, int frames, double* world, double* skin,
                             const double* rest, const double* points, const double* vertices, int64_t n_vertices,
                             const int32_t* slot_bind, const double* slot_weight, double* scratch, double* frame_errors,
                             double* max_error2, amb_stream_t stream) {
  RG_CHECK_RIG("rig_error", parent, n_joints, scale, above, rotations, translations, binds, bind_joint, n_binds, frames,
               world, skin);
  RG_CHECK_VERTS("rig_error", n_vertices);
  AMB_CHECK_ARG(rest && points && vertices && slot_bind && slot_weight && scratch && frame_errors && max_error2,
                "rig_error: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  const Rig r = make_rig(parent, n_joints, scale, above, binds, bind_joint, n_binds, world, skin);
  if (int rc = launch_forward(r, rotations, translations, frames, s)) return rc;
  const int tiles = tiles_of(n_vertices);
  AMB_CHECK_CUDA(cudaMemsetAsync(max_error2, 0, sizeof(double), s));
  rig_error_partial_kernel<<<dim3(tiles, frames), FP64_THREADS, 0, s>>>(
      r, rest, points, vertices, n_vertices, slot_bind, slot_weight, scratch,
      reinterpret_cast<unsigned long long*>(max_error2));
  AMB_CHECK_CUDA(cudaGetLastError());
  error_sum_kernel<<<1, 256, 0, s>>>(scratch, frames, tiles, frame_errors);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}
