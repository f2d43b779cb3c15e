// Gradient ICP for the ActionBench scores CD-3D / CD-4D / CD-M (actionbench/icp.py:53-112).
//
// The reference aligns a predicted point cloud x (P points) to the ground truth g (Q points) with 200 Adam steps over 24
// candidate rotations at once: for candidate n, y_i = (s ⊙ x_i) @ R + T (row vectors, icp.py:94) with R = R_init[n] @
// rotation_6d_to_matrix(d6), and the loss is pytorch3d's chamfer_distance (squared L2, mean over points, both directions).
// Here F frames x C candidates are one batch, and every step is two launches of our own:
//
//  amb_icp_chamfer_grad: both nearest-neighbour directions of every (frame, candidate) in one grid.
//   * pred->gt blocks: a thread owns one pred point under ICP_CB candidate transforms; the gt set (shared by all candidates)
//     streams through shared memory, so each staged point feeds ICP_CB distance evaluations.
//   * gt->pred blocks: a thread owns ICP_QB gt points of one candidate; the block stages that candidate's transformed
//     prediction (the transform is recomputed, bit for bit, when the nearest point's contribution is formed).
//   Every query adds its own contribution right after its search (nothing is scattered): the squared distance, e = y - g and
//   x ⊗ e over the UNTRANSFORMED x.  Each block reduces them in a fixed order (fp64) into its own partial slot; a second
//   kernel sums the slots in slot order.  No float atomics: two runs give identical bits.  Ties go to the lowest index.
//  amb_icp_adam_step: one thread per (frame, candidate): the closed-form backward through R = R_init @ M(d6), torch's Adam,
//   the reference's best-candidate bookkeeping, and R for the next step.
#include <cmath>

#include "common.cuh"
#include "../../include/actionmesh_b200.h"

namespace amb {

constexpr int ICP_THREADS = 128;
constexpr int ICP_TILE = 1024;   // staged points per shared-memory tile (16 KB of float4)
constexpr int ICP_CB = 8;        // candidates per pred->gt thread
constexpr int ICP_QB = 4;        // gt points per gt->pred thread
constexpr int ICP_NSUM = 13;     // squared distance, e (3), x ⊗ e (9)
constexpr int ICP_MAX_C = 1024;  // the Adam step runs one block of C threads per frame

struct IcpGrid {
  int groups;   // candidate groups of ICP_CB
  int tiles_p;  // pred->gt blocks per (frame, group) = partial slots of the pred->gt direction
  int tiles_q;  // gt->pred blocks per (frame, candidate)
  __host__ __device__ int slots() const { return tiles_p + tiles_q; }
};

static IcpGrid icp_grid(int c, int p, int q) {
  return {(c + ICP_CB - 1) / ICP_CB, (p + ICP_THREADS - 1) / ICP_THREADS,
          (q + ICP_THREADS * ICP_QB - 1) / (ICP_THREADS * ICP_QB)};
}

// y = (s ⊙ x) @ R + T, every operation rounded on its own in this order (the gt->pred search and its contribution must agree).
__device__ __forceinline__ float3 icp_transform(const float* __restrict__ rot, const float* __restrict__ par, float3 x) {
  const float a = __fmul_rn(par[9], x.x), b = __fmul_rn(par[10], x.y), c = __fmul_rn(par[11], x.z);
  float3 y;
  y.x = __fadd_rn(__fmaf_rn(c, rot[6], __fmaf_rn(b, rot[3], __fmul_rn(a, rot[0]))), par[0]);
  y.y = __fadd_rn(__fmaf_rn(c, rot[7], __fmaf_rn(b, rot[4], __fmul_rn(a, rot[1]))), par[1]);
  y.z = __fadd_rn(__fmaf_rn(c, rot[8], __fmaf_rn(b, rot[5], __fmul_rn(a, rot[2]))), par[2]);
  return y;
}

__device__ __forceinline__ float icp_dist2(float3 a, float4 b) {
  const float dx = __fsub_rn(a.x, b.x), dy = __fsub_rn(a.y, b.y), dz = __fsub_rn(a.z, b.z);
  return __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
}

__device__ __forceinline__ float3 load3(const float* p, int64_t i) { return make_float3(p[3 * i], p[3 * i + 1], p[3 * i + 2]); }

// One query's contribution: v[0] = |y - g|^2, v[1..3] = e = y - g, v[4..12] = x ⊗ e (row-major, x index first).
__device__ __forceinline__ void icp_contribution(float3 x, float3 y, float3 g, double* v) {
  const double e[3] = {__fsub_rn(y.x, g.x), __fsub_rn(y.y, g.y), __fsub_rn(y.z, g.z)};
  const double xs[3] = {x.x, x.y, x.z};
  v[0] = e[0] * e[0] + e[1] * e[1] + e[2] * e[2];
  for (int l = 0; l < 3; ++l) v[1 + l] = e[l];
  for (int k = 0; k < 3; ++k)
    for (int l = 0; l < 3; ++l) v[4 + 3 * k + l] = xs[k] * e[l];
}

// Block sum of v[0..12] in a fixed order (shuffle tree per warp, then warps in order); thread k < 13 writes out[k].
__device__ __forceinline__ void icp_block_store(double* v, double (*red)[ICP_NSUM], double* __restrict__ out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < ICP_NSUM; ++k) {
    double a = v[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_down_sync(0xffffffffu, a, o);
    if (lane == 0) red[warp][k] = a;
  }
  __syncthreads();
  if (threadIdx.x < ICP_NSUM) {
    double a = 0.0;
#pragma unroll
    for (int w = 0; w < ICP_THREADS / 32; ++w) a += red[w][threadIdx.x];
    out[threadIdx.x] = a;
  }
  __syncthreads();
}

// partials: ((frame * C + candidate) * slots + slot) * 13 doubles; slot < tiles_p is a pred->gt block, the rest gt->pred.
__global__ void __launch_bounds__(ICP_THREADS) icp_nn_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                                                             int C, int P, int Q, const float* __restrict__ rot,
                                                             const float* __restrict__ params, IcpGrid grid,
                                                             double* __restrict__ partials) {
  __shared__ float4 tile[ICP_TILE];
  __shared__ double red[ICP_THREADS / 32][ICP_NSUM];
  const int64_t n_pg = (int64_t)grid.groups * grid.tiles_p;  // pred->gt blocks per frame
  const int64_t per_frame = n_pg + (int64_t)C * grid.tiles_q;
  const int f = (int)(blockIdx.x / per_frame);
  int64_t b = blockIdx.x % per_frame;
  const float* xs = pred + (int64_t)f * P * 3;
  const float* gs = gt + (int64_t)f * Q * 3;
  const int slots = grid.slots();

  if (b < n_pg) {
    // ---- pred -> gt: one pred point, ICP_CB candidates
    const int group = (int)(b / grid.tiles_p), ptile = (int)(b % grid.tiles_p);
    const int c0 = group * ICP_CB;
    const int i = ptile * ICP_THREADS + threadIdx.x;
    const bool live = i < P;
    const float3 x = load3(xs, live ? i : 0);
    float3 y[ICP_CB];
    float bd[ICP_CB];
    int bi[ICP_CB];
#pragma unroll
    for (int k = 0; k < ICP_CB; ++k) {
      const int64_t fc = (int64_t)f * C + min(c0 + k, C - 1);
      y[k] = icp_transform(rot + fc * 9, params + fc * 12, x);
      bd[k] = INFINITY;
      bi[k] = 0;
    }
    for (int t0 = 0; t0 < Q; t0 += ICP_TILE) {
      const int cnt = min(ICP_TILE, Q - t0);
      __syncthreads();
      for (int j = threadIdx.x; j < cnt; j += ICP_THREADS) {
        const float3 g = load3(gs, t0 + j);
        tile[j] = make_float4(g.x, g.y, g.z, 0.f);
      }
      __syncthreads();
#pragma unroll 2
      for (int j = 0; j < cnt; ++j) {
        const float4 g = tile[j];
#pragma unroll
        for (int k = 0; k < ICP_CB; ++k) {
          const float d = icp_dist2(y[k], g);
          if (d < bd[k]) {
            bd[k] = d;
            bi[k] = t0 + j;
          }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < ICP_CB; ++k) {
      double v[ICP_NSUM];
      if (live) {
        icp_contribution(x, y[k], load3(gs, bi[k]), v);
      } else {
        for (int e = 0; e < ICP_NSUM; ++e) v[e] = 0.0;
      }
      const int c = c0 + k;
      double* out = partials + (((int64_t)f * C + min(c, C - 1)) * slots + ptile) * ICP_NSUM;
      if (c < C) icp_block_store(v, red, out);  // block-uniform condition
    }
  } else {
    // ---- gt -> pred: ICP_QB gt points of one candidate
    b -= n_pg;
    const int c = (int)(b / grid.tiles_q), qtile = (int)(b % grid.tiles_q);
    const int64_t fc = (int64_t)f * C + c;
    const float* r = rot + fc * 9;
    const float* par = params + fc * 12;
    float3 g[ICP_QB];
    float bd[ICP_QB];
    int bi[ICP_QB];
#pragma unroll
    for (int u = 0; u < ICP_QB; ++u) {
      const int j = (qtile * ICP_QB + u) * ICP_THREADS + threadIdx.x;
      g[u] = load3(gs, j < Q ? j : 0);
      bd[u] = INFINITY;
      bi[u] = 0;
    }
    for (int t0 = 0; t0 < P; t0 += ICP_TILE) {
      const int cnt = min(ICP_TILE, P - t0);
      __syncthreads();
      for (int i = threadIdx.x; i < cnt; i += ICP_THREADS) {
        const float3 y = icp_transform(r, par, load3(xs, t0 + i));
        tile[i] = make_float4(y.x, y.y, y.z, 0.f);
      }
      __syncthreads();
#pragma unroll 4
      for (int i = 0; i < cnt; ++i) {
        const float4 y = tile[i];
#pragma unroll
        for (int u = 0; u < ICP_QB; ++u) {
          const float d = icp_dist2(g[u], y);
          if (d < bd[u]) {
            bd[u] = d;
            bi[u] = t0 + i;
          }
        }
      }
    }
    double v[ICP_NSUM];
    for (int e = 0; e < ICP_NSUM; ++e) v[e] = 0.0;
    for (int u = 0; u < ICP_QB; ++u) {
      const int j = (qtile * ICP_QB + u) * ICP_THREADS + threadIdx.x;
      if (j < Q) {
        const float3 x = load3(xs, bi[u]);
        double w[ICP_NSUM];
        icp_contribution(x, icp_transform(r, par, x), g[u], w);
        for (int e = 0; e < ICP_NSUM; ++e) v[e] += w[e];
      }
    }
    icp_block_store(v, red, partials + (fc * slots + grid.tiles_p + qtile) * ICP_NSUM);
  }
}

// sums (F, C, 13): loss = S_pg[0]/P + S_gp[0]/Q, then t and A with e scaled by 2/P (pred->gt) and 2/Q (gt->pred).
__global__ void icp_reduce_kernel(const double* __restrict__ partials, int64_t n_fc, int P, int Q, IcpGrid grid,
                                  double* __restrict__ sums) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_fc * ICP_NSUM) return;
  const int64_t fc = idx / ICP_NSUM;
  const int k = (int)(idx % ICP_NSUM);
  const double* p = partials + fc * grid.slots() * ICP_NSUM + k;
  double a = 0.0, b = 0.0;
  for (int s = 0; s < grid.tiles_p; ++s) a += p[(int64_t)s * ICP_NSUM];
  for (int s = grid.tiles_p; s < grid.slots(); ++s) b += p[(int64_t)s * ICP_NSUM];
  const double w = k ? 2.0 : 1.0;
  sums[idx] = w * a / P + w * b / Q;
}

// pytorch3d rotation_6d_to_matrix in fp32: b1 = normalize(a1), b2 = normalize(a2 - (b1 . a2) b1), b3 = b1 x b2, rows b1 b2 b3;
// normalize(v) = v / max(|v|, 1e-12) (F.normalize).
__device__ __forceinline__ void rot6d_to_matrix(const float* d6, float* m) {
  const float n1 = fmaxf(sqrtf(d6[0] * d6[0] + d6[1] * d6[1] + d6[2] * d6[2]), 1e-12f);
  const float b1[3] = {d6[0] / n1, d6[1] / n1, d6[2] / n1};
  const float dot = b1[0] * d6[3] + b1[1] * d6[4] + b1[2] * d6[5];
  const float u[3] = {d6[3] - dot * b1[0], d6[4] - dot * b1[1], d6[5] - dot * b1[2]};
  const float n2 = fmaxf(sqrtf(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]), 1e-12f);
  const float b2[3] = {u[0] / n2, u[1] / n2, u[2] / n2};
  for (int l = 0; l < 3; ++l) {
    m[l] = b1[l];
    m[3 + l] = b2[l];
  }
  m[6] = b1[1] * b2[2] - b1[2] * b2[1];
  m[7] = b1[2] * b2[0] - b1[0] * b2[2];
  m[8] = b1[0] * b2[1] - b1[1] * b2[0];
}

// Backward of normalize at v (|v| = n): g -> (g - b (b . g)) / n with b = v / n, or g / eps where the norm is clamped.
__device__ __forceinline__ void normalize_backward(const double* v, const double* g, double* out) {
  const double n = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  if (n > 1e-12) {
    const double b[3] = {v[0] / n, v[1] / n, v[2] / n};
    const double bg = b[0] * g[0] + b[1] * g[1] + b[2] * g[2];
    for (int l = 0; l < 3; ++l) out[l] = (g[l] - b[l] * bg) / n;
  } else {
    for (int l = 0; l < 3; ++l) out[l] = g[l] / 1e-12;
  }
}

// dL/d(d6) from gm = dL/dM (rows gb1, gb2, gb3), in fp64.
__device__ void rot6d_backward(const float* d6f, const double* gm, double* g6) {
  const double a1[3] = {d6f[0], d6f[1], d6f[2]}, a2[3] = {d6f[3], d6f[4], d6f[5]};
  const double n1 = fmax(sqrt(a1[0] * a1[0] + a1[1] * a1[1] + a1[2] * a1[2]), 1e-12);
  const double b1[3] = {a1[0] / n1, a1[1] / n1, a1[2] / n1};
  const double dot = b1[0] * a2[0] + b1[1] * a2[1] + b1[2] * a2[2];
  const double u[3] = {a2[0] - dot * b1[0], a2[1] - dot * b1[1], a2[2] - dot * b1[2]};
  const double n2 = fmax(sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]), 1e-12);
  const double b2[3] = {u[0] / n2, u[1] / n2, u[2] / n2};
  const double* g3 = gm + 6;
  // b3 = b1 x b2: d/db1 = b2 x g3, d/db2 = g3 x b1
  double gb1[3] = {gm[0] + (b2[1] * g3[2] - b2[2] * g3[1]), gm[1] + (b2[2] * g3[0] - b2[0] * g3[2]),
                   gm[2] + (b2[0] * g3[1] - b2[1] * g3[0])};
  const double gb2[3] = {gm[3] + (g3[1] * b1[2] - g3[2] * b1[1]), gm[4] + (g3[2] * b1[0] - g3[0] * b1[2]),
                         gm[5] + (g3[0] * b1[1] - g3[1] * b1[0])};
  double gu[3];
  normalize_backward(u, gb2, gu);
  // u = a2 - (b1 . a2) b1
  const double b1gu = b1[0] * gu[0] + b1[1] * gu[1] + b1[2] * gu[2];
  for (int l = 0; l < 3; ++l) {
    g6[3 + l] = gu[l] - b1[l] * b1gu;
    gb1[l] -= dot * gu[l] + a2[l] * b1gu;
  }
  normalize_backward(a1, gb1, g6);
}

// One block per frame, one thread per candidate.  params (T 3, d6 6, s 3), m and v: (F, C, 12); rot: (F, C, 9), R of the
// parameters the sums were taken at, replaced by R of the updated parameters; best: (F, 16) = loss, R, T, s.
__global__ void icp_adam_kernel(const double* __restrict__ sums, const float* __restrict__ rot_init, int C, float step_size,
                                float bias2_sqrt, float* __restrict__ params, float* __restrict__ m_state,
                                float* __restrict__ v_state, float* __restrict__ rot, float* __restrict__ best) {
  __shared__ float losses[ICP_MAX_C];
  __shared__ int winner;
  const int f = blockIdx.x, c = threadIdx.x;
  const bool live = c < C;
  const int64_t fc = (int64_t)f * C + (live ? c : 0);
  float r_old[9], par[12];
  float loss = 0.f;
  if (live) {
    const double* sm = sums + fc * ICP_NSUM;
    loss = (float)sm[0];
    for (int e = 0; e < 9; ++e) r_old[e] = rot[fc * 9 + e];
    for (int e = 0; e < 12; ++e) par[e] = params[fc * 12 + e];
    // 1. the reference back-propagates loss.mean() over the C candidates
    const double inv_c = 1.0 / C;
    double t[3], A[9];
    for (int l = 0; l < 3; ++l) t[l] = sm[1 + l] * inv_c;
    for (int e = 0; e < 9; ++e) A[e] = sm[4 + e] * inv_c;
    // 2. dT = t, dR[k,l] = s_k A[k,l], ds_k = sum_l R[k,l] A[k,l]; dM = R_init^T dR
    double grad[12], gm[9];
    for (int l = 0; l < 3; ++l) grad[l] = t[l];
    const float* ri = rot_init + (int64_t)c * 9;
    for (int a = 0; a < 3; ++a)
      for (int l = 0; l < 3; ++l) {
        double acc = 0.0;
        for (int k = 0; k < 3; ++k) acc += (double)ri[3 * k + a] * (double)par[9 + k] * A[3 * k + l];
        gm[3 * a + l] = acc;
      }
    for (int k = 0; k < 3; ++k)
      grad[9 + k] = (double)r_old[3 * k] * A[3 * k] + (double)r_old[3 * k + 1] * A[3 * k + 1] + (double)r_old[3 * k + 2] * A[3 * k + 2];
    rot6d_backward(par + 3, gm, grad + 3);
    // 3. torch.optim.Adam (defaults: betas 0.9 / 0.999, eps 1e-8), the fp32 operations of its foreach path:
    //    m = lerp(m, g, 0.1); v = v * 0.999 + 0.001 g g; p += step_size * m / (sqrt(v) / bias2_sqrt + eps),
    //    step_size = -lr / (1 - 0.9^t) and bias2_sqrt = sqrt(1 - 0.999^t) computed in double by the caller.
    for (int e = 0; e < 12; ++e) {
      const float g = (float)grad[e];
      float m = m_state[fc * 12 + e], v = v_state[fc * 12 + e];
      m = __fmaf_rn(0.1f, __fsub_rn(g, m), m);
      v = __fmaf_rn(__fmul_rn(0.001f, g), g, __fmul_rn(v, 0.999f));
      const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bias2_sqrt), 1e-8f);
      par[e] = __fmaf_rn(step_size, __fdiv_rn(m, denom), par[e]);
      m_state[fc * 12 + e] = m;
      v_state[fc * 12 + e] = v;
      params[fc * 12 + e] = par[e];
    }
    losses[c] = loss;
  }
  __syncthreads();
  // 4. best candidate as icp.py:99-106: `loss.min(0)` of the PRE-step losses (lowest index among equal minima; a NaN anywhere
  //    makes the minimum NaN, and NaN < best is false, so that step records nothing), kept when strictly below the best so far.
  if (c == 0) {
    int w = 0;
    bool nan = false;
    for (int k = 0; k < C; ++k) {
      nan |= isnan(losses[k]);
      if (losses[k] < losses[w]) w = k;
    }
    winner = (!nan && losses[w] < best[(int64_t)f * 16]) ? w : -1;
  }
  __syncthreads();
  if (live && c == winner) {
    // The reference clones R as it was computed for this step (before opt.step()), but T and s after opt.step() updated
    // them in place: the recorded transform mixes the two.  Reproduced as is.
    float* bst = best + (int64_t)f * 16;
    bst[0] = loss;
    for (int e = 0; e < 9; ++e) bst[1 + e] = r_old[e];
    for (int l = 0; l < 3; ++l) {
      bst[10 + l] = par[l];
      bst[13 + l] = par[9 + l];
    }
  }
  // 5. R = R_init @ rotation_6d_to_matrix(d6) for the next step
  if (live) {
    float mm[9];
    rot6d_to_matrix(par + 3, mm);
    const float* ri = rot_init + (int64_t)c * 9;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j)
        rot[fc * 9 + 3 * i + j] = ri[3 * i] * mm[j] + ri[3 * i + 1] * mm[3 + j] + ri[3 * i + 2] * mm[6 + j];
  }
}

// out = p @ M + T with M[k][l] = s_k R[k][l]: the product pytorch3d's Scale(s).compose(Rotate(R), Translate(T)) applies.
// transform: R (9), T (3), s (3) per frame, transform_stride floats apart (0: one transform for every frame).
__global__ void icp_transform_points_kernel(const float* __restrict__ points, int64_t n, const float* __restrict__ transform,
                                            int64_t transform_stride, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t f = blockIdx.y;
  const float* tf = transform + f * transform_stride;
  const float3 p = load3(points, f * n + i);
  float* o = out + (f * n + i) * 3;
  for (int l = 0; l < 3; ++l) {
    const float m0 = __fmul_rn(tf[12], tf[l]), m1 = __fmul_rn(tf[13], tf[3 + l]), m2 = __fmul_rn(tf[14], tf[6 + l]);
    o[l] = __fadd_rn(__fmaf_rn(p.z, m2, __fmaf_rn(p.y, m1, __fmul_rn(p.x, m0))), tf[9 + l]);
  }
}

}  // namespace amb

using namespace amb;

extern "C" int amb_icp_scratch_doubles(int frames, int candidates, int n_pred, int n_gt, int64_t* out_doubles) {
  AMB_CHECK_ARG(out_doubles, "icp_scratch_doubles: null pointer");
  AMB_CHECK_ARG(frames >= 1 && candidates >= 1 && candidates <= ICP_MAX_C && n_pred >= 1 && n_gt >= 1,
                "icp_scratch_doubles: bad sizes (frames %d, candidates %d, n_pred %d, n_gt %d)", frames, candidates, n_pred,
                n_gt);
  *out_doubles = (int64_t)frames * candidates * icp_grid(candidates, n_pred, n_gt).slots() * ICP_NSUM;
  return AMB_OK;
}

extern "C" int amb_icp_chamfer_grad(const float* pred, const float* gt, int frames, int candidates, int n_pred, int n_gt,
                                    const float* rot, const float* params, double* scratch, double* sums,
                                    amb_stream_t stream) {
  AMB_CHECK_ARG(pred && gt && rot && params && scratch && sums, "icp_chamfer_grad: null pointer");
  AMB_CHECK_ARG(frames >= 1 && candidates >= 1 && candidates <= ICP_MAX_C && n_pred >= 1 && n_gt >= 1,
                "icp_chamfer_grad: bad sizes (frames %d, candidates %d, n_pred %d, n_gt %d)", frames, candidates, n_pred,
                n_gt);
  AMB_CHECK_ARG(n_pred <= (1 << 29) && n_gt <= (1 << 29), "icp_chamfer_grad: too many points");
  const IcpGrid grid = icp_grid(candidates, n_pred, n_gt);
  const int64_t blocks = (int64_t)frames * ((int64_t)grid.groups * grid.tiles_p + (int64_t)candidates * grid.tiles_q);
  AMB_CHECK_ARG(blocks < (1ll << 31), "icp_chamfer_grad: grid too large");
  cudaStream_t s = (cudaStream_t)stream;
  icp_nn_kernel<<<(unsigned)blocks, ICP_THREADS, 0, s>>>(pred, gt, candidates, n_pred, n_gt, rot, params, grid, scratch);
  AMB_CHECK_CUDA(cudaGetLastError());
  const int64_t n = (int64_t)frames * candidates * ICP_NSUM;
  icp_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(scratch, (int64_t)frames * candidates, n_pred, n_gt, grid,
                                                                  sums);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

extern "C" int amb_icp_adam_step(const double* sums, const float* rot_init, int frames, int candidates, float step_size,
                                 float bias2_sqrt, float* params, float* adam_m, float* adam_v, float* rot, float* best,
                                 amb_stream_t stream) {
  AMB_CHECK_ARG(sums && rot_init && params && adam_m && adam_v && rot && best, "icp_adam_step: null pointer");
  AMB_CHECK_ARG(frames >= 1 && candidates >= 1 && candidates <= ICP_MAX_C,
                "icp_adam_step: bad sizes (frames %d, candidates %d)", frames, candidates);
  const int threads = (candidates + 31) / 32 * 32;
  icp_adam_kernel<<<frames, threads, 0, (cudaStream_t)stream>>>(sums, rot_init, candidates, step_size, bias2_sqrt, params,
                                                                adam_m, adam_v, rot, best);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

extern "C" int amb_icp_transform_points(const float* points, int frames, int64_t n_points, const float* transform,
                                        int64_t transform_stride, float* out, amb_stream_t stream) {
  AMB_CHECK_ARG(frames >= 0 && n_points >= 0 && transform_stride >= 0, "icp_transform_points: bad sizes");
  if (frames == 0 || n_points == 0) return AMB_OK;
  AMB_CHECK_ARG(points && transform && out, "icp_transform_points: null pointer");
  AMB_CHECK_ARG(frames <= 65535 && n_points < (1ll << 40), "icp_transform_points: too many frames or points");
  icp_transform_points_kernel<<<dim3((unsigned)((n_points + 255) / 256), frames), 256, 0, (cudaStream_t)stream>>>(
      points, n_points, transform, transform_stride, out);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}
