// Skinning decomposition of a fixed-topology vertex animation: Smooth Skinning Decomposition with Rigid Bones (SSDR, Le &
// Deng 2012), fitted by alternating least squares.  actionmesh_b200/skinning.py drives the kernels; DESIGN.md §20 states the
// model and every rule below, and tests/skinning_ref.py restates them in numpy float64 with the same operation order.  Every
// fp64 product, sum, quotient and square root is an explicit round-to-nearest intrinsic (nvcc never contracts them into an
// FMA), every sum runs in a fixed order, and atomics are used only for a maximum: two runs give identical bits.
//
// Layout: rest (V, 3), vertices (T, V, 3), transforms (T, B, 12) = R row-major then t, with u = R p + t; joints (V, 4) int32
// and weights (V, 4) fp64, a slot being used when its weight is > 0.
//
//  seeds        farthest-point sampling of B rest vertices from vertex 0 (ties to the lowest index); labels = nearest seed.
//  rigid_error  e_ij = sum_t |R_j^t p_i + t_j^t - v_i^t|^2 for every bone; per vertex the arg-min and the 8 lowest (e, j).
//  bone_update  one bone j: per frame the weighted moments of the residual q_i = v_i - sum_{k != j} w_ik u_ik over the vertices j
//               influences (block partials over 256-vertex tiles, summed in tile order), then Horn's quaternion rotation.
//  weight_update per vertex: candidates = current support + lowest-error bones (<= 8); every subset of <= 4 candidates solves
//               its simplex-constrained least squares exactly (KKT system), the lowest-error non-negative solution wins.
//  error        sum_i |v^_i - v_i|^2 per frame (same tiles and order) and the maximum |v^_i - v_i|^2 (atomic max).
#include <cuda_runtime.h>
#include <cstdint>
#include "common.cuh"
#include "fp64.cuh"
#include "../../include/actionmesh_b200.h"

namespace amb {
namespace {

constexpr int SK_THREADS = FP64_THREADS;  // reduction kernels: one vertex per thread; a tile is 256 vertices
constexpr int SK_NMOM = 16;          // bone moments: sum w^2, sum w^2 p (3), sum w q (3), sum w p q^T (9)
constexpr int SK_MAX_BONES = 256;    // joints are written as glTF JOINTS_0 u8
constexpr int SK_CAND = 8;           // weight candidates per vertex
constexpr int SK_WU_THREADS = 64;    // weight update: per-thread Gram matrices live in shared memory
constexpr int SK_NGRAM = SK_CAND * (SK_CAND + 1) / 2;
constexpr double kDetMin = 1e-12;    // a subset's KKT matrix (Gram scaled to max diagonal 1) is singular unless |det| > this

// sum over the used slots k = 0..3 whose joint is not `skip` of w_k u_k, from 0, in slot order (skip = -1: every slot)
__device__ __forceinline__ V3 blend(const double* __restrict__ xf_t, const int32_t* __restrict__ joints,
                                    const double* __restrict__ weights, int64_t i, V3 p, int skip) {
  V3 s = {0.0, 0.0, 0.0};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double w = weights[4 * i + k];
    const int j = joints[4 * i + k];
    if (w > 0.0 && j != skip) {
      const V3 u = apply_xf(xf_t + 12 * (int64_t)j, p);
      s = {dadd(s.x, dmul(w, u.x)), dadd(s.y, dmul(w, u.y)), dadd(s.z, dmul(w, u.z))};
    }
  }
  return s;
}

// ---- seeds -------------------------------------------------------------------------------------------------------------------

// One block.  dist[i] = squared distance to the nearest seed so far, labels[i] = that seed (ties to the earlier seed); the next
// seed is the vertex of largest dist, ties to the lowest index.
__global__ void __launch_bounds__(1024) skin_seeds_kernel(const double* __restrict__ rest, int64_t V, int B,
                                                          double* __restrict__ dist, int32_t* __restrict__ seeds,
                                                          int32_t* __restrict__ labels, double* __restrict__ centres) {
  __shared__ double wd[32];
  __shared__ int64_t wi[32];
  __shared__ int64_t cur;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) cur = 0;
  __syncthreads();
  for (int b = 0; b < B; ++b) {
    const int64_t s = cur;
    const V3 ps = load3(rest, s);
    if (threadIdx.x == 0) {
      seeds[b] = (int32_t)s;
      centres[3 * b] = ps.x;
      centres[3 * b + 1] = ps.y;
      centres[3 * b + 2] = ps.z;
    }
    double bd = -1.0;
    int64_t bi = V;
    for (int64_t i = threadIdx.x; i < V; i += blockDim.x) {
      const double d = norm2(sub3(load3(rest, i), ps));
      double di = b ? dist[i] : d;
      if (b == 0 || d < di) {
        di = d;
        dist[i] = d;
        labels[i] = b;
      }
      if (di > bd) {
        bd = di;
        bi = i;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double od = __shfl_down_sync(0xffffffffu, bd, o);
      const int64_t oi = __shfl_down_sync(0xffffffffu, bi, o);
      if (od > bd || (od == bd && oi < bi)) {
        bd = od;
        bi = oi;
      }
    }
    if (lane == 0) {
      wd[warp] = bd;
      wi[warp] = bi;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
        if (wd[w] > bd || (wd[w] == bd && wi[w] < bi)) {
          bd = wd[w];
          bi = wi[w];
        }
      cur = bi;
    }
    __syncthreads();
  }
}

// ---- rigid error and candidates ----------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(128) skin_rigid_error_kernel(const double* __restrict__ rest, const double* __restrict__ verts,
                                                               int T, int64_t V, int B, const double* __restrict__ xf,
                                                               int32_t* __restrict__ argmin, double* __restrict__ min_error,
                                                               int32_t* __restrict__ cand) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V) return;
  const V3 p = load3(rest, i);
  double be[SK_CAND];
  int bj[SK_CAND];
#pragma unroll
  for (int k = 0; k < SK_CAND; ++k) {
    be[k] = 0.0;
    bj[k] = -1;
  }
  int filled = 0;
  for (int j = 0; j < B; ++j) {
    double e = 0.0;
    for (int t = 0; t < T; ++t)
      e = dadd(e, norm2(sub3(apply_xf(xf + ((int64_t)t * B + j) * 12, p), load3(verts, (int64_t)t * V + i))));
    // insert (e, j) into the ascending list; an equal error goes after the lower bone index already there
    double ce = e;
    int cj = j;
    bool moved = false;
#pragma unroll
    for (int k = 0; k < SK_CAND; ++k) {
      if (moved || k >= filled || ce < be[k]) {
        const double te = be[k];
        const int tj = bj[k];
        be[k] = ce;
        bj[k] = cj;
        ce = te;
        cj = tj;
        moved = true;
      }
    }
    filled = min(filled + 1, SK_CAND);
  }
  argmin[i] = bj[0];
  min_error[i] = be[0];
#pragma unroll
  for (int k = 0; k < SK_CAND; ++k) cand[SK_CAND * i + k] = bj[k];
}

// ---- bone update -------------------------------------------------------------------------------------------------------------

// grid (tiles, T): partials[(t * tiles + tile) * 16 + k] = the block sum of moment k over the tile's vertices (0 for the vertices
// bone j does not influence and past V).
__global__ void __launch_bounds__(SK_THREADS) skin_bone_partial_kernel(const double* __restrict__ rest,
                                                                       const double* __restrict__ verts, int64_t V, int B,
                                                                       const double* __restrict__ xf,
                                                                       const int32_t* __restrict__ joints,
                                                                       const double* __restrict__ weights, int bone,
                                                                       double* __restrict__ partials) {
  __shared__ double red[SK_THREADS / 32][SK_NMOM];
  const int t = blockIdx.y;
  const int64_t i = (int64_t)blockIdx.x * SK_THREADS + threadIdx.x;
  double c[SK_NMOM];
#pragma unroll
  for (int k = 0; k < SK_NMOM; ++k) c[k] = 0.0;
  if (i < V) {
    double a = 0.0;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (joints[4 * i + k] == bone && weights[4 * i + k] > 0.0) a = weights[4 * i + k];
    if (a > 0.0) {
      const V3 p = load3(rest, i);
      const V3 s = blend(xf + (int64_t)t * B * 12, joints, weights, i, p, bone);
      const V3 q = sub3(load3(verts, (int64_t)t * V + i), s);
      const double a2 = dmul(a, a);
      const double pv[3] = {p.x, p.y, p.z}, qv[3] = {q.x, q.y, q.z};
      c[0] = a2;
#pragma unroll
      for (int l = 0; l < 3; ++l) {
        c[1 + l] = dmul(a2, pv[l]);
        c[4 + l] = dmul(a, qv[l]);
      }
#pragma unroll
      for (int l = 0; l < 3; ++l) {
        const double wp = dmul(a, pv[l]);
#pragma unroll
        for (int m = 0; m < 3; ++m) c[7 + 3 * l + m] = dmul(wp, qv[m]);
      }
    }
  }
  block_sum<SK_NMOM>(c, red, partials + ((int64_t)t * gridDim.x + blockIdx.x) * SK_NMOM);
}

// One thread per frame: the moments summed over the tiles in tile order, then p* = sum w^2 p / sum w^2, q* = sum w q / sum w^2,
// H = sum w p q^T - p* (sum w q)^T, R by Horn's method and t = q* - R p*.  A bone with sum w^2 == 0 keeps its transform.
__global__ void skin_bone_solve_kernel(const double* __restrict__ partials, int T, int tiles, int B, int bone,
                                       double* __restrict__ xf, double* __restrict__ centres) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  double m[SK_NMOM];
#pragma unroll
  for (int k = 0; k < SK_NMOM; ++k) m[k] = 0.0;
  const double* pt = partials + (int64_t)t * tiles * SK_NMOM;
  for (int s = 0; s < tiles; ++s)
#pragma unroll
    for (int k = 0; k < SK_NMOM; ++k) m[k] = dadd(m[k], pt[(int64_t)s * SK_NMOM + k]);
  if (!(m[0] > 0.0)) return;
  double ps[3], qs[3], H[3][3], R[9];
#pragma unroll
  for (int l = 0; l < 3; ++l) {
    ps[l] = ddiv(m[1 + l], m[0]);
    qs[l] = ddiv(m[4 + l], m[0]);
  }
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) H[a][b] = dsub(m[7 + 3 * a + b], dmul(ps[a], m[4 + b]));
  horn_rotation(H, R);
  double* o = xf + ((int64_t)t * B + bone) * 12;
#pragma unroll
  for (int k = 0; k < 9; ++k) o[k] = R[k];
#pragma unroll
  for (int a = 0; a < 3; ++a)
    o[9 + a] = dsub(qs[a], dadd(dadd(dmul(R[3 * a], ps[0]), dmul(R[3 * a + 1], ps[1])), dmul(R[3 * a + 2], ps[2])));
  if (t == 0)
#pragma unroll
    for (int a = 0; a < 3; ++a) centres[3 * bone + a] = ps[a];
}

// ---- weight update -----------------------------------------------------------------------------------------------------------

// packed upper triangle of the 8x8 Gram matrix, a <= b
__device__ __forceinline__ int gram_index(int a, int b) { return a * SK_CAND - a * (a - 1) / 2 + (b - a); }

struct Best {
  double e;
  int n;
  int c[4];
  double w[4];
};

// Subset idx[0] < ... < idx[S-1] of the candidate positions: minimise w^T G_S w subject to sum w = 1 through the KKT system
// [[G_S / s, 1], [1^T, 0]] [w; mu] = [0; 1] with s = max diag G_S, by Gaussian elimination with partial pivoting (largest
// |pivot|, ties to the upper row).  Skipped when s == 0, when |det| (the product of the pivots' magnitudes) <= kDetMin, or when
// a weight is negative; kept when its error w^T G_S w is below the best so far.
template <int S>
__device__ __forceinline__ void try_subset(const double* __restrict__ g_base, const int (&idx)[S], Best& best) {
  constexpr int M = S + 1;
  double g[S][S];
#pragma unroll
  for (int a = 0; a < S; ++a)
#pragma unroll
    for (int b = a; b < S; ++b) {
      g[a][b] = g_base[gram_index(idx[a], idx[b]) * SK_WU_THREADS];
      g[b][a] = g[a][b];
    }
  double s = g[0][0];
#pragma unroll
  for (int a = 1; a < S; ++a) s = fmax(s, g[a][a]);
  if (!(s > 0.0)) return;
  double A[M][M], x[M];
#pragma unroll
  for (int a = 0; a < S; ++a) {
#pragma unroll
    for (int b = 0; b < S; ++b) A[a][b] = ddiv(g[a][b], s);
    A[a][S] = 1.0;
    A[S][a] = 1.0;
    x[a] = 0.0;
  }
  A[S][S] = 0.0;
  x[S] = 1.0;
  double det = 1.0;
#pragma unroll
  for (int k = 0; k < M; ++k) {
    int piv = k;
    double pv = fabs(A[k][k]);
#pragma unroll
    for (int r = k + 1; r < M; ++r)
      if (fabs(A[r][k]) > pv) {
        piv = r;
        pv = fabs(A[r][k]);
      }
    if (!(pv > 0.0)) return;
#pragma unroll
    for (int r = k + 1; r < M; ++r)
      if (r == piv) {
#pragma unroll
        for (int c = 0; c < M; ++c) {
          const double tmp = A[k][c];
          A[k][c] = A[r][c];
          A[r][c] = tmp;
        }
        const double tmp = x[k];
        x[k] = x[r];
        x[r] = tmp;
      }
    det = dmul(det, pv);
#pragma unroll
    for (int r = k + 1; r < M; ++r) {
      const double f = ddiv(A[r][k], A[k][k]);
#pragma unroll
      for (int c = k + 1; c < M; ++c) A[r][c] = dsub(A[r][c], dmul(f, A[k][c]));
      x[r] = dsub(x[r], dmul(f, x[k]));
    }
  }
  if (!(det > kDetMin)) return;
#pragma unroll
  for (int k = M - 1; k >= 0; --k) {
    double acc = x[k];
#pragma unroll
    for (int c = k + 1; c < M; ++c) acc = dsub(acc, dmul(A[k][c], x[c]));
    x[k] = ddiv(acc, A[k][k]);
  }
#pragma unroll
  for (int a = 0; a < S; ++a)
    if (!(x[a] >= 0.0)) return;
  double e = 0.0;
#pragma unroll
  for (int a = 0; a < S; ++a) {
    double gw = 0.0;
#pragma unroll
    for (int b = 0; b < S; ++b) gw = dadd(gw, dmul(g[a][b], x[b]));
    e = dadd(e, dmul(x[a], gw));
  }
  if (e < best.e) {
    best.e = e;
    best.n = S;
#pragma unroll
    for (int a = 0; a < S; ++a) {
      best.c[a] = idx[a];
      best.w[a] = x[a];
    }
  }
}

// One thread per vertex.  Candidates: the used slots in slot order, then the rigid-error list in rank order, skipping repeats,
// up to 8.  G_ab = sum_t r_a . r_b with r_a = u_a - v (the error of weights w with sum w = 1 is w^T G w).  Subsets are tried by
// size 1, 2, 3, 4 and lexicographically within a size; singletons (w = 1, error G_aa) are always feasible.
__global__ void __launch_bounds__(SK_WU_THREADS) skin_weight_update_kernel(const double* __restrict__ rest,
                                                                           const double* __restrict__ verts, int T, int64_t V,
                                                                           int B, const double* __restrict__ xf,
                                                                           const int32_t* __restrict__ cand,
                                                                           int32_t* __restrict__ joints,
                                                                           double* __restrict__ weights) {
  __shared__ double sg[SK_NGRAM * SK_WU_THREADS];
  __shared__ int sc[SK_CAND * SK_WU_THREADS];
  const int64_t i = (int64_t)blockIdx.x * SK_WU_THREADS + threadIdx.x;
  if (i >= V) return;
  double* g = sg + threadIdx.x;
  int* c = sc + threadIdx.x;
  int n = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (weights[4 * i + k] > 0.0) c[SK_WU_THREADS * n++] = joints[4 * i + k];
  for (int k = 0; k < SK_CAND && n < SK_CAND; ++k) {
    const int j = cand[SK_CAND * i + k];
    if (j < 0) break;
    bool dup = false;
    for (int m = 0; m < n; ++m) dup |= c[SK_WU_THREADS * m] == j;
    if (!dup) c[SK_WU_THREADS * n++] = j;
  }
  int cj[SK_CAND];
#pragma unroll
  for (int a = 0; a < SK_CAND; ++a) cj[a] = a < n ? c[SK_WU_THREADS * a] : 0;
  const V3 p = load3(rest, i);
#pragma unroll
  for (int k = 0; k < SK_NGRAM; ++k) g[k * SK_WU_THREADS] = 0.0;
  for (int t = 0; t < T; ++t) {
    const V3 v = load3(verts, (int64_t)t * V + i);
    const double* xf_t = xf + (int64_t)t * B * 12;
    V3 r[SK_CAND];
#pragma unroll
    for (int a = 0; a < SK_CAND; ++a)
      if (a < n) r[a] = sub3(apply_xf(xf_t + 12 * (int64_t)cj[a], p), v);
#pragma unroll
    for (int a = 0; a < SK_CAND; ++a)
#pragma unroll
      for (int b = a; b < SK_CAND; ++b)
        if (b < n) {
          double* gk = g + gram_index(a, b) * SK_WU_THREADS;
          *gk = dadd(*gk, dot3(r[a], r[b]));
        }
  }

  Best best;
  best.e = g[0];
  best.n = 1;
  best.c[0] = 0;
  best.w[0] = 1.0;
  for (int a = 1; a < n; ++a) {
    const double e = g[gram_index(a, a) * SK_WU_THREADS];
    if (e < best.e) {
      best.e = e;
      best.c[0] = a;
    }
  }
  for (int a = 0; a < n; ++a)
    for (int b = a + 1; b < n; ++b) {
      const int idx[2] = {a, b};
      try_subset<2>(g, idx, best);
    }
  for (int a = 0; a < n; ++a)
    for (int b = a + 1; b < n; ++b)
      for (int d = b + 1; d < n; ++d) {
        const int idx[3] = {a, b, d};
        try_subset<3>(g, idx, best);
      }
  for (int a = 0; a < n; ++a)
    for (int b = a + 1; b < n; ++b)
      for (int d = b + 1; d < n; ++d)
        for (int e = d + 1; e < n; ++e) {
          const int idx[4] = {a, b, d, e};
          try_subset<4>(g, idx, best);
        }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const bool used = k < best.n && best.w[k] > 0.0;
    joints[4 * i + k] = used ? c[SK_WU_THREADS * best.c[k]] : 0;
    weights[4 * i + k] = used ? best.w[k] : 0.0;
  }
}

// ---- reconstruction error ----------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(SK_THREADS) skin_error_partial_kernel(const double* __restrict__ rest,
                                                                        const double* __restrict__ verts, int64_t V, int B,
                                                                        const double* __restrict__ xf,
                                                                        const int32_t* __restrict__ joints,
                                                                        const double* __restrict__ weights,
                                                                        double* __restrict__ partials,
                                                                        unsigned long long* __restrict__ max_bits) {
  __shared__ double red[SK_THREADS / 32][1];
  const int t = blockIdx.y;
  const int64_t i = (int64_t)blockIdx.x * SK_THREADS + threadIdx.x;
  double d2 = 0.0;
  if (i < V) {
    const V3 p = load3(rest, i);
    d2 = norm2(sub3(blend(xf + (int64_t)t * B * 12, joints, weights, i, p, -1), load3(verts, (int64_t)t * V + i)));
  }
  error_tile(d2, red, partials + (int64_t)t * gridDim.x + blockIdx.x, max_bits);
}

}  // namespace
}  // namespace amb

using namespace amb;

#define SK_CHECK_SIZES(fn, frames, V, B)                                                                                   \
  AMB_CHECK_ARG((frames) >= 1 && (frames) <= 65535 && (V) >= 1 && (V) < (1ll << 31) - SK_THREADS && (B) >= 1 &&          \
                    (B) <= SK_MAX_BONES && (B) <= (V),                                                                     \
                fn ": bad sizes (frames %d, vertices %lld, bones %d)", (int)(frames), (long long)(V), (int)(B))

extern "C" int amb_skin_scratch_doubles(int frames, int64_t n_vertices, int64_t* out_doubles) {
  AMB_CHECK_ARG(out_doubles, "skin_scratch_doubles: null pointer");
  SK_CHECK_SIZES("skin_scratch_doubles", frames, n_vertices, 1);
  *out_doubles = (int64_t)frames * tiles_of(n_vertices) * SK_NMOM;
  return AMB_OK;
}

extern "C" int amb_skin_seeds(const double* rest, int64_t n_vertices, int n_bones, double* dist, int32_t* seeds,
                              int32_t* labels, double* centres, amb_stream_t stream) {
  AMB_CHECK_ARG(rest && dist && seeds && labels && centres, "skin_seeds: null pointer");
  SK_CHECK_SIZES("skin_seeds", 1, n_vertices, n_bones);
  skin_seeds_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(rest, n_vertices, n_bones, dist, seeds, labels, centres);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

extern "C" int amb_skin_rigid_error(const double* rest, const double* vertices, int frames, int64_t n_vertices,
                                    const double* transforms, int n_bones, int32_t* argmin, double* min_error,
                                    int32_t* candidates, amb_stream_t stream) {
  AMB_CHECK_ARG(rest && vertices && transforms && argmin && min_error && candidates, "skin_rigid_error: null pointer");
  SK_CHECK_SIZES("skin_rigid_error", frames, n_vertices, n_bones);
  skin_rigid_error_kernel<<<(unsigned)((n_vertices + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      rest, vertices, frames, n_vertices, n_bones, transforms, argmin, min_error, candidates);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

extern "C" int amb_skin_bone_update(const double* rest, const double* vertices, int frames, int64_t n_vertices,
                                    double* transforms, int n_bones, const int32_t* joints, const double* weights, int bone,
                                    double* scratch, double* centres, amb_stream_t stream) {
  AMB_CHECK_ARG(rest && vertices && transforms && joints && weights && scratch && centres, "skin_bone_update: null pointer");
  SK_CHECK_SIZES("skin_bone_update", frames, n_vertices, n_bones);
  AMB_CHECK_ARG(bone >= 0 && bone < n_bones, "skin_bone_update: bone %d outside [0, %d)", bone, n_bones);
  cudaStream_t s = (cudaStream_t)stream;
  const int tiles = tiles_of(n_vertices);
  skin_bone_partial_kernel<<<dim3(tiles, frames), SK_THREADS, 0, s>>>(rest, vertices, n_vertices, n_bones, transforms,
                                                                        joints, weights, bone, scratch);
  AMB_CHECK_CUDA(cudaGetLastError());
  skin_bone_solve_kernel<<<(frames + 63) / 64, 64, 0, s>>>(scratch, frames, tiles, n_bones, bone, transforms, centres);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

extern "C" int amb_skin_weight_update(const double* rest, const double* vertices, int frames, int64_t n_vertices,
                                      const double* transforms, int n_bones, const int32_t* candidates, int32_t* joints,
                                      double* weights, amb_stream_t stream) {
  AMB_CHECK_ARG(rest && vertices && transforms && candidates && joints && weights, "skin_weight_update: null pointer");
  SK_CHECK_SIZES("skin_weight_update", frames, n_vertices, n_bones);
  skin_weight_update_kernel<<<(unsigned)((n_vertices + SK_WU_THREADS - 1) / SK_WU_THREADS), SK_WU_THREADS, 0,
                              (cudaStream_t)stream>>>(rest, vertices, frames, n_vertices, n_bones, transforms, candidates,
                                                      joints, weights);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

extern "C" int amb_skin_error(const double* rest, const double* vertices, int frames, int64_t n_vertices,
                              const double* transforms, int n_bones, const int32_t* joints, const double* weights,
                              double* scratch, double* frame_errors, double* max_error2, amb_stream_t stream) {
  AMB_CHECK_ARG(rest && vertices && transforms && joints && weights && scratch && frame_errors && max_error2,
                "skin_error: null pointer");
  SK_CHECK_SIZES("skin_error", frames, n_vertices, n_bones);
  cudaStream_t s = (cudaStream_t)stream;
  const int tiles = tiles_of(n_vertices);
  AMB_CHECK_CUDA(cudaMemsetAsync(max_error2, 0, sizeof(double), s));
  skin_error_partial_kernel<<<dim3(tiles, frames), SK_THREADS, 0, s>>>(rest, vertices, n_vertices, n_bones, transforms,
                                                                         joints, weights, scratch,
                                                                         reinterpret_cast<unsigned long long*>(max_error2));
  AMB_CHECK_CUDA(cudaGetLastError());
  error_sum_kernel<<<1, 256, 0, s>>>(scratch, frames, tiles, frame_errors);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}
