// A joint hierarchy found from SSDR bones (Le & Deng 2014), and the device side of refitting it (DESIGN.md §22).
// actionmesh_b200/autorig.py drives the kernels and tests/autorig_ref.py restates them in numpy float64 with the same
// operation order.  Every fp64 product, sum, quotient and square root is an explicit round-to-nearest intrinsic (fp64.cuh),
// every sum runs in a fixed order and no floating-point value is accumulated atomically: two runs give identical bits.
//
// Bones i < j of B form pair p(i, j) = i (2B - i - 1) / 2 + (j - i - 1), the pairs in lexicographic order.
//   pair_stats    dominant bone of every vertex (its used slot of largest weight, ties to the earlier slot); every face edge
//                 e = 3f + k, k-th edge (f_k, f_(k+1) mod 3), whose ends have different dominant bones is compacted in edge
//                 order with its pair key (scan.cuh), sorted stably by key (two 8-bit counting passes over 256-item tiles),
//                 and each pair sums its edges' rest midpoints in edge order: count n_p and prior m_p = sum / n_p.
//   bone_weights  per 256-vertex tile, bone b's sum of its used-slot weights (vertex order, then slot order), then the tiles'
//                 sums in tile order.
//   joint_solve   one thread per pair: c = (sum_t D^T D + lambda T I)^-1 (sum_t D^T d + lambda T m_bar) by Cholesky, with
//                 D = R_i - R_j and d = t_j - t_i; cost = (sum_t |D c - d|^2) / T.
//   slots         (V, 4) joints / weights -> the rig's (V, 8) slots, used slots first in slot order, then bind 0 weight 0.
//   joint_lists   joint k's list = the vertices whose used slots hold a bind of a joint in [k, end_k), ascending; the lists
//                 concatenated in joint order, by a count -> scan -> emit pass over the J V items (k, i).
#include <cuda_runtime.h>
#include <cstdint>
#include "common.cuh"
#include "fp64.cuh"
#include "scan.cuh"
#include "../../include/actionmesh_b200.h"

namespace amb {
namespace {

constexpr int AR_MAX_BONES = 256;
constexpr int AR_SORT_TILE = 256;     // items per counting-sort tile (one thread each)
constexpr int AR_DIGITS = 256;        // 8-bit digits
constexpr int AR_SOLVE_THREADS = 128;

__host__ __device__ __forceinline__ int pair_index(int i, int j, int B) { return i * (2 * B - i - 1) / 2 + (j - i - 1); }
__host__ __device__ __forceinline__ int64_t pair_count_of(int B) { return (int64_t)B * (B - 1) / 2; }

// The dominant bone of every vertex, -1 when no slot is used.
__global__ void dominant_kernel(const int32_t* __restrict__ joints, const double* __restrict__ weights, int64_t V,
                                int32_t* __restrict__ dom) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  int best = -1;
  double bw = 0.0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double w = weights[4 * v + k];
    if (w > 0.0 && (best < 0 || w > bw)) {
      best = joints[4 * v + k];
      bw = w;
    }
  }
  dom[v] = best;
}

__device__ __forceinline__ void edge_ends(const int32_t* __restrict__ faces, long long e, int& a, int& b) {
  const long long f = e / 3;
  const int k = (int)(e - 3 * f);
  a = faces[3 * f + k];
  b = faces[3 * f + (k == 2 ? 0 : k + 1)];
}

// scan.cuh functor: every edge whose ends have different dominant bones, with its pair key, in edge order.
struct CrossEdges {
  const int32_t* faces;
  const int32_t* dom;
  int B;
  int32_t* keys;
  int32_t* edges;
  __device__ int key(long long e) const {
    int a, b;
    edge_ends(faces, e, a, b);
    const int da = dom[a], db = dom[b];
    if (da < 0 || db < 0 || da == db) return -1;
    return da < db ? pair_index(da, db, B) : pair_index(db, da, B);
  }
  __device__ int count(long long e) const { return key(e) >= 0 ? 1 : 0; }
  __device__ void emit(long long e, int off) const {
    const int k = key(e);
    if (k >= 0) {
      keys[off] = k;
      edges[off] = (int)e;
    }
  }
};

// scan.cuh functor: the exclusive prefix sum of an int array.
struct PrefixOf {
  const int32_t* in;
  int32_t* out;
  __device__ int count(long long i) const { return in[i]; }
  __device__ void emit(long long i, int off) const { out[i] = off; }
};

// hist[d * tiles + tile] = the number of the tile's items (of the first *n) whose digit (key >> shift) & 255 is d.
__global__ void __launch_bounds__(AR_SORT_TILE) sort_histogram_kernel(const int32_t* __restrict__ keys,
                                                                     const int32_t* __restrict__ n, int shift,
                                                                     int32_t* __restrict__ hist) {
  __shared__ int digit[AR_SORT_TILE];
  const int64_t idx = (int64_t)blockIdx.x * AR_SORT_TILE + threadIdx.x;
  digit[threadIdx.x] = idx < *n ? (keys[idx] >> shift) & (AR_DIGITS - 1) : -1;
  __syncthreads();
  int c = 0;
  for (int k = 0; k < AR_SORT_TILE; ++k) c += digit[k] == (int)threadIdx.x;
  hist[(int64_t)threadIdx.x * gridDim.x + blockIdx.x] = c;
}

// Stable scatter: an item goes to offs[d * tiles + tile] + the number of earlier items of its tile with the same digit.
__global__ void __launch_bounds__(AR_SORT_TILE) sort_scatter_kernel(const int32_t* __restrict__ keys,
                                                                   const int32_t* __restrict__ edges,
                                                                   const int32_t* __restrict__ n, int shift,
                                                                   const int32_t* __restrict__ offs,
                                                                   int32_t* __restrict__ out_keys,
                                                                   int32_t* __restrict__ out_edges) {
  __shared__ int digit[AR_SORT_TILE];
  const int64_t idx = (int64_t)blockIdx.x * AR_SORT_TILE + threadIdx.x;
  const bool live = idx < *n;
  const int d = live ? (keys[idx] >> shift) & (AR_DIGITS - 1) : -1;
  digit[threadIdx.x] = d;
  __syncthreads();
  if (!live) return;
  int rank = 0;
  for (int k = 0; k < (int)threadIdx.x; ++k) rank += digit[k] == d;
  const int pos = offs[(int64_t)d * gridDim.x + blockIdx.x] + rank;
  out_keys[pos] = keys[idx];
  out_edges[pos] = edges[idx];
}

// start[key] = the first sorted position holding key (start was filled with -1).
__global__ void segment_start_kernel(const int32_t* __restrict__ keys, const int32_t* __restrict__ n,
                                     int32_t* __restrict__ start) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= *n) return;
  if (idx == 0 || keys[idx - 1] != keys[idx]) start[keys[idx]] = (int)idx;
}

// One thread per pair: n_p and the mean of its edges' rest midpoints ((p_a + p_b) * 0.5 per component), summed in edge
// order from 0 and divided by n_p; 0 and (0, 0, 0) for a pair without an edge.
__global__ void pair_sum_kernel(const double* __restrict__ rest, const int32_t* __restrict__ faces,
                                const int32_t* __restrict__ keys, const int32_t* __restrict__ edges,
                                const int32_t* __restrict__ n, const int32_t* __restrict__ start, int64_t P,
                                int32_t* __restrict__ pair_count, double* __restrict__ pair_prior) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int total = *n;
  int cnt = 0;
  V3 s = {0.0, 0.0, 0.0};
  for (int idx = start[p]; idx >= 0 && idx < total && keys[idx] == (int)p; ++idx) {
    int a, b;
    edge_ends(faces, edges[idx], a, b);
    const V3 pa = load3(rest, a), pb = load3(rest, b);
    s = {dadd(s.x, dmul(dadd(pa.x, pb.x), 0.5)), dadd(s.y, dmul(dadd(pa.y, pb.y), 0.5)),
         dadd(s.z, dmul(dadd(pa.z, pb.z), 0.5))};
    ++cnt;
  }
  pair_count[p] = cnt;
  const double c = (double)cnt;
  pair_prior[3 * p] = cnt ? ddiv(s.x, c) : 0.0;
  pair_prior[3 * p + 1] = cnt ? ddiv(s.y, c) : 0.0;
  pair_prior[3 * p + 2] = cnt ? ddiv(s.z, c) : 0.0;
}

// partials[tile * B + b] = bone b's used-slot weights over the tile's vertices, vertex order then slot order, from 0.
__global__ void __launch_bounds__(FP64_THREADS) bone_weight_partial_kernel(const int32_t* __restrict__ joints,
                                                                          const double* __restrict__ weights, int64_t V,
                                                                          int B, double* __restrict__ partials) {
  __shared__ int sj[FP64_THREADS * 4];
  __shared__ double sw[FP64_THREADS * 4];
  const int64_t v0 = (int64_t)blockIdx.x * FP64_THREADS;
  const int nv = (int)(V - v0 < FP64_THREADS ? V - v0 : FP64_THREADS);
  for (int k = threadIdx.x; k < 4 * nv; k += FP64_THREADS) {
    sj[k] = joints[4 * v0 + k];
    sw[k] = weights[4 * v0 + k];
  }
  __syncthreads();
  if ((int)threadIdx.x >= B) return;
  double s = 0.0;
  for (int k = 0; k < 4 * nv; ++k)
    if (sw[k] > 0.0 && sj[k] == (int)threadIdx.x) s = dadd(s, sw[k]);
  partials[(int64_t)blockIdx.x * B + threadIdx.x] = s;
}

__global__ void bone_weight_sum_kernel(const double* __restrict__ partials, int tiles, int B, double* __restrict__ out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double s = 0.0;
  for (int t = 0; t < tiles; ++t) s = dadd(s, partials[(int64_t)t * B + b]);
  out[b] = s;
}

// One thread per pair (i, j): the normal equations summed in frame order, per frame (D^T D)_ab = (D_0a D_0b + D_1a D_1b)
// + D_2a D_2b and (D^T d)_a = (D_0a d_0 + D_1a d_1) + D_2a d_2; A = N + lambda T on the diagonal, b = r + (lambda T) m_bar;
// Cholesky A = L L^T, then L y = b and L^T c = y (each row's products subtracted in ascending column order).
__global__ void __launch_bounds__(AR_SOLVE_THREADS) joint_solve_kernel(const double* __restrict__ xf, int T, int B,
                                                                      const double* __restrict__ centres,
                                                                      const int32_t* __restrict__ pair_count,
                                                                      const double* __restrict__ pair_prior,
                                                                      const double* __restrict__ lambda,
                                                                      double* __restrict__ pair_joint,
                                                                      double* __restrict__ pair_cost) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (int)pair_count_of(B)) return;
  int i = 0, rem = p;
  while (rem >= B - 1 - i) {
    rem -= B - 1 - i;
    ++i;
  }
  const int j = i + 1 + rem;
  double N[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};   // 00 01 02 11 12 22
  double r[3] = {0.0, 0.0, 0.0};
  for (int t = 0; t < T; ++t) {
    const double* Xi = xf + ((int64_t)t * B + i) * 12;
    const double* Xj = xf + ((int64_t)t * B + j) * 12;
    double D[9], d[3];
#pragma unroll
    for (int k = 0; k < 9; ++k) D[k] = dsub(Xi[k], Xj[k]);
#pragma unroll
    for (int k = 0; k < 3; ++k) d[k] = dsub(Xj[9 + k], Xi[9 + k]);
    int q = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = a; b < 3; ++b, ++q)
        N[q] = dadd(N[q], dadd(dadd(dmul(D[a], D[b]), dmul(D[3 + a], D[3 + b])), dmul(D[6 + a], D[6 + b])));
#pragma unroll
    for (int a = 0; a < 3; ++a) r[a] = dadd(r[a], dadd(dadd(dmul(D[a], d[0]), dmul(D[3 + a], d[1])), dmul(D[6 + a], d[2])));
  }
  double m[3];
  if (pair_count[p] > 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) m[a] = pair_prior[3 * p + a];
  } else {
#pragma unroll
    for (int a = 0; a < 3; ++a) m[a] = dmul(dadd(centres[3 * i + a], centres[3 * j + a]), 0.5);
  }
  const double lt = dmul(*lambda, (double)T);
  const double a00 = dadd(N[0], lt), a11 = dadd(N[3], lt), a22 = dadd(N[5], lt);
  const double b0 = dadd(r[0], dmul(lt, m[0])), b1 = dadd(r[1], dmul(lt, m[1])), b2 = dadd(r[2], dmul(lt, m[2]));
  const double l00 = __dsqrt_rn(a00);
  const double l10 = ddiv(N[1], l00), l20 = ddiv(N[2], l00);
  const double l11 = __dsqrt_rn(dsub(a11, dmul(l10, l10)));
  const double l21 = ddiv(dsub(N[4], dmul(l20, l10)), l11);
  const double l22 = __dsqrt_rn(dsub(dsub(a22, dmul(l20, l20)), dmul(l21, l21)));
  const double y0 = ddiv(b0, l00);
  const double y1 = ddiv(dsub(b1, dmul(l10, y0)), l11);
  const double y2 = ddiv(dsub(dsub(b2, dmul(l20, y0)), dmul(l21, y1)), l22);
  const double c2 = ddiv(y2, l22);
  const double c1 = ddiv(dsub(y1, dmul(l21, c2)), l11);
  const double c0 = ddiv(dsub(dsub(y0, dmul(l10, c1)), dmul(l20, c2)), l00);
  double e = 0.0;
  for (int t = 0; t < T; ++t) {
    const double* Xi = xf + ((int64_t)t * B + i) * 12;
    const double* Xj = xf + ((int64_t)t * B + j) * 12;
    double res[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double Da0 = dsub(Xi[3 * a], Xj[3 * a]), Da1 = dsub(Xi[3 * a + 1], Xj[3 * a + 1]),
                   Da2 = dsub(Xi[3 * a + 2], Xj[3 * a + 2]);
      res[a] = dsub(dadd(dadd(dmul(Da0, c0), dmul(Da1, c1)), dmul(Da2, c2)), dsub(Xj[9 + a], Xi[9 + a]));
    }
    e = dadd(e, dadd(dadd(dmul(res[0], res[0]), dmul(res[1], res[1])), dmul(res[2], res[2])));
  }
  pair_joint[3 * p] = c0;
  pair_joint[3 * p + 1] = c1;
  pair_joint[3 * p + 2] = c2;
  pair_cost[p] = ddiv(e, (double)T);
}

__global__ void slots_kernel(const int32_t* __restrict__ joints, const double* __restrict__ weights, int64_t V,
                             int32_t* __restrict__ slot_bind, double* __restrict__ slot_weight) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  int s = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double w = weights[4 * v + k];
    if (w > 0.0) {
      slot_bind[8 * v + s] = joints[4 * v + k];
      slot_weight[8 * v + s] = w;
      ++s;
    }
  }
  for (; s < 8; ++s) {
    slot_bind[8 * v + s] = 0;
    slot_weight[8 * v + s] = 0.0;
  }
}

// scan.cuh functor over the J V items q = k V + i: item q is in joint k's list when a used slot of vertex i holds a bind
// of a joint in [k, end_k).  emit also writes offsets[k] at i = 0 and offsets[J] at the last item.
struct JointLists {
  const int32_t* bind_joint;
  const int32_t* slot_bind;
  const double* slot_weight;
  const int32_t* end;
  long long V;
  int J;
  int32_t* lists;
  long long capacity;
  int32_t* offsets;
  __device__ int count(long long q) const {
    const int k = (int)(q / V);
    const long long i = q - (long long)k * V;
    const int e = end[k];
    for (int s = 0; s < 8; ++s) {
      if (!(slot_weight[8 * i + s] > 0.0)) continue;
      const int jb = bind_joint[slot_bind[8 * i + s]];
      if (jb >= k && jb < e) return 1;
    }
    return 0;
  }
  __device__ void emit(long long q, int off) const {
    const int k = (int)(q / V);
    const long long i = q - (long long)k * V;
    const int c = count(q);
    if (i == 0) offsets[k] = off;
    if (c && off < capacity) lists[off] = (int)i;
    if (q == (long long)J * V - 1) offsets[J] = off + c;
  }
};

struct PairScratch {
  int32_t *dom, *keys0, *edges0, *keys1, *edges1, *hist, *offs, *edge_scan, *hist_scan, *start;
};

static int64_t pair_scratch_layout(int64_t V, int64_t F, int B, PairScratch* s, int32_t* base) {
  const int64_t E = 3 * F;
  const int64_t tiles = (E + AR_SORT_TILE - 1) / AR_SORT_TILE;
  const int64_t sizes[10] = {V, E, E, E, E, AR_DIGITS * tiles, AR_DIGITS * tiles, scan_tiles(E) + 1,
                             scan_tiles(AR_DIGITS * tiles) + 1, pair_count_of(B)};
  int32_t** ptrs[10] = {&s->dom, &s->keys0, &s->edges0, &s->keys1, &s->edges1, &s->hist, &s->offs, &s->edge_scan,
                        &s->hist_scan, &s->start};
  int64_t off = 0;
  for (int k = 0; k < 10; ++k) {
    *ptrs[k] = base + off;
    off += (sizes[k] + 3) & ~int64_t(3);   // 16-byte aligned pieces
  }
  return off;
}

}  // namespace
}  // namespace amb

using namespace amb;

#define AR_CHECK_BONES(fn, V, B)                                                                                      \
  AMB_CHECK_ARG((V) >= 1 && (V) < (1ll << 31) - FP64_THREADS && (B) >= 1 && (B) <= AR_MAX_BONES && (B) <= (V),          \
                fn ": bad sizes (vertices %lld, bones %d)", (long long)(V), (int)(B))

extern "C" int amb_autorig_pair_scratch_ints(int64_t n_vertices, int64_t n_faces, int n_bones, int64_t* out_ints) {
  AMB_CHECK_ARG(out_ints, "autorig_pair_scratch_ints: null pointer");
  AR_CHECK_BONES("autorig_pair_scratch_ints", n_vertices, n_bones);
  AMB_CHECK_ARG(n_faces >= 1 && n_faces <= ((1ll << 31) - 1) / 3 - AR_SORT_TILE, "autorig_pair_scratch_ints: bad face count %lld",
                (long long)n_faces);
  PairScratch s;
  *out_ints = pair_scratch_layout(n_vertices, n_faces, n_bones, &s, nullptr);
  return AMB_OK;
}

extern "C" int amb_autorig_pair_stats(const double* rest, int64_t n_vertices, const int32_t* faces, int64_t n_faces,
                                      const int32_t* joints, const double* weights, int n_bones, int32_t* scratch,
                                      int32_t* pair_count, double* pair_prior, amb_stream_t stream) {
  AR_CHECK_BONES("autorig_pair_stats", n_vertices, n_bones);
  AMB_CHECK_ARG(n_faces >= 1 && n_faces <= ((1ll << 31) - 1) / 3 - AR_SORT_TILE, "autorig_pair_stats: bad face count %lld",
                (long long)n_faces);
  const int64_t P = pair_count_of(n_bones);
  if (P == 0) return AMB_OK;  // one bone: no pair, and the (empty) outputs may be null
  AMB_CHECK_ARG(rest && faces && joints && weights && scratch && pair_count && pair_prior, "autorig_pair_stats: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  PairScratch s;
  pair_scratch_layout(n_vertices, n_faces, n_bones, &s, scratch);
  const int64_t E = 3 * n_faces;
  const int tiles = (int)((E + AR_SORT_TILE - 1) / AR_SORT_TILE);
  dominant_kernel<<<(unsigned)((n_vertices + 255) / 256), 256, 0, st>>>(joints, weights, n_vertices, s.dom);
  AMB_CHECK_CUDA(cudaGetLastError());
  const CrossEdges ce{faces, s.dom, n_bones, s.keys0, s.edges0};
  if (int rc = scan_count(E, ce, s.edge_scan, st)) return rc;
  if (int rc = scan_emit(E, ce, s.edge_scan, st)) return rc;
  const int32_t* n = s.edge_scan + scan_tiles(E);   // the number of crossing edges (device)
  int32_t *kin = s.keys0, *ein = s.edges0, *kout = s.keys1, *eout = s.edges1;
  for (int shift = 0; shift < 16; shift += 8) {
    sort_histogram_kernel<<<tiles, AR_SORT_TILE, 0, st>>>(kin, n, shift, s.hist);
    AMB_CHECK_CUDA(cudaGetLastError());
    const PrefixOf pf{s.hist, s.offs};
    if (int rc = scan_count((long long)AR_DIGITS * tiles, pf, s.hist_scan, st)) return rc;
    if (int rc = scan_emit((long long)AR_DIGITS * tiles, pf, s.hist_scan, st)) return rc;
    sort_scatter_kernel<<<tiles, AR_SORT_TILE, 0, st>>>(kin, ein, n, shift, s.offs, kout, eout);
    AMB_CHECK_CUDA(cudaGetLastError());
    int32_t* t = kin;
    kin = kout;
    kout = t;
    t = ein;
    ein = eout;
    eout = t;
  }
  AMB_CHECK_CUDA(cudaMemsetAsync(s.start, 0xff, sizeof(int32_t) * P, st));
  segment_start_kernel<<<tiles, AR_SORT_TILE, 0, st>>>(kin, n, s.start);
  AMB_CHECK_CUDA(cudaGetLastError());
  pair_sum_kernel<<<(unsigned)((P + 127) / 128), 128, 0, st>>>(rest, faces, kin, ein, n, s.start, P, pair_count, pair_prior);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

extern "C" int amb_autorig_bone_weights(const int32_t* joints, const double* weights, int64_t n_vertices, int n_bones,
                                        double* scratch, double* totals, amb_stream_t stream) {
  AMB_CHECK_ARG(joints && weights && scratch && totals, "autorig_bone_weights: null pointer");
  AR_CHECK_BONES("autorig_bone_weights", n_vertices, n_bones);
  cudaStream_t st = (cudaStream_t)stream;
  const int tiles = tiles_of(n_vertices);
  bone_weight_partial_kernel<<<tiles, FP64_THREADS, 0, st>>>(joints, weights, n_vertices, n_bones, scratch);
  AMB_CHECK_CUDA(cudaGetLastError());
  bone_weight_sum_kernel<<<1, AR_MAX_BONES, 0, st>>>(scratch, tiles, n_bones, totals);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

extern "C" int amb_autorig_joint_solve(const double* transforms, int frames, int n_bones, const double* centres,
                                       const int32_t* pair_count, const double* pair_prior, const double* lambda,
                                       double* pair_joint, double* pair_cost, amb_stream_t stream) {
  AMB_CHECK_ARG(frames >= 1 && frames <= 65535 && n_bones >= 1 && n_bones <= AR_MAX_BONES,
                "autorig_joint_solve: bad frames %d or bones %d", frames, n_bones);
  const int64_t P = pair_count_of(n_bones);
  if (P == 0) return AMB_OK;  // one bone: no pair, and the (empty) outputs may be null
  AMB_CHECK_ARG(transforms && centres && pair_count && pair_prior && lambda && pair_joint && pair_cost,
                "autorig_joint_solve: null pointer");
  joint_solve_kernel<<<(unsigned)((P + AR_SOLVE_THREADS - 1) / AR_SOLVE_THREADS), AR_SOLVE_THREADS, 0,
                       (cudaStream_t)stream>>>(transforms, frames, n_bones, centres, pair_count, pair_prior, lambda,
                                               pair_joint, pair_cost);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

extern "C" int amb_autorig_slots(const int32_t* joints, const double* weights, int64_t n_vertices, int32_t* slot_bind,
                                 double* slot_weight, amb_stream_t stream) {
  AMB_CHECK_ARG(joints && weights && slot_bind && slot_weight, "autorig_slots: null pointer");
  AMB_CHECK_ARG(n_vertices >= 1 && n_vertices < (1ll << 31), "autorig_slots: bad vertex count %lld", (long long)n_vertices);
  slots_kernel<<<(unsigned)((n_vertices + 255) / 256), 256, 0, (cudaStream_t)stream>>>(joints, weights, n_vertices,
                                                                                       slot_bind, slot_weight);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

extern "C" int amb_autorig_list_scratch_ints(int64_t n_vertices, int n_joints, int64_t* out_ints) {
  AMB_CHECK_ARG(out_ints, "autorig_list_scratch_ints: null pointer");
  AMB_CHECK_ARG(n_vertices >= 1 && n_joints >= 1 && n_joints <= 1024 && n_vertices * n_joints < (1ll << 31) - 1,
                "autorig_list_scratch_ints: bad sizes (vertices %lld, joints %d)", (long long)n_vertices, n_joints);
  *out_ints = scan_tiles(n_vertices * n_joints) + 1;
  return AMB_OK;
}

extern "C" int amb_autorig_joint_lists(const int32_t* bind_joint, const int32_t* slot_bind, const double* slot_weight,
                                       int64_t n_vertices, const int32_t* subtree_end, int n_joints, int32_t* scratch,
                                       int32_t* lists, int64_t capacity, int32_t* offsets, amb_stream_t stream) {
  AMB_CHECK_ARG(bind_joint && slot_bind && slot_weight && subtree_end && scratch && lists && offsets,
                "autorig_joint_lists: null pointer");
  AMB_CHECK_ARG(n_vertices >= 1 && n_joints >= 1 && n_joints <= 1024 && n_vertices * n_joints < (1ll << 31) - 1 &&
                    capacity >= 0 && capacity < (1ll << 31),
                "autorig_joint_lists: bad sizes (vertices %lld, joints %d, capacity %lld)", (long long)n_vertices,
                n_joints, (long long)capacity);
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)n_vertices * n_joints;
  const JointLists jl{bind_joint, slot_bind, slot_weight, subtree_end, n_vertices, n_joints, lists, capacity, offsets};
  if (int rc = scan_count(n, jl, scratch, st)) return rc;
  return scan_emit(n, jl, scratch, st);
}
