// Post-processing of Stage 0's anchor mesh: parallel quadric edge-collapse decimation and floater removal.
//
// Replaces the reference's MeshPostprocessor.process_mesh (actionmesh/preprocessing/mesh_processor.py:104-161,288-325,374-425),
// which calls trimesh's simplify_quadric_decimation (fast_simplification) and split(only_watertight=False).  The host loop is
// actionmesh_b200/mesh_process.py; tests/mesh_process_ref.py restates every rule below in numpy float64 with the same operation
// order, and the kernels reproduce it bit for bit: every fp64 product, sum, quotient and square root is an explicit
// round-to-nearest intrinsic (nvcc never contracts them into an FMA), and every per-vertex sum runs in a fixed order.
//
// Meshes: positions (V, 3) fp64, faces (F, 3) int32 with three distinct indices in [0, V).  Decimation keeps V fixed and only
// rewrites faces; collapsed vertices become unreferenced and are compacted away at the end.
//
// One decimation round:
//   adjacency   vertex -> face CSR (count, scan, fill, then each list sorted by face index) and, per vertex, the sorted list of
//               the other two corners of its faces ("neighbour slots": a neighbour w appears once per face holding the edge).
//   edges       per vertex a, its distinct neighbours b > a in ascending order (so edges are ordered by (a, b)), with the
//               number of faces holding the edge and, for edges with <= 2 faces, those faces in ascending order.  Vertex flags:
//               bit 0 boundary (an edge with 1 face), bit 1 non-manifold (an edge with > 2 faces).
//   select      validity, target x* and cost per edge; key = (fp32 bits of cost, rounded up) << 32 | edge index; m1(v) = min
//               key of the valid edges at v; m2(v) = min of m1 over v and its 1-ring; an edge wins iff key == m2(a) == m2(b).
//               Two winners never share or neighbour an endpoint, so their collapses do not interact.
//   apply       winners with key <= limit: b -> a, a moves to x*, Q_a += Q_b.  Faces that repeat an index are dropped.
#include <cuda_runtime.h>
#include <cstdint>
#include "common.cuh"
#include "scan.cuh"
#include "../../include/actionmesh_b200.h"

namespace amb {
namespace {

constexpr double kDetRel = 1e-10;          // x* = A^-1 (-b) only when |det A| > kDetRel * A00 A11 A22 (Hadamard: det <= product)
constexpr double kBoundaryWeight = 100.0;  // boundary-edge plane weight, times |edge|^2
constexpr double kMinCos2 = 0.0625;        // a surviving face's new unit normal . old >= 0.25 (squared, with dot > 0)
constexpr unsigned long long kNoKey = ~0ull;

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }

struct V3 {
  double x, y, z;
};

__device__ __forceinline__ V3 load3(const double* p, long long i) { return {p[3 * i], p[3 * i + 1], p[3 * i + 2]}; }
__device__ __forceinline__ V3 sub3(V3 a, V3 b) { return {dsub(a.x, b.x), dsub(a.y, b.y), dsub(a.z, b.z)}; }
__device__ __forceinline__ V3 cross3(V3 a, V3 b) {
  return {dsub(dmul(a.y, b.z), dmul(a.z, b.y)), dsub(dmul(a.z, b.x), dmul(a.x, b.z)), dsub(dmul(a.x, b.y), dmul(a.y, b.x))};
}
__device__ __forceinline__ double dot3(V3 a, V3 b) { return dadd(dadd(dmul(a.x, b.x), dmul(a.y, b.y)), dmul(a.z, b.z)); }
// cross(p1 - p0, p2 - p0): twice the area times the unit normal
__device__ __forceinline__ V3 tri_normal(V3 p0, V3 p1, V3 p2) { return cross3(sub3(p1, p0), sub3(p2, p0)); }

// q += w * (p p^T) for the plane p = (u, d) with unit normal u; q = [xx xy xz xd yy yz yd zz zd dd]
__device__ __forceinline__ void add_plane(double* q, V3 u, double d, double w) {
  const double p[4] = {u.x, u.y, u.z, d};
  int k = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = i; j < 4; ++j, ++k) q[k] = dadd(q[k], dmul(w, dmul(p[i], p[j])));
}

// plane through p0 with normal n, weight w(|n|); nothing when |n| == 0
__device__ __forceinline__ void add_face_plane(double* q, V3 p0, V3 n) {
  const double nn = dot3(n, n);
  if (!(nn > 0.0)) return;
  const double len = __dsqrt_rn(nn);
  const V3 u = {__ddiv_rn(n.x, len), __ddiv_rn(n.y, len), __ddiv_rn(n.z, len)};
  add_plane(q, u, -dot3(u, p0), dmul(0.5, len));                                 // area-weighted
}

// boundary edge pa -> pb (a < b) of a face with normal n: the plane through the edge perpendicular to the face
__device__ __forceinline__ void add_boundary_plane(double* q, V3 pa, V3 pb, V3 n) {
  const V3 e = sub3(pb, pa);
  const V3 m = cross3(e, n);
  const double mm = dot3(m, m);
  if (!(mm > 0.0)) return;
  const double len = __dsqrt_rn(mm);
  const V3 u = {__ddiv_rn(m.x, len), __ddiv_rn(m.y, len), __ddiv_rn(m.z, len)};
  add_plane(q, u, -dot3(u, pa), dmul(kBoundaryWeight, dot3(e, e)));
}

// v^T Q v for v = (x, 1)
__device__ __forceinline__ double quadric_error(const double* q, V3 p) {
  const double r0 = dadd(dadd(dadd(dmul(q[0], p.x), dmul(q[1], p.y)), dmul(q[2], p.z)), q[3]);
  const double r1 = dadd(dadd(dadd(dmul(q[1], p.x), dmul(q[4], p.y)), dmul(q[5], p.z)), q[6]);
  const double r2 = dadd(dadd(dadd(dmul(q[2], p.x), dmul(q[5], p.y)), dmul(q[7], p.z)), q[8]);
  const double r3 = dadd(dadd(dadd(dmul(q[3], p.x), dmul(q[6], p.y)), dmul(q[8], p.z)), q[9]);
  return dadd(dadd(dadd(dmul(p.x, r0), dmul(p.y, r1)), dmul(p.z, r2)), r3);
}

__device__ void sift_down(int32_t* a, int root, int n) {
  const int32_t v = a[root];
  for (;;) {
    int child = 2 * root + 1;
    if (child >= n) break;
    if (child + 1 < n && a[child + 1] > a[child]) ++child;
    if (a[child] <= v) break;
    a[root] = a[child];
    root = child;
  }
  a[root] = v;
}

// in-place heap sort: O(d log d) for vertices of any degree (a 1000-face fan's centre included)
__device__ void heap_sort(int32_t* a, int n) {
  for (int s = n / 2 - 1; s >= 0; --s) sift_down(a, s, n);
  for (int e = n - 1; e > 0; --e) {
    const int32_t t = a[0];
    a[0] = a[e];
    a[e] = t;
    sift_down(a, 0, e);
  }
}

__device__ __forceinline__ bool has_vertex(const int32_t* faces, int f, int v) {
  return faces[3LL * f] == v || faces[3LL * f + 1] == v || faces[3LL * f + 2] == v;
}

// ---- adjacency -------------------------------------------------------------------------------------------------------------

__global__ void degree_kernel(const int32_t* __restrict__ faces, long long n3, int32_t* __restrict__ deg) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n3; i += (long long)gridDim.x * blockDim.x)
    atomicAdd(&deg[faces[i]], 1);
}

struct Offsets {
  const int32_t* deg;
  int32_t* off;
  __device__ int count(long long v) const { return deg[v]; }
  __device__ void emit(long long v, int o) const { off[v] = o; }
};

__global__ void fill_kernel(const int32_t* __restrict__ faces, long long n3, const int32_t* __restrict__ off,
                            int32_t* __restrict__ cursor, int32_t* __restrict__ vf) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n3; i += (long long)gridDim.x * blockDim.x) {
    const int v = faces[i];
    vf[off[v] + atomicAdd(&cursor[v], 1)] = (int32_t)(i / 3);
  }
}

// sort each vertex's faces, then write and sort its neighbour slots (the other two corners of each face)
__global__ void sort_kernel(const int32_t* __restrict__ faces, int n_vertices, const int32_t* __restrict__ off,
                            int32_t* __restrict__ vf, int32_t* __restrict__ nb) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n_vertices; v += gridDim.x * blockDim.x) {
    const int s = off[v], d = off[v + 1] - s;
    heap_sort(vf + s, d);
    int32_t* slots = nb + 2LL * s;
    for (int k = 0; k < d; ++k) {
      const int f = vf[s + k];
      int j = 0;
      for (int c = 0; c < 3; ++c) {
        const int w = faces[3LL * f + c];
        if (w != v && j < 2) slots[2 * k + j++] = w;
      }
    }
    heap_sort(slots, 2 * d);
  }
}

// number of edges (a, b > a): distinct neighbour slots above a; emit records each vertex's first edge index
struct EdgeOffsets {
  const int32_t* off;
  const int32_t* nb;
  int32_t* first;
  __device__ int count(long long a) const {
    const long long s = 2LL * off[a], e = 2LL * off[a + 1];
    int n = 0;
    for (long long k = s; k < e; ++k) n += (nb[k] > a && (k == s || nb[k] != nb[k - 1])) ? 1 : 0;
    return n;
  }
  __device__ void emit(long long a, int o) const { first[a] = o; }
};

// edges of vertex a from its sorted neighbour slots, and its flags
__global__ void edges_kernel(const int32_t* __restrict__ faces, int n_vertices, const int32_t* __restrict__ off,
                             const int32_t* __restrict__ vf, const int32_t* __restrict__ nb, const int32_t* __restrict__ first,
                             int32_t* __restrict__ edges, uint8_t* __restrict__ flags) {
  for (int a = blockIdx.x * blockDim.x + threadIdx.x; a < n_vertices; a += gridDim.x * blockDim.x) {
    const long long s = 2LL * off[a], e = 2LL * off[a + 1];
    int o = first[a];
    uint8_t fl = 0;
    for (long long k = s; k < e;) {
      const int w = nb[k];
      long long r = k;
      while (r < e && nb[r] == w) ++r;
      const int len = (int)(r - k);
      fl |= (len == 1 ? 1 : 0) | (len > 2 ? 2 : 0);
      if (w > a) {
        int f0 = -1, f1 = -1;
        if (len <= 2) {
          for (int t = off[a]; t < off[a + 1] && f1 < 0; ++t) {
            if (!has_vertex(faces, vf[t], w)) continue;
            if (f0 < 0) f0 = vf[t]; else f1 = vf[t];
          }
        }
        int32_t* ed = edges + 5LL * o++;
        ed[0] = a; ed[1] = w; ed[2] = len; ed[3] = f0; ed[4] = f1;
      }
      k = r;
    }
    flags[a] = fl;
  }
}

// ---- quadrics --------------------------------------------------------------------------------------------------------------

// Q_v = the area-weighted face planes in face order, then the boundary-edge planes in ascending order of the other endpoint
__global__ void quadrics_kernel(const double* __restrict__ pos, const int32_t* __restrict__ faces, int n_vertices,
                                const int32_t* __restrict__ off, const int32_t* __restrict__ vf, const int32_t* __restrict__ nb,
                                double* __restrict__ quadrics) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n_vertices; v += gridDim.x * blockDim.x) {
    double q[10];
#pragma unroll
    for (int i = 0; i < 10; ++i) q[i] = 0.0;
    for (int t = off[v]; t < off[v + 1]; ++t) {
      const int f = vf[t];
      const V3 p0 = load3(pos, faces[3LL * f]), p1 = load3(pos, faces[3LL * f + 1]), p2 = load3(pos, faces[3LL * f + 2]);
      add_face_plane(q, p0, tri_normal(p0, p1, p2));
    }
    const long long s = 2LL * off[v], e = 2LL * off[v + 1];
    for (long long k = s; k < e;) {
      const int w = nb[k];
      long long r = k;
      while (r < e && nb[r] == w) ++r;
      if (r - k == 1) {
        int f = -1;
        for (int t = off[v]; t < off[v + 1] && f < 0; ++t)
          if (has_vertex(faces, vf[t], w)) f = vf[t];
        const V3 p0 = load3(pos, faces[3LL * f]), p1 = load3(pos, faces[3LL * f + 1]), p2 = load3(pos, faces[3LL * f + 2]);
        const int a = v < w ? v : w, b = v < w ? w : v;
        add_boundary_plane(q, load3(pos, a), load3(pos, b), tri_normal(p0, p1, p2));
      }
      k = r;
    }
#pragma unroll
    for (int i = 0; i < 10; ++i) quadrics[10LL * v + i] = q[i];
  }
}

// ---- selection ---------------------------------------------------------------------------------------------------------------

// every face of v that does not hold `other` keeps a positive area and turns by less than acos(0.25) when v moves to x
__device__ bool faces_stay_valid(const double* pos, const int32_t* faces, const int32_t* off, const int32_t* vf, int v,
                                 int other, V3 x) {
  for (int t = off[v]; t < off[v + 1]; ++t) {
    const int f = vf[t];
    const int c0 = faces[3LL * f], c1 = faces[3LL * f + 1], c2 = faces[3LL * f + 2];
    if (c0 == other || c1 == other || c2 == other) continue;
    const V3 p0 = load3(pos, c0), p1 = load3(pos, c1), p2 = load3(pos, c2);
    const V3 n_old = tri_normal(p0, p1, p2);
    const V3 n_new = tri_normal(c0 == v ? x : p0, c1 == v ? x : p1, c2 == v ? x : p2);
    const double nn_new = dot3(n_new, n_new), nn_old = dot3(n_old, n_old);
    if (!(nn_new > 0.0)) return false;
    if (nn_old > 0.0) {
      const double d = dot3(n_new, n_old);
      if (!(d > 0.0) || dmul(d, d) < dmul(kMinCos2, dmul(nn_new, nn_old))) return false;
    }
  }
  return true;
}

__global__ void select_kernel(const double* __restrict__ pos, const double* __restrict__ quadrics,
                              const int32_t* __restrict__ faces, const int32_t* __restrict__ off, const int32_t* __restrict__ vf,
                              const int32_t* __restrict__ nb, const int32_t* __restrict__ edges, int n_edges,
                              const uint8_t* __restrict__ flags, unsigned long long* __restrict__ keys,
                              double* __restrict__ targets, unsigned long long* __restrict__ m1) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n_edges; e += gridDim.x * blockDim.x) {
    const int a = edges[5LL * e], b = edges[5LL * e + 1], nf = edges[5LL * e + 2];
    const uint8_t fa = flags[a], fb = flags[b];
    // manifold edge, no endpoint on a non-manifold edge, and an edge between two boundary vertices must be a boundary edge
    bool ok = nf <= 2 && !((fa | fb) & 2) && !((fa & fb & 1) && nf != 1);
    if (ok) {   // link condition: |N(a) ∩ N(b)| == face count
      long long i = 2LL * off[a], ie = 2LL * off[a + 1], j = 2LL * off[b], je = 2LL * off[b + 1];
      int common = 0;
      while (i < ie && j < je) {
        const int x = nb[i], y = nb[j];
        if (x < y) {
          ++i;
        } else if (y < x) {
          ++j;
        } else {
          ++common;
          while (i < ie && nb[i] == x) ++i;
          while (j < je && nb[j] == x) ++j;
        }
      }
      ok = common == nf;
    }
    V3 x = {0.0, 0.0, 0.0};
    double cost = 0.0;
    if (ok) {
      double q[10];
#pragma unroll
      for (int k = 0; k < 10; ++k) q[k] = dadd(quadrics[10LL * a + k], quadrics[10LL * b + k]);
      const V3 pa = load3(pos, a), pb = load3(pos, b);
      const V3 pm = {dmul(dadd(pa.x, pb.x), 0.5), dmul(dadd(pa.y, pb.y), 0.5), dmul(dadd(pa.z, pb.z), 0.5)};
      // best of a, b and the midpoint, ties to a
      x = pa;
      cost = quadric_error(q, pa);
      const double eb = quadric_error(q, pb), em = quadric_error(q, pm);
      if (eb < cost) { x = pb; cost = eb; }
      if (em < cost) { x = pm; cost = em; }
      // the minimiser of Q_a + Q_b by the adjugate, when well conditioned and no worse than those
      const double c00 = dsub(dmul(q[4], q[7]), dmul(q[5], q[5])), c01 = dsub(dmul(q[2], q[5]), dmul(q[1], q[7]));
      const double c02 = dsub(dmul(q[1], q[5]), dmul(q[2], q[4])), c11 = dsub(dmul(q[0], q[7]), dmul(q[2], q[2]));
      const double c12 = dsub(dmul(q[1], q[2]), dmul(q[0], q[5])), c22 = dsub(dmul(q[0], q[4]), dmul(q[1], q[1]));
      const double det = dadd(dadd(dmul(q[0], c00), dmul(q[1], c01)), dmul(q[2], c02));
      if (fabs(det) > dmul(kDetRel, dmul(dmul(q[0], q[4]), q[7]))) {
        const V3 xs = {__ddiv_rn(-dadd(dadd(dmul(c00, q[3]), dmul(c01, q[6])), dmul(c02, q[8])), det),
                       __ddiv_rn(-dadd(dadd(dmul(c01, q[3]), dmul(c11, q[6])), dmul(c12, q[8])), det),
                       __ddiv_rn(-dadd(dadd(dmul(c02, q[3]), dmul(c12, q[6])), dmul(c22, q[8])), det)};
        const double es = quadric_error(q, xs);
        if (es <= cost) { x = xs; cost = es; }
      }
      if (!(cost > 0.0)) cost = 0.0;
      ok = faces_stay_valid(pos, faces, off, vf, a, b, x) && faces_stay_valid(pos, faces, off, vf, b, a, x);
    }
    unsigned long long key = kNoKey;
    if (ok) {
      key = ((unsigned long long)__float_as_uint(__double2float_ru(cost)) << 32) | (unsigned int)e;
      atomicMin(&m1[a], key);
      atomicMin(&m1[b], key);
    }
    keys[e] = key;
    targets[3LL * e] = x.x;
    targets[3LL * e + 1] = x.y;
    targets[3LL * e + 2] = x.z;
  }
}

// m2(v) = min of m1 over v and its 1-ring; the round's remap starts as the identity
__global__ void ring_min_kernel(int n_vertices, const int32_t* __restrict__ off, const int32_t* __restrict__ nb,
                                const unsigned long long* __restrict__ m1, unsigned long long* __restrict__ m2,
                                int32_t* __restrict__ remap) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n_vertices; v += gridDim.x * blockDim.x) {
    unsigned long long m = m1[v];
    for (long long k = 2LL * off[v]; k < 2LL * off[v + 1]; ++k) {
      const unsigned long long w = m1[nb[k]];
      m = w < m ? w : m;
    }
    m2[v] = m;
    remap[v] = v;
  }
}

__device__ __forceinline__ bool wins(const unsigned long long* keys, const unsigned long long* m2, int e, int a, int b) {
  const unsigned long long key = keys[e];
  return key != kNoKey && key == m2[a] && key == m2[b];
}

// counters[0] += winners, counters[1] += faces they remove; winners[2i], winners[2i+1] = key, face count (unordered)
__global__ void winners_kernel(const int32_t* __restrict__ edges, int n_edges, const unsigned long long* __restrict__ keys,
                               const unsigned long long* __restrict__ m2, unsigned long long* __restrict__ counters,
                               unsigned long long* __restrict__ winners) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n_edges; e += gridDim.x * blockDim.x) {
    const int a = edges[5LL * e], b = edges[5LL * e + 1], nf = edges[5LL * e + 2];
    if (!wins(keys, m2, e, a, b)) continue;
    const unsigned long long i = atomicAdd(&counters[0], 1ull);
    atomicAdd(&counters[1], (unsigned long long)nf);
    winners[2 * i] = keys[e];
    winners[2 * i + 1] = (unsigned long long)nf;
  }
}

__global__ void apply_kernel(const int32_t* __restrict__ edges, int n_edges, const unsigned long long* __restrict__ keys,
                             const unsigned long long* __restrict__ m2, const double* __restrict__ targets,
                             unsigned long long limit, int32_t* __restrict__ remap, double* __restrict__ pos,
                             double* __restrict__ quadrics) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n_edges; e += gridDim.x * blockDim.x) {
    const int a = edges[5LL * e], b = edges[5LL * e + 1];
    if (!wins(keys, m2, e, a, b) || keys[e] > limit) continue;
    remap[b] = a;
    pos[3LL * a] = targets[3LL * e];
    pos[3LL * a + 1] = targets[3LL * e + 1];
    pos[3LL * a + 2] = targets[3LL * e + 2];
#pragma unroll
    for (int k = 0; k < 10; ++k) quadrics[10LL * a + k] = dadd(quadrics[10LL * a + k], quadrics[10LL * b + k]);
  }
}

// ---- compaction ------------------------------------------------------------------------------------------------------------

// faces whose (remapped) corners are distinct and, with labels, whose component has >= min_size faces
struct FaceCompact {
  const int32_t* faces;
  const int32_t* remap;
  const int32_t* labels;
  const int32_t* sizes;
  int min_size;
  int32_t* out;
  __device__ bool corners(long long f, int c[3]) const {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      c[k] = faces[3 * f + k];
      if (remap) c[k] = remap[c[k]];
    }
    return c[0] != c[1] && c[1] != c[2] && c[0] != c[2] && (!labels || sizes[labels[f]] >= min_size);
  }
  __device__ int count(long long f) const {
    int c[3];
    return corners(f, c) ? 1 : 0;
  }
  __device__ void emit(long long f, int o) const {
    int c[3];
    if (!corners(f, c)) return;
    out[3LL * o] = c[0]; out[3LL * o + 1] = c[1]; out[3LL * o + 2] = c[2];
  }
};

__global__ void mark_used_kernel(const int32_t* __restrict__ faces, long long n3, int32_t* __restrict__ used) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n3; i += (long long)gridDim.x * blockDim.x)
    used[faces[i]] = 1;
}

// referenced vertices in index order; index[v] becomes the new index (-1 for dropped vertices)
struct VertexCompact {
  const double* pos;
  int32_t* index;
  double* out;
  __device__ int count(long long v) const { return index[v]; }
  __device__ void emit(long long v, int o) const {
    const bool used = index[v] != 0;
    index[v] = used ? o : -1;
    if (!used) return;
    out[3LL * o] = pos[3 * v]; out[3LL * o + 1] = pos[3 * v + 1]; out[3LL * o + 2] = pos[3 * v + 2];
  }
};

__global__ void reindex_kernel(const int32_t* __restrict__ faces, long long n3, const int32_t* __restrict__ index,
                               int32_t* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n3; i += (long long)gridDim.x * blockDim.x)
    out[i] = index[faces[i]];
}

// ---- connected components over faces ----------------------------------------------------------------------------------------

__global__ void iota_kernel(int32_t* __restrict__ labels, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) labels[i] = i;
}

__device__ __forceinline__ int find_root(const int32_t* labels, int x) {
  int p = labels[x];
  while (p != x) {
    x = p;
    p = labels[x];
  }
  return x;
}

// union over edges with exactly 2 faces: the larger root is hooked under the smaller, so labels only ever decrease and
// every tree's root is the smallest face index in it
__global__ void hook_kernel(const int32_t* __restrict__ edges, int n_edges, int32_t* labels, int32_t* __restrict__ changed) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n_edges; e += gridDim.x * blockDim.x) {
    if (edges[5LL * e + 2] != 2) continue;
    const int u = find_root(labels, edges[5LL * e + 3]), v = find_root(labels, edges[5LL * e + 4]);
    if (u == v) continue;
    atomicMin(&labels[u > v ? u : v], u < v ? u : v);
    *changed = 1;
  }
}

__global__ void compress_kernel(int32_t* labels, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) labels[i] = find_root(labels, i);
}

__global__ void sizes_kernel(const int32_t* __restrict__ labels, int n, int32_t* __restrict__ sizes) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) atomicAdd(&sizes[labels[i]], 1);
}

constexpr int kThreads = 256;

bool mesh_size_ok(int64_t n_vertices, int64_t n_faces) {
  return n_vertices >= 0 && n_faces >= 0 && n_vertices < (1LL << 31) - 1 && 6 * n_faces < (1LL << 31);
}

}  // namespace
}  // namespace amb

using namespace amb;

#define AMB_MESH_SIZES(fn, nv, nf)                                                                                      \
  AMB_CHECK_ARG(mesh_size_ok(nv, nf), fn ": bad mesh size (%lld vertices, %lld faces)", (long long)(nv), (long long)(nf))

extern "C" {

int amb_mesh_adjacency(const int32_t* faces, int64_t n_faces, int64_t n_vertices, int32_t* work, int32_t* scan,
                       int32_t* vf_offsets, int32_t* vf_faces, int32_t* neighbours, amb_stream_t stream) {
  AMB_CHECK_ARG(faces && work && scan && vf_offsets && vf_faces && neighbours, "mesh_adjacency: null pointer");
  AMB_MESH_SIZES("mesh_adjacency", n_vertices, n_faces);
  if (!n_faces || !n_vertices) return AMB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const long long n3 = 3 * n_faces;
  const int nv = (int)n_vertices;
  AMB_CHECK_CUDA(cudaMemsetAsync(work, 0, sizeof(int32_t) * nv, st));
  degree_kernel<<<blocks_for(n3, kThreads), kThreads, 0, st>>>(faces, n3, work);
  AMB_CHECK_CUDA(cudaGetLastError());
  Offsets fo{work, vf_offsets};
  if (int rc = scan_count(nv, fo, scan, st)) return rc;
  if (int rc = scan_emit(nv, fo, scan, st)) return rc;
  AMB_CHECK_CUDA(cudaMemcpyAsync(vf_offsets + nv, scan + scan_tiles(nv), sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  AMB_CHECK_CUDA(cudaMemsetAsync(work, 0, sizeof(int32_t) * nv, st));
  fill_kernel<<<blocks_for(n3, kThreads), kThreads, 0, st>>>(faces, n3, vf_offsets, work, vf_faces);
  sort_kernel<<<blocks_for(nv, kThreads), kThreads, 0, st>>>(faces, nv, vf_offsets, vf_faces, neighbours);
  AMB_CHECK_CUDA(cudaGetLastError());
  EdgeOffsets fe{vf_offsets, neighbours, nullptr};
  return scan_count(nv, fe, scan, st);
}

int amb_mesh_edges(const int32_t* faces, int64_t n_faces, int64_t n_vertices, const int32_t* vf_offsets,
                   const int32_t* vf_faces, const int32_t* neighbours, int32_t* work, const int32_t* scan, int32_t* edges,
                   uint8_t* flags, amb_stream_t stream) {
  AMB_CHECK_ARG(faces && vf_offsets && vf_faces && neighbours && work && scan && edges && flags, "mesh_edges: null pointer");
  AMB_MESH_SIZES("mesh_edges", n_vertices, n_faces);
  if (!n_faces || !n_vertices) return AMB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  EdgeOffsets fe{vf_offsets, neighbours, work};
  if (int rc = scan_emit(n_vertices, fe, scan, st)) return rc;
  edges_kernel<<<blocks_for(n_vertices, kThreads), kThreads, 0, st>>>(faces, (int)n_vertices, vf_offsets, vf_faces, neighbours,
                                                                      work, edges, flags);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_mesh_quadrics(const double* positions, const int32_t* faces, int64_t n_vertices, const int32_t* vf_offsets,
                      const int32_t* vf_faces, const int32_t* neighbours, double* quadrics, amb_stream_t stream) {
  AMB_CHECK_ARG(positions && faces && vf_offsets && vf_faces && neighbours && quadrics, "mesh_quadrics: null pointer");
  AMB_MESH_SIZES("mesh_quadrics", n_vertices, 0);
  if (!n_vertices) return AMB_OK;
  quadrics_kernel<<<blocks_for(n_vertices, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      positions, faces, (int)n_vertices, vf_offsets, vf_faces, neighbours, quadrics);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_mesh_collapse_select(const double* positions, const double* quadrics, const int32_t* faces, int64_t n_vertices,
                             const int32_t* vf_offsets, const int32_t* vf_faces, const int32_t* neighbours,
                             const int32_t* edges, int64_t n_edges, const uint8_t* flags, uint64_t* keys, double* targets,
                             uint64_t* vertex_min, int32_t* remap, uint64_t* counters, uint64_t* winners,
                             amb_stream_t stream) {
  AMB_CHECK_ARG(positions && quadrics && faces && vf_offsets && vf_faces && neighbours && edges && flags && keys && targets &&
                    vertex_min && remap && counters && winners,
                "mesh_collapse_select: null pointer");
  AMB_MESH_SIZES("mesh_collapse_select", n_vertices, 0);
  AMB_CHECK_ARG(n_edges >= 0 && n_edges < (1LL << 31), "mesh_collapse_select: bad edge count %lld", (long long)n_edges);
  cudaStream_t st = (cudaStream_t)stream;
  AMB_CHECK_CUDA(cudaMemsetAsync(counters, 0, 2 * sizeof(uint64_t), st));
  if (!n_edges || !n_vertices) return AMB_OK;
  const int nv = (int)n_vertices, ne = (int)n_edges;
  unsigned long long* m1 = reinterpret_cast<unsigned long long*>(vertex_min);
  unsigned long long* m2 = m1 + nv;
  AMB_CHECK_CUDA(cudaMemsetAsync(m1, 0xff, sizeof(uint64_t) * nv, st));
  select_kernel<<<blocks_for(ne, kThreads), kThreads, 0, st>>>(positions, quadrics, faces, vf_offsets, vf_faces, neighbours,
                                                               edges, ne, flags, reinterpret_cast<unsigned long long*>(keys),
                                                               targets, m1);
  ring_min_kernel<<<blocks_for(nv, kThreads), kThreads, 0, st>>>(nv, vf_offsets, neighbours, m1, m2, remap);
  winners_kernel<<<blocks_for(ne, kThreads), kThreads, 0, st>>>(edges, ne, reinterpret_cast<unsigned long long*>(keys), m2,
                                                                reinterpret_cast<unsigned long long*>(counters),
                                                                reinterpret_cast<unsigned long long*>(winners));
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_mesh_collapse_apply(const int32_t* edges, int64_t n_edges, int64_t n_vertices, const uint64_t* keys,
                            const double* targets, const uint64_t* vertex_min, uint64_t key_limit, int32_t* remap,
                            double* positions, double* quadrics, amb_stream_t stream) {
  AMB_CHECK_ARG(edges && keys && targets && vertex_min && remap && positions && quadrics, "mesh_collapse_apply: null pointer");
  AMB_MESH_SIZES("mesh_collapse_apply", n_vertices, 0);
  AMB_CHECK_ARG(n_edges >= 0 && n_edges < (1LL << 31), "mesh_collapse_apply: bad edge count %lld", (long long)n_edges);
  if (!n_edges || !n_vertices) return AMB_OK;
  const unsigned long long* m2 = reinterpret_cast<const unsigned long long*>(vertex_min) + n_vertices;
  apply_kernel<<<blocks_for(n_edges, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      edges, (int)n_edges, reinterpret_cast<const unsigned long long*>(keys), m2, targets, key_limit, remap, positions,
      quadrics);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_mesh_compact_faces(const int32_t* faces, int64_t n_faces, const int32_t* remap, const int32_t* labels,
                           const int32_t* sizes, int min_size, int32_t* scan, int32_t* out_faces, amb_stream_t stream) {
  AMB_CHECK_ARG(faces && scan && out_faces && (!labels || sizes), "mesh_compact_faces: null pointer");
  AMB_CHECK_ARG(faces != out_faces, "mesh_compact_faces: out_faces must not alias faces");
  AMB_MESH_SIZES("mesh_compact_faces", 0, n_faces);
  if (!n_faces) return AMB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  FaceCompact fc{faces, remap, labels, sizes, min_size, out_faces};
  if (int rc = scan_count(n_faces, fc, scan, st)) return rc;
  return scan_emit(n_faces, fc, scan, st);
}

int amb_mesh_compact_vertices(const double* positions, int64_t n_vertices, const int32_t* faces, int64_t n_faces,
                              int32_t* work, int32_t* scan, double* out_positions, int32_t* out_faces, amb_stream_t stream) {
  AMB_CHECK_ARG(positions && faces && work && scan && out_positions && out_faces, "mesh_compact_vertices: null pointer");
  AMB_CHECK_ARG(faces != out_faces, "mesh_compact_vertices: out_faces must not alias faces");
  AMB_MESH_SIZES("mesh_compact_vertices", n_vertices, n_faces);
  if (!n_vertices) return AMB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const long long n3 = 3 * n_faces;
  AMB_CHECK_CUDA(cudaMemsetAsync(work, 0, sizeof(int32_t) * n_vertices, st));
  if (n3) mark_used_kernel<<<blocks_for(n3, kThreads), kThreads, 0, st>>>(faces, n3, work);
  AMB_CHECK_CUDA(cudaGetLastError());
  VertexCompact fv{positions, work, out_positions};
  if (int rc = scan_count(n_vertices, fv, scan, st)) return rc;
  if (int rc = scan_emit(n_vertices, fv, scan, st)) return rc;
  if (n3) reindex_kernel<<<blocks_for(n3, kThreads), kThreads, 0, st>>>(faces, n3, work, out_faces);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_mesh_components(const int32_t* edges, int64_t n_edges, int64_t n_faces, int first, int32_t* labels, int32_t* changed,
                        amb_stream_t stream) {
  AMB_CHECK_ARG(edges && labels && changed, "mesh_components: null pointer");
  AMB_MESH_SIZES("mesh_components", 0, n_faces);
  AMB_CHECK_ARG(n_edges >= 0 && n_edges < (1LL << 31), "mesh_components: bad edge count %lld", (long long)n_edges);
  cudaStream_t st = (cudaStream_t)stream;
  AMB_CHECK_CUDA(cudaMemsetAsync(changed, 0, sizeof(int32_t), st));
  if (!n_faces) return AMB_OK;
  const int nf = (int)n_faces;
  if (first) iota_kernel<<<blocks_for(nf, kThreads), kThreads, 0, st>>>(labels, nf);
  if (n_edges) hook_kernel<<<blocks_for(n_edges, kThreads), kThreads, 0, st>>>(edges, (int)n_edges, labels, changed);
  compress_kernel<<<blocks_for(nf, kThreads), kThreads, 0, st>>>(labels, nf);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_mesh_component_sizes(const int32_t* labels, int64_t n_faces, int32_t* sizes, amb_stream_t stream) {
  AMB_CHECK_ARG(labels && sizes, "mesh_component_sizes: null pointer");
  AMB_MESH_SIZES("mesh_component_sizes", 0, n_faces);
  if (!n_faces) return AMB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  AMB_CHECK_CUDA(cudaMemsetAsync(sizes, 0, sizeof(int32_t) * n_faces, st));
  sizes_kernel<<<blocks_for(n_faces, kThreads), kThreads, 0, st>>>(labels, (int)n_faces, sizes);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

}  // extern "C"
