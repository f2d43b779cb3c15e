// fp64 building blocks shared by the skinning decomposition (skinning.cu, DESIGN.md §20) and the rig fit (rig.cu, §21).
// Every product, sum, quotient and square root is an explicit round-to-nearest intrinsic, so nvcc never contracts two of
// them into an FMA, and every sum runs in a fixed order: results do not depend on scheduling.  Transforms are 12 doubles,
// the 3x3 linear part row-major then the translation, mapping p to L p + t.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace amb {
namespace {

constexpr int FP64_THREADS = 256;   // reduction kernels: one item per thread, 8 warps; a tile is 256 items
constexpr int HORN_SWEEPS = 10;     // cyclic Jacobi sweeps of Horn's 4x4 matrix

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

struct V3 {
  double x, y, z;
};

__device__ __forceinline__ V3 load3(const double* p, int64_t i) { return {p[3 * i], p[3 * i + 1], p[3 * i + 2]}; }
__device__ __forceinline__ V3 sub3(V3 a, V3 b) { return {dsub(a.x, b.x), dsub(a.y, b.y), dsub(a.z, b.z)}; }
__device__ __forceinline__ double norm2(V3 r) { return dadd(dadd(dmul(r.x, r.x), dmul(r.y, r.y)), dmul(r.z, r.z)); }
__device__ __forceinline__ double dot3(V3 a, V3 b) { return dadd(dadd(dmul(a.x, b.x), dmul(a.y, b.y)), dmul(a.z, b.z)); }

// u_a = ((R_a0 p_x + R_a1 p_y) + R_a2 p_z) + t_a
__device__ __forceinline__ V3 apply_xf(const double* __restrict__ m, V3 p) {
  return {dadd(dadd(dadd(dmul(m[0], p.x), dmul(m[1], p.y)), dmul(m[2], p.z)), m[9]),
          dadd(dadd(dadd(dmul(m[3], p.x), dmul(m[4], p.y)), dmul(m[5], p.z)), m[10]),
          dadd(dadd(dadd(dmul(m[6], p.x), dmul(m[7], p.y)), dmul(m[8], p.z)), m[11])};
}

// Block sum of v[0..N) into out[0..N): a halving tree over the 32 lanes of each warp (shuffle down 16, 8, 4, 2, 1), then a
// halving tree over the 8 warps (4, 2, 1).
template <int N>
__device__ __forceinline__ void block_sum(const double* v, double (*red)[N], double* __restrict__ out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    double a = v[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a = dadd(a, __shfl_down_sync(0xffffffffu, a, o));
    if (lane == 0) red[warp][k] = a;
  }
  __syncthreads();
  if (threadIdx.x < N) {
    double w[FP64_THREADS / 32];
#pragma unroll
    for (int i = 0; i < FP64_THREADS / 32; ++i) w[i] = red[i][threadIdx.x];
#pragma unroll
    for (int n = FP64_THREADS / 64; n > 0; n >>= 1)
#pragma unroll
      for (int i = 0; i < n; ++i) w[i] = dadd(w[i], w[i + n]);
    out[threadIdx.x] = w[0];
  }
}

// One Jacobi rotation of the symmetric 4x4 A at (p, q), accumulated into the eigenvectors E (columns).
template <int P, int Q>
__device__ __forceinline__ void jacobi_rotate(double (&A)[4][4], double (&E)[4][4]) {
  const double apq = A[P][Q];
  if (apq == 0.0) return;
  const double theta = ddiv(dsub(A[Q][Q], A[P][P]), dmul(2.0, apq));
  const double t = ddiv(theta >= 0.0 ? 1.0 : -1.0, dadd(fabs(theta), __dsqrt_rn(dadd(dmul(theta, theta), 1.0))));
  const double c = ddiv(1.0, __dsqrt_rn(dadd(dmul(t, t), 1.0)));
  const double s = dmul(t, c);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double kp = A[k][P], kq = A[k][Q];
    A[k][P] = dsub(dmul(c, kp), dmul(s, kq));
    A[k][Q] = dadd(dmul(s, kp), dmul(c, kq));
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double pk = A[P][k], qk = A[Q][k];
    A[P][k] = dsub(dmul(c, pk), dmul(s, qk));
    A[Q][k] = dadd(dmul(s, pk), dmul(c, qk));
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double kp = E[k][P], kq = E[k][Q];
    E[k][P] = dsub(dmul(c, kp), dmul(s, kq));
    E[k][Q] = dadd(dmul(s, kp), dmul(c, kq));
  }
}

// Horn's method: the rotation R maximising sum p~ . R^T q~ for the cross-covariance H = sum p~ q~^T (H[a][b] = S_ab) is the
// unit quaternion (w, x, y, z) of the largest eigenvalue of Horn's symmetric 4x4 matrix N (ties to the lower index).
__device__ void horn_rotation(const double (&H)[3][3], double* __restrict__ R) {
  const double sxx = H[0][0], sxy = H[0][1], sxz = H[0][2], syx = H[1][0], syy = H[1][1], syz = H[1][2], szx = H[2][0],
               szy = H[2][1], szz = H[2][2];
  double A[4][4], E[4][4];
  A[0][0] = dadd(dadd(sxx, syy), szz);
  A[0][1] = dsub(syz, szy);
  A[0][2] = dsub(szx, sxz);
  A[0][3] = dsub(sxy, syx);
  A[1][1] = dsub(dsub(sxx, syy), szz);
  A[1][2] = dadd(sxy, syx);
  A[1][3] = dadd(szx, sxz);
  A[2][2] = dsub(dsub(syy, sxx), szz);
  A[2][3] = dadd(syz, szy);
  A[3][3] = dsub(dsub(szz, sxx), syy);
#pragma unroll
  for (int r = 0; r < 4; ++r) {
#pragma unroll
    for (int c = 0; c < r; ++c) A[r][c] = A[c][r];
#pragma unroll
    for (int c = 0; c < 4; ++c) E[r][c] = r == c ? 1.0 : 0.0;
  }
#pragma unroll 1
  for (int sweep = 0; sweep < HORN_SWEEPS; ++sweep) {
    jacobi_rotate<0, 1>(A, E);
    jacobi_rotate<0, 2>(A, E);
    jacobi_rotate<0, 3>(A, E);
    jacobi_rotate<1, 2>(A, E);
    jacobi_rotate<1, 3>(A, E);
    jacobi_rotate<2, 3>(A, E);
  }
  double best = A[0][0], qw = E[0][0], qx = E[1][0], qy = E[2][0], qz = E[3][0];
#pragma unroll
  for (int k = 1; k < 4; ++k)
    if (A[k][k] > best) {
      best = A[k][k];
      qw = E[0][k];
      qx = E[1][k];
      qy = E[2][k];
      qz = E[3][k];
    }
  const double n = __dsqrt_rn(dadd(dadd(dadd(dmul(qw, qw), dmul(qx, qx)), dmul(qy, qy)), dmul(qz, qz)));
  qw = ddiv(qw, n);
  qx = ddiv(qx, n);
  qy = ddiv(qy, n);
  qz = ddiv(qz, n);
  R[0] = dsub(1.0, dmul(2.0, dadd(dmul(qy, qy), dmul(qz, qz))));
  R[1] = dmul(2.0, dsub(dmul(qx, qy), dmul(qw, qz)));
  R[2] = dmul(2.0, dadd(dmul(qx, qz), dmul(qw, qy)));
  R[3] = dmul(2.0, dadd(dmul(qx, qy), dmul(qw, qz)));
  R[4] = dsub(1.0, dmul(2.0, dadd(dmul(qx, qx), dmul(qz, qz))));
  R[5] = dmul(2.0, dsub(dmul(qy, qz), dmul(qw, qx)));
  R[6] = dmul(2.0, dsub(dmul(qx, qz), dmul(qw, qy)));
  R[7] = dmul(2.0, dadd(dmul(qy, qz), dmul(qw, qx)));
  R[8] = dsub(1.0, dmul(2.0, dadd(dmul(qx, qx), dmul(qy, qy))));
}

// Per-frame squared errors: |v^ - v|^2 per item, summed per 256-item tile (block_sum) and written to
// partials[t * tiles + tile], then, in one block, frame_err[t] = the tiles' partials in tile order and frame_err[T] = the
// frames' sums in frame order.
__global__ void error_sum_kernel(const double* __restrict__ partials, int T, int tiles, double* __restrict__ frame_err) {
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    double a = 0.0;
    for (int s = 0; s < tiles; ++s) a = dadd(a, partials[(int64_t)t * tiles + s]);
    frame_err[t] = a;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    for (int t = 0; t < T; ++t) a = dadd(a, frame_err[t]);
    frame_err[T] = a;
  }
}

// The per-tile error partial of one vertex's squared error d2 (0 past the end), and the running maximum of d2 over the warp
// folded into max_bits by an atomic maximum (d2 >= 0: the order of the bit patterns is the order of the values).
__device__ __forceinline__ void error_tile(double d2, double (*red)[1], double* __restrict__ partial,
                                           unsigned long long* __restrict__ max_bits) {
  double mx = d2;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_down_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) atomicMax(max_bits, (unsigned long long)__double_as_longlong(mx));
  block_sum<1>(&d2, red, partial);
}

inline int tiles_of(int64_t n) { return (int)((n + FP64_THREADS - 1) / FP64_THREADS); }

}  // namespace
}  // namespace amb
