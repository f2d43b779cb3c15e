// Mesh-input path of the TripoSG VAE encoder: farthest-point sampling of the surface points and the posterior sample.
//
// farthest_point_sample replaces pytorch3d's sample_farthest_points(points[..., :3], K, random_start_point=True) as called by
// actionmesh/model/utils/pointcloud_sampling.py:54-62 from TripoSGVAE._sample_features (actionmesh/external/triposg.py:144-149):
// 2048 strictly serial argmax rounds over 8192 points, one CTA per batch element.
//   - The cloud's xyz is staged once in shared memory (SoA, so lane i of a warp reads word i: no bank conflicts); reading
//     the winner's coordinates each round is then a broadcast load.
//   - Each thread owns the points t, t + 1024, t + 2048, ... and keeps their running minimum distance in registers.
//   - One 64-bit key per point and round, (float bits of d) << 32 | (0xFFFFFFFF - index): d >= 0 orders like its bit
//     pattern, so the largest key is the largest d and, among equal d, the lowest index.  A warp max (redux.sync), then one
//     shared-memory step over the 32 warp winners in a double-buffered slot: one __syncthreads per round.
//   d = ((dx*dx) + (dy*dy)) + (dz*dz) with every operation rounded on its own (no FMA contraction), initialised to +inf, so a
//   numpy float32 restatement gives the same indices.
//
// gaussian_sample is DiagonalGaussianDistribution (third_party/TripoSG/triposg/models/autoencoders/vae.py:8-36) on the fp32
// `quant` output read in place: logvar = clamp(params[:, C:2C], -30, 20), std = exp(0.5 logvar), z = mean + std * eps.
#include <cuda_runtime.h>
#include <cstdint>
#include "common.cuh"
#include "../../include/actionmesh_b200.h"

namespace amb {
namespace {

constexpr int kFpsThreads = 1024;
constexpr int kFpsWarps = kFpsThreads / 32;
constexpr int kFpsMaxPoints = 16384;

// Warp max of a 64-bit key as two 32-bit redux.sync: the largest high word, then the largest low word among the lanes
// holding it.  Two instructions on the serial path of every round instead of a chain of ten 32-bit shuffles.
__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
  const unsigned int hi = static_cast<unsigned int>(v >> 32), lo = static_cast<unsigned int>(v);
  const unsigned int mhi = __reduce_max_sync(0xffffffffu, hi);
  const unsigned int mlo = __reduce_max_sync(0xffffffffu, hi == mhi ? lo : 0u);
  return (static_cast<unsigned long long>(mhi) << 32) | mlo;
}

// PPT: points per thread (a power of two with PPT * kFpsThreads >= n).
template <int PPT>
__global__ void __launch_bounds__(kFpsThreads, 1)
    fps_kernel(const float* __restrict__ points, int n, long long ld, long long batch_stride, const int64_t* __restrict__ start,
               int k, int64_t* __restrict__ out) {
  extern __shared__ float smem[];
  float* sx = smem;
  float* sy = sx + n;
  float* sz = sy + n;
  __shared__ unsigned long long red[2][kFpsWarps];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* p = points + (long long)b * batch_stride;
  for (int i = tid; i < n; i += kFpsThreads) {
    sx[i] = p[(long long)i * ld];
    sy[i] = p[(long long)i * ld + 1];
    sz[i] = p[(long long)i * ld + 2];
  }
  float d[PPT];
#pragma unroll
  for (int j = 0; j < PPT; ++j) d[j] = INFINITY;
  long long s = start[b];
  int sel = (int)(s < 0 ? 0 : (s >= n ? n - 1 : s));   // out-of-range starts are the caller's error; never read outside
  int64_t* o = out + (long long)b * k;
  if (tid == 0) o[0] = sel;
  __syncthreads();
  for (int r = 1; r < k; ++r) {
    const float wx = sx[sel], wy = sy[sel], wz = sz[sel];
    unsigned long long best = 0ull;   // below every valid key (index < 0xFFFFFFFF)
#pragma unroll
    for (int j = 0; j < PPT; ++j) {
      const int i = tid + j * kFpsThreads;
      if (i < n) {
        const float dx = __fsub_rn(sx[i], wx), dy = __fsub_rn(sy[i], wy), dz = __fsub_rn(sz[i], wz);
        const float e = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        d[j] = fminf(d[j], e);
        const unsigned long long key =
            (static_cast<unsigned long long>(__float_as_uint(d[j])) << 32) | (0xFFFFFFFFu - static_cast<unsigned int>(i));
        best = key > best ? key : best;
      }
    }
    best = warp_max_u64(best);
    unsigned long long* slot = red[r & 1];
    if (lane == 0) slot[warp] = best;
    __syncthreads();
    best = warp_max_u64(slot[lane]);      // kFpsWarps == 32: one slot per lane
    sel = (int)(0xFFFFFFFFu - static_cast<unsigned int>(best & 0xFFFFFFFFull));
    if (tid == 0) o[r] = sel;
  }
}

template <int PPT>
int launch_fps(const float* points, int batch, int n, long long ld, long long batch_stride, const int64_t* start, int k,
               int64_t* out, cudaStream_t st) {
  const int smem = 3 * n * (int)sizeof(float);
  // the opt-in is remembered per kernel, so it is made once for the largest cloud this instantiation serves
  if (int rc = ensure_smem_optin(fps_kernel<PPT>, 3 * PPT * kFpsThreads * (int)sizeof(float))) return rc;
  fps_kernel<PPT><<<batch, kFpsThreads, smem, st>>>(points, n, ld, batch_stride, start, k, out);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

__global__ void gaussian_sample_kernel(const float* __restrict__ params, long long ld, long long rows, int c,
                                       const float* __restrict__ eps, float* __restrict__ z, float* __restrict__ logvar,
                                       float* __restrict__ std_out) {
  const long long total = rows * c;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / c;
    const int j = (int)(i - r * c);
    const float mean = params[r * ld + j];
    const float lv = fminf(fmaxf(params[r * ld + c + j], -30.0f), 20.0f);
    const float sd = expf(0.5f * lv);
    if (logvar) logvar[i] = lv;
    if (std_out) std_out[i] = sd;
    if (z) z[i] = __fadd_rn(mean, __fmul_rn(sd, eps[i]));
  }
}

}  // namespace
}  // namespace amb

using namespace amb;

extern "C" int amb_farthest_point_sample(const float* points, int batch, int n, int64_t ld, int64_t batch_stride,
                                         const int64_t* start, int k, int64_t* out, amb_stream_t stream) {
  AMB_CHECK_ARG(points && start && out, "farthest_point_sample: null pointer");
  AMB_CHECK_ARG(n > 0 && n <= kFpsMaxPoints, "farthest_point_sample: %d points (1..%d supported)", n, kFpsMaxPoints);
  AMB_CHECK_ARG(ld >= 3 && batch_stride >= (int64_t)(n - 1) * ld + 3,
                "farthest_point_sample: bad strides ld=%lld batch_stride=%lld", (long long)ld, (long long)batch_stride);
  AMB_CHECK_ARG(batch >= 0 && batch <= 65535 && k >= 0, "farthest_point_sample: bad shape batch=%d k=%d", batch, k);
  if (batch == 0 || k == 0) return AMB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int ppt = (n + kFpsThreads - 1) / kFpsThreads;
  if (ppt <= 1) return launch_fps<1>(points, batch, n, ld, batch_stride, start, k, out, st);
  if (ppt <= 2) return launch_fps<2>(points, batch, n, ld, batch_stride, start, k, out, st);
  if (ppt <= 4) return launch_fps<4>(points, batch, n, ld, batch_stride, start, k, out, st);
  if (ppt <= 8) return launch_fps<8>(points, batch, n, ld, batch_stride, start, k, out, st);
  return launch_fps<16>(points, batch, n, ld, batch_stride, start, k, out, st);
}

extern "C" int amb_gaussian_sample(const float* params, int64_t ld, int64_t rows, int channels, const float* eps, float* z,
                                   float* logvar, float* std_out, amb_stream_t stream) {
  AMB_CHECK_ARG(params && (z || logvar || std_out), "gaussian_sample: null pointer");
  AMB_CHECK_ARG(!z || eps, "gaussian_sample: z needs eps");
  AMB_CHECK_ARG(channels > 0 && ld >= 2LL * channels, "gaussian_sample: bad geometry channels=%d ld=%lld", channels, (long long)ld);
  if (rows <= 0) return AMB_OK;
  const long long total = rows * (long long)channels;
  long long blocks = (total + 255) / 256;
  if (blocks > (1LL << 20)) blocks = 1LL << 20;
  gaussian_sample_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(params, ld, rows, channels, eps, z, logvar, std_out);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}
