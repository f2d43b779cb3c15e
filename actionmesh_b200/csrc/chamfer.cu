// Nearest-neighbour search for the ActionBench Chamfer metrics on the GPU (SURVEY 8(f) rank 4).
//
// Replaces scipy's KDTree.query at actionbench/chamfer.py:44-50 (compute_chamfer_score) and :78-82
// (compute_motion_chamfer_score): for every query point the Euclidean distance to, and the index of, its nearest reference
// point.  Brute force: a query per thread, reference points streamed through shared memory in tiles, the reference set split
// over blockIdx.y so a few thousand queries still fill 132 SMs; partial results meet in one 64-bit atomicMin per query on
// (float bits of d^2 << 32 | index) — valid because d^2 >= 0 orders like its bit pattern, and ties resolve to the lowest
// index.  fp32 FMA work: 10 000 x 100 000 pairs are 8 GFLOP — microseconds on an H100, where the reference's KD-tree build
// + query takes seconds on the host.
#include "common.cuh"
#include "../../include/actionmesh_b200.h"

namespace amb {

constexpr int NN_THREADS = 128;
constexpr int NN_TILE = 1024;

__global__ void nn_init_kernel(unsigned long long* best, int nq) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nq) best[i] = ~0ull;
}

__global__ void __launch_bounds__(NN_THREADS) nn_search_kernel(const float* __restrict__ q, int nq, const float* __restrict__ r,
                                                               int nr, int chunk, unsigned long long* __restrict__ best) {
  __shared__ float sx[NN_TILE], sy[NN_TILE], sz[NN_TILE];
  const int qi = blockIdx.x * NN_THREADS + threadIdx.x;
  const bool live = qi < nq;
  float qx = 0.f, qy = 0.f, qz = 0.f;
  if (live) {
    qx = q[3 * qi];
    qy = q[3 * qi + 1];
    qz = q[3 * qi + 2];
  }
  const int r0 = blockIdx.y * chunk;
  const int r1 = min(nr, r0 + chunk);
  float bd = INFINITY;
  int bi = 0;
  for (int t0 = r0; t0 < r1; t0 += NN_TILE) {
    const int cnt = min(NN_TILE, r1 - t0);
    __syncthreads();
    for (int i = threadIdx.x; i < cnt; i += NN_THREADS) {
      sx[i] = r[3 * (t0 + i)];
      sy[i] = r[3 * (t0 + i) + 1];
      sz[i] = r[3 * (t0 + i) + 2];
    }
    __syncthreads();
    if (live) {
#pragma unroll 4
      for (int i = 0; i < cnt; ++i) {
        const float dx = qx - sx[i], dy = qy - sy[i], dz = qz - sz[i];
        const float d = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
        if (d < bd) {
          bd = d;
          bi = t0 + i;
        }
      }
    }
  }
  if (live && r1 > r0)
    atomicMin(best + qi, (static_cast<unsigned long long>(__float_as_uint(bd)) << 32) | static_cast<unsigned int>(bi));
}

__global__ void nn_finish_kernel(const unsigned long long* __restrict__ best, int nq, float* __restrict__ dist,
                                 int32_t* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nq) {
    const unsigned long long b = best[i];
    if (dist) dist[i] = sqrtf(__uint_as_float(static_cast<unsigned int>(b >> 32)));
    if (idx) idx[i] = static_cast<int32_t>(b & 0xffffffffu);
  }
}

}  // namespace amb

using namespace amb;

extern "C" int amb_nearest_neighbors(const float* query, int n_query, const float* reference, int n_reference,
                                     void* scratch_u64, float* out_dist, int32_t* out_index, amb_stream_t stream) {
  AMB_CHECK_ARG(query && reference && scratch_u64 && (out_dist || out_index), "nearest_neighbors: null pointer");
  AMB_CHECK_ARG(n_reference > 0, "nearest_neighbors: empty reference set");
  if (n_query <= 0) return AMB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned long long* best = reinterpret_cast<unsigned long long*>(scratch_u64);
  const int qblocks = (n_query + NN_THREADS - 1) / NN_THREADS;
  int split = (4 * num_sms() + qblocks - 1) / qblocks;            // >= 4 blocks per SM in flight
  const int max_split = (n_reference + NN_TILE - 1) / NN_TILE;
  if (split > max_split) split = max_split;
  if (split < 1) split = 1;
  int chunk = (n_reference + split - 1) / split;
  chunk = (chunk + NN_TILE - 1) / NN_TILE * NN_TILE;
  split = (n_reference + chunk - 1) / chunk;
  nn_init_kernel<<<(n_query + 255) / 256, 256, 0, s>>>(best, n_query);
  AMB_CHECK_CUDA(cudaGetLastError());
  nn_search_kernel<<<dim3(qblocks, split), NN_THREADS, 0, s>>>(query, n_query, reference, n_reference, chunk, best);
  AMB_CHECK_CUDA(cudaGetLastError());
  nn_finish_kernel<<<(n_query + 255) / 256, 256, 0, s>>>(best, n_query, out_dist, out_index);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}
