// Count -> scan -> emit compaction shared by the geometry kernels (octree points, DMC) and the mesh post-processing.
//
// A functor F supplies count(i) (outputs of item i) and emit(i, off) (write them from global offset `off`).  scan_count runs
// the count pass and scans the per-tile totals into `tile_sums` (amb_scan_scratch_ints(n) ints; the last entry receives the
// grand total, in device memory); scan_emit then calls emit for every item in order.  Outputs are therefore in item order
// and two runs give identical arrays.
#pragma once
#include <cuda_runtime.h>
#include "common.cuh"

namespace amb {
namespace {

constexpr int kScanThreads = 256;
constexpr int kScanItems = 8;                          // consecutive items per thread
constexpr int kScanTile = kScanThreads * kScanItems;   // items per block

inline int blocks_for(long long n, int threads) {
  long long b = (n + threads - 1) / threads;
  return (int)(b < 1 ? 1 : (b > (1LL << 20) ? (1LL << 20) : b));
}

// exclusive block-wide prefix sum of one int per thread (kScanThreads threads); returns the block total in *total
__device__ int block_exclusive_scan(int v, int* total) {
  __shared__ int warp_sums[kScanThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = lane < kScanThreads / 32 ? warp_sums[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    if (lane < kScanThreads / 32) warp_sums[lane] = w;
  }
  __syncthreads();
  const int before = (warp > 0 ? warp_sums[warp - 1] : 0) + x - v;
  *total = warp_sums[kScanThreads / 32 - 1];
  __syncthreads();
  return before;
}

// Pass 1: per-tile totals of f.count(i), i in [0, n).
template <class F>
__global__ void __launch_bounds__(kScanThreads) tile_count_kernel(long long n, F f, int* tile_sums) {
  const long long base = (long long)blockIdx.x * kScanTile + (long long)threadIdx.x * kScanItems;
  int s = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k)
    if (base + k < n) s += f.count(base + k);
  int total;
  block_exclusive_scan(s, &total);
  if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}

// Pass 2: exclusive scan of the tile totals in place (one block); tile_sums[n_tiles] receives the grand total.
__global__ void __launch_bounds__(kScanThreads) scan_tiles_kernel(int* tile_sums, int n_tiles) {
  int carry = 0;
  for (int t0 = 0; t0 < n_tiles; t0 += kScanThreads) {
    const int t = t0 + threadIdx.x;
    const int v = t < n_tiles ? tile_sums[t] : 0;
    int total;
    const int ex = block_exclusive_scan(v, &total);
    if (t < n_tiles) tile_sums[t] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) tile_sums[n_tiles] = carry;
}

// Pass 3: every item i emits f.count(i) outputs starting at its global exclusive offset.
template <class F>
__global__ void __launch_bounds__(kScanThreads) tile_emit_kernel(long long n, F f, const int* tile_offsets) {
  const long long base = (long long)blockIdx.x * kScanTile + (long long)threadIdx.x * kScanItems;
  int c[kScanItems];
  int s = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    c[k] = base + k < n ? f.count(base + k) : 0;
    s += c[k];
  }
  int total;
  int off = tile_offsets[blockIdx.x] + block_exclusive_scan(s, &total);
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    if (base + k < n) f.emit(base + k, off);
    off += c[k];
  }
}

inline long long scan_tiles(long long n) { return (n + kScanTile - 1) / kScanTile; }

// count pass + scan: tile_sums must hold scan_tiles(n) + 1 ints; tile_sums[scan_tiles(n)] receives the total (device).
template <class F>
int scan_count(long long n, const F& f, int* tile_sums, cudaStream_t st) {
  const long long nt = scan_tiles(n);
  AMB_CHECK_ARG(nt < (1LL << 31), "geometry: %lld items is too many", n);
  if (nt > 0) tile_count_kernel<F><<<(unsigned)nt, kScanThreads, 0, st>>>(n, f, tile_sums);
  scan_tiles_kernel<<<1, kScanThreads, 0, st>>>(tile_sums, (int)nt);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

template <class F>
int scan_emit(long long n, const F& f, const int* tile_sums, cudaStream_t st) {
  const long long nt = scan_tiles(n);
  if (nt > 0) tile_emit_kernel<F><<<(unsigned)nt, kScanThreads, 0, st>>>(n, f, tile_sums);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

}  // namespace
}  // namespace amb
