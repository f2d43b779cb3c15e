// wgmma GEMM for sm_90a:  C = epilogue(A · Wᵀ),  A:(M,K) bf16, W:(N,K) bf16 (nn.Linear layout), fp32 accumulate in registers.
//
// Persistent, warp-specialized kernel on 2-CTA clusters.  Output tiles are 128 x BN (BN = 256, 128, or 64 when N is not a
// multiple of 128).  The two CTAs of a cluster run tiles (m, n) and (m + 1, n) of one unit of the schedule together;
// every CTA of a cluster runs the units cluster, cluster + clusters, ... in turn.  Three warpgroups per CTA:
//   warpgroup 0     TMA producer   (one elected lane; cp.async.bulk.tensor 2D, 128B swizzle, STAGES-deep mbarrier ring).
//                                  It loads its own A box and half of the W box, multicast into both CTAs of the pair, and
//                                  runs ahead across tile boundaries so the ring never drains between tiles.
//   warpgroups 1-2  consumers, in one of two organisations:
//     BN = 128, 64  ping-pong: they take alternate tiles, each a whole 128 x BN tile = two wgmma m64nBNk16 per k16 step,
//                   one k-block of MMAs in flight while the previous stage is released.  Named barriers hand the tensor
//                   cores from one to the other after its last k-block, so one warpgroup's epilogue — bias / GELU /
//                   LayerScale / residual / per-head RMSNorm + RoPE straight from the accumulator fragment — runs under
//                   the other's MMAs.
//     BN = 256      cooperative: both run every tile, warpgroup 1 rows [0, 64) and warpgroup 2 rows [64, 128), one wgmma
//                   m64n256k16 per k16 step.  Each W element is read from shared memory once per k16 step instead of
//                   twice: a fifth fewer shared-memory bytes (TMA writes + wgmma reads) per FLOP.  Nothing computes
//                   during the epilogue, so amb_gemm_bf16 takes this organisation only for long K.
// Units are rastered in bands of GROUP_M M-tile pairs: a band sweeps every N-tile before the next band starts, so its A
// rows stay L2-resident while W panels stream past.
#include <atomic>
#include <cstdlib>
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/actionmesh_b200.h"

namespace amb {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle-128B row
constexpr int GEMM_THREADS = 384;
constexpr int CLUSTER = 2;  // CTAs per cluster: M-tiles (m, m + 1) sharing each W box
constexpr int GROUP_M = 8;    // M-tile pairs per raster band
constexpr int EPI_BATCH = 4;  // column groups of residual loads in flight together (8 spills at 128 accumulator registers)

struct GemmParams {
  int M, N, K;
  int k_split_blocks;  // k-blocks >= this come from the second A source (INT_MAX: single source)
  void* C;
  long long ldc;
  int c_fp32;
  const float* bias;
  const void* residual;
  long long ldr;
  int res_fp32;
  int act;
  const float* col_scale;
  int grp_rows, grp_stride, row_off;
  int norm_cols, norm_seg;
  const float* norm_w0;
  const float* norm_w1;
  float norm_eps;
  int rope_cols;
  const float* rope_cos;
  const float* rope_sin;
  int rope_rows_per_pos;
  void* C2;        // optional bf16 copy of the output
  long long ldc2;
};

// Exact (erf) GELU, x·Φ(x), as the reference's FeedForward uses (diffusers GELU, approximate="none").  Φ(-|x|) =
// ½·erfc(|x|/√2) through Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7): one MUFU.RCP, one MUFU.EX2 and six FMAs instead of
// libdevice erff's two divergent branches (~28 instructions); the absolute error of the result (4.2e-7 over |x| <= 12) is
// that of the fp32 erf formula itself (4.5e-7).
__device__ __forceinline__ float gelu_erf(float x) {
  const float ax = fabsf(x);
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f * 0.70710678118654752440f, ax, 1.0f)));
  float p = fmaf(t, 1.061405429f, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = ex2_approx(ax * ax * (-0.5f * 1.4426950408889634f));
  const float q = 0.5f * (p * t) * e;  // Φ(-|x|)
  return x * (x >= 0.0f ? 1.0f - q : q);
}

template <int BN>
struct GemmSmem {
  static constexpr int STAGES = BN == 256 ? 4 : BN == 128 ? 6 : 8;  // 192 KB of operand ring in every case
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int TOTAL = BAR_OFFSET + 2 * STAGES * 8 + 1024;  // + alignment slack
};

// Four column groups of one row leave the accumulator fragment as pairs: thread q of a quad holds v[j] = columns
// 8 (i0 + j) + 2q + {0, 1} of groups j = 0..3.  A 4 x 4 transpose inside the quad (four shuffles per word, selects only,
// no local memory) leaves thread q with the 8 consecutive columns of group i0 + q, in order, so each row goes out in
// 16-byte stores: a quarter of the store instructions, and every 32-byte sector written whole by one of them.
__device__ __forceinline__ void quad_transpose(uint32_t (&x)[4], int q) {
  const bool hi = q & 2, odd = q & 1;
#pragma unroll
  for (int k = 0; k < 2; ++k) {  // swap with thread q ^ 2 the groups whose bit 1 differs from q's
    const uint32_t got = __shfl_xor_sync(0xffffffffu, hi ? x[k] : x[2 + k], 2);
    if (hi) x[k] = got; else x[2 + k] = got;
  }
#pragma unroll
  for (int m = 0; m < 2; ++m) {  // then with thread q ^ 1 the groups whose bit 0 differs
    const uint32_t got = __shfl_xor_sync(0xffffffffu, odd ? x[2 * m] : x[2 * m + 1], 1);
    if (odd) x[2 * m] = got; else x[2 * m + 1] = got;
  }
}
// v[j] as above -> w[0..7] = columns 8 (i0 + q) + 0..7 of the row
__device__ __forceinline__ void pairs_to_row8(const float2 (&v)[4], int q, float (&w)[8]) {
  uint32_t lo[4], hi[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) { lo[j] = __float_as_uint(v[j].x); hi[j] = __float_as_uint(v[j].y); }
  quad_transpose(lo, q);
  quad_transpose(hi, q);
#pragma unroll
  for (int s = 0; s < 4; ++s) { w[2 * s] = __uint_as_float(lo[s]); w[2 * s + 1] = __uint_as_float(hi[s]); }
}
// 8 consecutive columns of one row, 16-byte aligned (checked at launch)
__device__ __forceinline__ void store8(void* C, int c_fp32, long long off, const float (&w)[8]) {
  if (c_fp32) {
    float4* d = reinterpret_cast<float4*>(reinterpret_cast<float*>(C) + off);
    d[0] = make_float4(w[0], w[1], w[2], w[3]);
    d[1] = make_float4(w[4], w[5], w[6], w[7]);
  } else {
    *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(C) + off) =
        make_uint4(pack_bf16(w[0], w[1]), pack_bf16(w[2], w[3]), pack_bf16(w[4], w[5]), pack_bf16(w[6], w[7]));
  }
}
__device__ __forceinline__ void load8(const void* R, int r_fp32, long long off, float (&w)[8]) {
  if (r_fp32) {
    const float4* s = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(R) + off);
    const float4 a = s[0], b = s[1];
    w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
  } else {
    const uint4 u = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(R) + off);
    const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16(uu[j]);
      w[2 * j] = f.x; w[2 * j + 1] = f.y;
    }
  }
}

// bias -> activation -> column scale of one column pair; the residual is added after the quad transpose (epilogue_tile)
__device__ __forceinline__ float2 finish_pair(const GemmParams& p, float v0, float v1, int col) {
  if (p.bias) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
    v0 += b.x; v1 += b.y;
  }
  if (p.act == 1) {
    v0 = gelu_erf(v0);
    v1 = gelu_erf(v1);
  } else if (p.act == 2) {  // ReLU (RMBG's REBNCONV, csrc/rmbg.cu)
    v0 = fmaxf(v0, 0.f);
    v1 = fmaxf(v1, 0.f);
  }
  if (p.col_scale) {
    const float2 s = __ldg(reinterpret_cast<const float2*>(p.col_scale + col));
    v0 *= s.x; v1 *= s.y;
  }
  return make_float2(v0, v1);
}

template <int BN>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, const float* acc, int n0, int r0) {
  const int q = threadIdx.x & 3;
  long long drow[2];
  bool valid[2];
  int row[2] = {r0, r0 + 8};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    valid[h] = row[h] < p.M;
    drow[h] = row[h];
    if (p.grp_rows > 0) drow[h] = (long long)(row[h] / p.grp_rows) * p.grp_stride + (row[h] % p.grp_rows) + p.row_off;
  }
  if constexpr (BN == 128) {
    const bool do_norm = n0 < p.norm_cols, do_rope = n0 < p.rope_cols;
    if (do_norm || do_rope) {
      // ---- per-head RMSNorm and/or RoPE (the launch checks exclude residual / activation / col_scale / c2 here)
      float rs[2] = {1.0f, 1.0f};
      const float* nwp = (n0 < p.norm_seg) ? p.norm_w0 : p.norm_w1;
      if (do_norm) {
        float ss0 = 0.f, ss1 = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          ss0 += acc[4 * i] * acc[4 * i] + acc[4 * i + 1] * acc[4 * i + 1];
          ss1 += acc[4 * i + 2] * acc[4 * i + 2] + acc[4 * i + 3] * acc[4 * i + 3];
        }
        ss0 += __shfl_xor_sync(0xffffffffu, ss0, 1);
        ss1 += __shfl_xor_sync(0xffffffffu, ss1, 1);
        ss0 += __shfl_xor_sync(0xffffffffu, ss0, 2);
        ss1 += __shfl_xor_sync(0xffffffffu, ss1, 2);
        rs[0] = rsqrtf(ss0 * (1.0f / 128.0f) + p.norm_eps);
        rs[1] = rsqrtf(ss1 * (1.0f / 128.0f) + p.norm_eps);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float rc[16], rsn[16];  // RoPE cos / sin of my 16 pairs at this row's position
        if (do_rope) {
          const int pos = (valid[h] ? row[h] : 0) / p.rope_rows_per_pos;
          const float* cs = p.rope_cos + (long long)pos * 64;
          const float* sn = p.rope_sin + (long long)pos * 64;
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            rc[i] = __ldg(cs + 4 * i + q);  // angle index lc / 2 of column lc = 8i + 2q
            rsn[i] = __ldg(sn + 4 * i + q);
          }
        }
#pragma unroll
        for (int i0 = 0; i0 < 16; i0 += 4) {
          float2 v[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int i = i0 + j;
            float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
            if (do_norm) {
              const float2 nw = __ldg(reinterpret_cast<const float2*>(nwp + 8 * i + 2 * q));
              v0 *= rs[h] * nw.x;
              v1 *= rs[h] * nw.y;
            }
            if (do_rope) {  // interleaved pair (lc, lc + 1), lc = 8i + 2q, rotates by angle lc / 2 of the row's position
              const float c = rc[i], s = rsn[i];
              const float x = v0, y = v1;
              v0 = x * c - y * s;
              v1 = y * c + x * s;
            }
            v[j] = make_float2(v0, v1);
          }
          float w[8];
          pairs_to_row8(v, q, w);
          if (valid[h]) store8(p.C, p.c_fp32, drow[h] * p.ldc + n0 + 8 * (i0 + q), w);
        }
      }
      return;
    }
  }
  // The residual may alias C, so a residual load placed after a store cannot move above it: loaded group by group, every
  // load of the tile would wait out a full HBM latency behind the previous group's stores.  Instead the residuals of
  // EPI_BATCH column groups (after the transpose: this thread's group of the batch, both rows) are loaded together,
  // before any of their stores.
  static_assert(EPI_BATCH == 4, "one column group per thread of the quad");
#pragma unroll
  for (int i0 = 0; i0 < BN / 8; i0 += EPI_BATCH) {
    const int col = n0 + 8 * (i0 + q);  // this thread's 8 columns after the transpose
    float r[2][8];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (p.residual && valid[h]) load8(p.residual, p.res_fp32, drow[h] * p.ldr + col, r[h]);
      else
#pragma unroll
        for (int c = 0; c < 8; ++c) r[h][c] = 0.f;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float2 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float* a = acc + 4 * (i0 + j) + 2 * h;
        v[j] = finish_pair(p, a[0], a[1], n0 + 8 * (i0 + j) + 2 * q);
      }
      float w[8];
      pairs_to_row8(v, q, w);
      if (!valid[h]) continue;
      if (p.residual)
#pragma unroll
        for (int c = 0; c < 8; ++c) w[c] += r[h][c];
      store8(p.C, p.c_fp32, drow[h] * p.ldc + col, w);
      if (p.C2) store8(p.C2, 0, drow[h] * p.ldc2 + col, w);
    }
  }
}

template <int BN>
__device__ __forceinline__ void wgmma_tile_k16(float* acc, uint64_t adesc, uint64_t bdesc) {
  if constexpr (BN == 256) wgmma_ss_n256(acc, adesc, bdesc, 1u);
  else if constexpr (BN == 128) wgmma_ss_n128(acc, adesc, bdesc, 1u);
  else wgmma_ss_n64(acc, adesc, bdesc, 1u);
}

// First row m0 and N-tile index nt of schedule unit u for cluster CTA `rank`: bands of GROUP_M M-tile pairs, the M pair
// fastest inside a band.
__device__ __forceinline__ void unit_tile(int u, int num_mp, int num_n, uint32_t rank, int& m0, int& nt) {
  const int band = u / (GROUP_M * num_n);
  const int first = band * GROUP_M;
  const int rows = min(GROUP_M, num_mp - first);
  const int r = u - band * GROUP_M * num_n;
  m0 = ((first + r % rows) * CLUSTER + (int)rank) * BM;
  nt = r / rows;
}

template <int BN>
__global__ void __cluster_dims__(CLUSTER, 1, 1) __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
                 const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  using L = GemmSmem<BN>;
  constexpr int STAGES = L::STAGES;
  constexpr int B_HALF = L::B_BYTES / CLUSTER;  // the W rows one CTA loads for the pair: a whole number of 1024-B swizzle atoms
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);  // warp-uniform role
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = cluster_ctarank();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmA2);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      // one arrival per consumer warp of both CTAs that read the stage (each wrote a W half here): one warpgroup per CTA
      // in ping-pong, both in the cooperative organisation
      mbar_init(&empty_bar[s], (BN == 256 ? 8 : 4) * CLUSTER);
    }
    fence_mbar_init();
  }
  cluster_sync();  // both CTAs' barriers exist before any multicast copy or remote arrival reaches them

  const int num_n = p.N / BN;
  const int num_mp = (p.M + CLUSTER * BM - 1) / (CLUSTER * BM);  // M-tile pairs; the odd last tile's peer has no valid row
  const int num_units = num_mp * num_n;
  const int cluster = blockIdx.x / CLUSTER, num_clusters = gridDim.x / CLUSTER;
  const int num_kb = p.K / BK;

  if (wg == 0) {
    // ===================== TMA producer =====================
    reg_dealloc<40>();
    if (warp == 0) {
      int s = 0;
      uint32_t phase = 0;
      for (int u = cluster; u < num_units; u += num_clusters) {
        int m0, nt;
        unit_tile(u, num_mp, num_n, rank, m0, nt);
        const int n0 = nt * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[s], phase ^ 1);  // released by the consumers of both CTAs
          if (elect_one()) {
            mbar_expect_tx(&full_bar[s], L::STAGE_BYTES);
            uint8_t* sa = smem + s * L::STAGE_BYTES;
            uint8_t* sb = sa + L::A_BYTES;
            if (kb < p.k_split_blocks) tma_load_2d(sa, &tmA, &full_bar[s], kb * BK, m0, kEvictNormal);
            else tma_load_2d(sa, &tmA2, &full_bar[s], (kb - p.k_split_blocks) * BK, m0, kEvictNormal);
            tma_load_2d_multicast(sb + rank * B_HALF, &tmB, &full_bar[s], kb * BK, n0 + (int)rank * (BN / CLUSTER),
                                  (uint16_t)((1u << CLUSTER) - 1), kEvictLast);
          }
          __syncwarp();
          if (++s == STAGES) { s = 0; phase ^= 1; }
        }
      }
      // Watchdog: the consumers wait without a timeout (see mbar_wait_watched), so this warp waits, bounded, until they
      // have released the last STAGES stages.  A stalled consumer makes that wait trap and the launch fail.
      for (int j = 0; j < STAGES; ++j) {
        mbar_wait(&empty_bar[s], phase ^ 1);
        if (++s == STAGES) { s = 0; phase ^= 1; }
      }
    }
  } else if constexpr (BN == 256) {
    // ===================== consumers, cooperative: warpgroup 1 rows [0, 64), warpgroup 2 rows [64, 128) of every tile =====
    reg_alloc<232>();
    const uint32_t a_row_off = (wg - 1) * 64 * 128;  // 64 rows of 128 B (a multiple of the 1024-B swizzle atom)
    const int n_local = (num_units - cluster + num_clusters - 1) / num_clusters;
    for (int i = 0; i < n_local; ++i) {
      int m0, nt;
      unit_tile(cluster + i * num_clusters, num_mp, num_n, rank, m0, nt);
      const int n0 = nt * BN;
      float acc[BN / 2];
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
      // the producer filled the ring in tile order: this tile's first k-block is ring slot i * num_kb
      const long long g0 = (long long)i * num_kb;
      int s = (int)(g0 % STAGES), s_prev = s;
      uint32_t phase = (uint32_t)((g0 / STAGES) & 1);
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait_watched(&full_bar[s], phase);
        const uint32_t a_addr = smem_u32(smem + s * L::STAGE_BYTES);
        const uint64_t adesc = make_desc_kmajor_sw128(a_addr + a_row_off);
        const uint64_t bdesc = make_desc_kmajor_sw128(a_addr + L::A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) wgmma_tile_k16<BN>(acc, adesc + 2 * k, bdesc + 2 * k);
        wgmma_commit();
        wgmma_wait<1>();  // the MMAs of the previous k-block are complete: its stage can be refilled
        if (kb > 0) {
          __syncwarp();
          if (lane < CLUSTER) mbar_arrive_cluster(&empty_bar[s_prev], lane);  // lane c releases the stage in CTA c
        }
        s_prev = s;
        if (++s == STAGES) { s = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) reg_fence(acc[j]);
      __syncwarp();
      if (lane < CLUSTER) mbar_arrive_cluster(&empty_bar[s_prev], lane);
      if (m0 < p.M) {
        // The m64n256 fragment is two 128-column heads in the m64n128 layout.  The thread index is read here rather than
        // kept from before the mainloop: a row offset held across it is one register too many and spills.
        uint32_t t;
        asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
        const int r0 = m0 + (int)((t - 128) >> 5) * 16 + (int)((t & 31) >> 2);  // (wg - 1) * 64 + (warp & 3) * 16 + lane / 4
        epilogue_tile<128>(p, acc, n0, r0);
        epilogue_tile<128>(p, acc + 64, n0 + 128, r0);
      }
    }
  } else {
    // ===================== consumers: warpgroup 1 takes this CTA's even tiles, warpgroup 2 its odd ones =====================
    reg_alloc<232>();
    // Issue turns: a warpgroup waits on named barrier `wg` before its mainloop and lets the other one go after issuing its
    // last k-block.  The first tile goes without waiting and the last gives no go-ahead, so every arrival meets a wait.
    const uint32_t my_turn = wg, other_turn = 3 - wg;
    const int n_local = (num_units - cluster + num_clusters - 1) / num_clusters;
    for (int i = wg - 1; i < n_local; i += 2) {
      int m0, nt;
      unit_tile(cluster + i * num_clusters, num_mp, num_n, rank, m0, nt);
      const int n0 = nt * BN;
      float acc[2][BN / 2];  // rows [0, 64) and [64, 128) of the tile
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) acc[h][j] = 0.f;
      // the producer filled the ring in tile order: this tile's first k-block is ring slot i * num_kb
      const long long g0 = (long long)i * num_kb;
      int s = (int)(g0 % STAGES), s_prev = s;
      uint32_t phase = (uint32_t)((g0 / STAGES) & 1);
      if (i > 0) named_bar_sync(my_turn, 256);
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait_watched(&full_bar[s], phase);
        const uint32_t a_addr = smem_u32(smem + s * L::STAGE_BYTES);
        const uint64_t adesc0 = make_desc_kmajor_sw128(a_addr);
        const uint64_t adesc1 = make_desc_kmajor_sw128(a_addr + 64 * 128);  // 64 rows of 128 B
        const uint64_t bdesc = make_desc_kmajor_sw128(a_addr + L::A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          wgmma_tile_k16<BN>(acc[0], adesc0 + 2 * k, bdesc + 2 * k);
          wgmma_tile_k16<BN>(acc[1], adesc1 + 2 * k, bdesc + 2 * k);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the MMAs of the previous k-block are complete: its stage can be refilled
        if (kb > 0) {
          __syncwarp();
          if (lane < CLUSTER) mbar_arrive_cluster(&empty_bar[s_prev], lane);  // lane c releases the stage in CTA c
        }
        s_prev = s;
        if (++s == STAGES) { s = 0; phase ^= 1; }
      }
      if (i + 1 < n_local) named_bar_arrive(other_turn, 256);
      wgmma_wait<0>();
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) reg_fence(acc[h][j]);
      __syncwarp();
      if (lane < CLUSTER) mbar_arrive_cluster(&empty_bar[s_prev], lane);
      if (m0 < p.M) {
        const int r0 = m0 + (warp & 3) * 16 + (lane >> 2);
        epilogue_tile<BN>(p, acc[0], n0, r0);
        epilogue_tile<BN>(p, acc[1], n0, r0 + 64);
      }
    }
  }
  __syncwarp();
  cluster_sync();  // no CTA leaves while its peer can still write into its shared memory or arrive on its barriers
}

static GemmParams make_params(const amb_gemm_args* a) {
  GemmParams p;
  p.M = a->m; p.N = a->n; p.K = a->k;
  p.k_split_blocks = a->a2 ? a->k_split / BK : 0x7fffffff;
  p.C = a->c; p.ldc = a->ldc; p.c_fp32 = a->c_fp32;
  p.bias = a->bias;
  p.residual = a->residual; p.ldr = a->ldr; p.res_fp32 = a->res_fp32;
  p.act = a->act;
  p.col_scale = a->col_scale;
  p.grp_rows = a->grp_rows; p.grp_stride = a->grp_stride; p.row_off = a->row_off;
  p.norm_cols = a->norm_cols; p.norm_seg = a->norm_seg;
  p.norm_w0 = a->norm_w0; p.norm_w1 = a->norm_w1 ? a->norm_w1 : a->norm_w0;
  p.norm_eps = a->norm_eps;
  p.rope_cols = a->rope_cols; p.rope_cos = a->rope_cos; p.rope_sin = a->rope_sin;
  p.rope_rows_per_pos = a->rope_rows_per_pos > 0 ? a->rope_rows_per_pos : 1;
  p.C2 = a->c2; p.ldc2 = a->ldc2;
  return p;
}

// Clusters of gemm_bf16_kernel<BN> that fit on the current device at once, queried once per device: the persistent grid
// never launches more, so no cluster waits for a second wave.
template <int BN>
static int max_active_clusters(int* out) {
  static std::atomic<int> cached[16];
  int dev = 0;
  AMB_CHECK_CUDA(cudaGetDevice(&dev));
  if (dev < 16 && cached[dev].load() > 0) {
    *out = cached[dev].load();
    return AMB_OK;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(CLUSTER * num_sms(), 1, 1);
  cfg.blockDim = dim3(GEMM_THREADS, 1, 1);
  cfg.dynamicSmemBytes = GemmSmem<BN>::TOTAL;
  int n = 0;
  AMB_CHECK_CUDA(cudaOccupancyMaxActiveClusters(&n, gemm_bf16_kernel<BN>, &cfg));
  AMB_CHECK_ARG(n > 0, "gemm: no %d-CTA cluster of %d B shared memory fits on device %d", CLUSTER, GemmSmem<BN>::TOTAL, dev);
  if (dev < 16) cached[dev].store(n);
  *out = n;
  return AMB_OK;
}

template <int BN>
static int launch_gemm(const amb_gemm_args* a, cudaStream_t stream) {
  using L = GemmSmem<BN>;
  CUtensorMap tmA, tmA2, tmB;
  const int k1 = (a->a2 != nullptr) ? a->k_split : a->k;
  {
    uint64_t dims[2] = {(uint64_t)k1, (uint64_t)a->m};
    uint64_t str[1] = {(uint64_t)a->lda * 2};
    uint32_t box[2] = {BK, BM};
    int r = encode_tmap_bf16(&tmA, a->a, 2, dims, str, box);
    if (r) return r;
  }
  if (a->a2) {
    uint64_t dims[2] = {(uint64_t)(a->k - a->k_split), (uint64_t)a->m};
    uint64_t str[1] = {(uint64_t)a->lda2 * 2};
    uint32_t box[2] = {BK, BM};
    int r = encode_tmap_bf16(&tmA2, a->a2, 2, dims, str, box);
    if (r) return r;
  } else {
    tmA2 = tmA;
  }
  {
    uint64_t dims[2] = {(uint64_t)a->k, (uint64_t)a->n};
    uint64_t str[1] = {(uint64_t)a->ldw * 2};
    uint32_t box[2] = {BK, BN / CLUSTER};  // each CTA of a pair loads half of the W tile
    int r = encode_tmap_bf16(&tmB, a->w, 2, dims, str, box);
    if (r) return r;
  }
  GemmParams p = make_params(a);
  auto kern = gemm_bf16_kernel<BN>;
  {
    int r = ensure_smem_optin(kern, L::TOTAL);
    if (r) return r;
  }
  int clusters = 0;
  {
    int r = max_active_clusters<BN>(&clusters);
    if (r) return r;
  }
  const long long num_mp = ((long long)a->m + CLUSTER * BM - 1) / (CLUSTER * BM);
  const long long num_units = (long long)(a->n / BN) * num_mp;
  AMB_CHECK_ARG(num_units < 0x7fffffffLL, "gemm: too many tiles (m=%d n=%d)", a->m, a->n);
  const unsigned grid = (unsigned)(CLUSTER * (num_units < clusters ? num_units : clusters));
  kern<<<grid, GEMM_THREADS, L::TOTAL, stream>>>(tmA, tmA2, tmB, p);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

}  // namespace amb

using namespace amb;

extern "C" int amb_gemm_bf16(const amb_gemm_args* a, amb_stream_t stream) {
  AMB_CHECK_ARG(a && a->a && a->w && a->c, "gemm: null pointer");
  AMB_CHECK_ARG(a->m > 0 && a->n > 0 && a->k > 0, "gemm: bad shape m=%d n=%d k=%d", a->m, a->n, a->k);
  AMB_CHECK_ARG(a->k % BK == 0, "gemm: k=%d must be a multiple of %d", a->k, BK);
  AMB_CHECK_ARG(a->n % 64 == 0, "gemm: n=%d must be a multiple of 64", a->n);
  AMB_CHECK_ARG(a->lda % 8 == 0 && a->ldw % 8 == 0 && a->ldc % 8 == 0, "gemm: lda/ldw/ldc must be multiples of 8 elements");
  AMB_CHECK_ARG(!a->a2 || (a->k_split > 0 && a->k_split < a->k && a->k_split % BK == 0 && a->lda2 % 8 == 0),
                "gemm: bad k_split %d", a->k_split);
  AMB_CHECK_ARG(!a->residual || a->ldr % 8 == 0, "gemm: ldr must be a multiple of 8");
  AMB_CHECK_ARG(a->act >= 0 && a->act <= 2, "gemm: unknown activation %d", a->act);
  AMB_CHECK_ARG(!a->c2 || a->ldc2 % 8 == 0, "gemm: ldc2 must be a multiple of 8");
  // the epilogue writes (and reads the residual in) 8-column, 16-byte vectors
  AMB_CHECK_ARG((uintptr_t)a->c % 16 == 0 && (uintptr_t)a->c2 % 16 == 0 && (uintptr_t)a->residual % 16 == 0,
                "gemm: c, c2 and residual must be 16-byte aligned");
  if (a->norm_cols > 0 || a->rope_cols > 0) {
    AMB_CHECK_ARG(a->n % 128 == 0 && a->norm_cols % 128 == 0 && a->rope_cols % 128 == 0,
                  "gemm: head epilogue needs n, norm_cols, rope_cols multiples of 128");
    AMB_CHECK_ARG(a->norm_cols == 0 || (a->norm_w0 && a->norm_seg % 128 == 0), "gemm: norm weights / norm_seg (multiple of 128) required");
    AMB_CHECK_ARG(a->rope_cols == 0 || (a->rope_cos && a->rope_sin), "gemm: rope tables required");
    AMB_CHECK_ARG(!a->residual && a->act == 0 && !a->col_scale && !a->c2, "gemm: head epilogue excludes residual/activation/col_scale/c2");
  }
  cudaStream_t s = (cudaStream_t)stream;
  // Cooperative 128 x 256 tiles where the mainloop is long enough to pay for the exposed epilogue.  Measured on the DiT's
  // block GEMMs (DESIGN 4.2): ff2 (K = 8192) and the skip linear (K = 4096) are 13-14 % faster than ping-pong; every
  // K = 2048 shape (QKV, ff1, x.q, and the o-projections) is 2-8 % slower.
  if (a->n % 256 == 0 && a->k > 2048) return launch_gemm<256>(a, s);
  if (a->n % 128 == 0) return launch_gemm<128>(a, s);
  return launch_gemm<64>(a, s);
}
