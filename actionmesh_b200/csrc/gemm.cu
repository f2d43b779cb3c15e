// wgmma GEMM for sm_90a:  C = epilogue(A · Wᵀ),  A:(M,K) bf16, W:(N,K) bf16 (nn.Linear layout), fp32 accumulate in registers.
//
// One CTA computes one 128 x BN output tile; three warpgroups:
//   warpgroup 0     TMA producer   (one elected lane; cp.async.bulk.tensor 2D, 128B swizzle, STAGES-deep mbarrier ring)
//   warpgroups 1-2  consumers      (each owns 64 of the 128 rows: wgmma m64nBNk16 from shared memory, one k-block of MMAs
//                                   in flight while the previous stage is released; then the epilogue straight from the
//                                   accumulator fragment: bias / GELU / LayerScale / residual / per-head RMSNorm + RoPE)
// Tiles are numbered n-fastest so the CTAs of one wave share A rows through L2 and W stays L2-resident.
#include <cstdlib>
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/actionmesh_b200.h"

namespace amb {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle-128B row
constexpr int GEMM_THREADS = 384;

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

// two consecutive output columns of one row (values already final)
__device__ __forceinline__ void store2(void* C, int c_fp32, long long off, float v0, float v1) {
  if (c_fp32) *reinterpret_cast<float2*>(reinterpret_cast<float*>(C) + off) = make_float2(v0, v1);
  else *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(C) + off) = pack_bf16(v0, v1);
}
__device__ __forceinline__ float2 load2(const void* R, int r_fp32, long long off) {
  if (r_fp32) return *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(R) + off);
  return unpack_bf16(*reinterpret_cast<const uint32_t*>(reinterpret_cast<const __nv_bfloat16*>(R) + off));
}

// bias -> activation -> column scale -> residual -> store for one (row, column pair)
__device__ __forceinline__ void finish_pair(const GemmParams& p, float v0, float v1, long long drow, int col, bool valid) {
  if (p.bias) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
    v0 += b.x; v1 += b.y;
  }
  if (p.act == 1) {
    v0 = gelu_erf(v0);
    v1 = gelu_erf(v1);
  }
  if (p.col_scale) {
    const float2 s = __ldg(reinterpret_cast<const float2*>(p.col_scale + col));
    v0 *= s.x; v1 *= s.y;
  }
  if (!valid) return;
  if (p.residual) {
    const float2 r = load2(p.residual, p.res_fp32, drow * p.ldr + col);
    v0 += r.x; v1 += r.y;
  }
  store2(p.C, p.c_fp32, drow * p.ldc + col, v0, v1);
  if (p.C2) store2(p.C2, 0, drow * p.ldc2 + col, v0, v1);
}

// Epilogue of one warpgroup's 64 x BN accumulator (fragment layout in ptx.cuh): thread holds rows r0 and r0 + 8, columns
// 8i + 2q + {0,1}.  One head = 128 columns = 16 fragment groups; its row statistics are reduced over the 4 threads of a quad.
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
  const int head_cols = p.norm_cols > p.rope_cols ? p.norm_cols : p.rope_cols;
  if constexpr (BN % 128 == 0) {
    if (n0 < head_cols) {
      // ---- per-head RMSNorm and/or RoPE (the launch checks exclude residual / activation / col_scale / c2 here)
#pragma unroll
      for (int hd = 0; hd < BN / 128; ++hd) {
        const int col0 = n0 + hd * 128;
        const bool do_norm = col0 < p.norm_cols, do_rope = col0 < p.rope_cols;
        const float* a = acc + hd * 64;
        if (!do_norm && !do_rope) {
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int col = col0 + 8 * i + 2 * q;
            finish_pair(p, a[4 * i], a[4 * i + 1], drow[0], col, valid[0]);
            finish_pair(p, a[4 * i + 2], a[4 * i + 3], drow[1], col, valid[1]);
          }
          continue;
        }
        float rs[2] = {1.0f, 1.0f};
        if (do_norm) {
          float ss0 = 0.f, ss1 = 0.f;
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            ss0 += a[4 * i] * a[4 * i] + a[4 * i + 1] * a[4 * i + 1];
            ss1 += a[4 * i + 2] * a[4 * i + 2] + a[4 * i + 3] * a[4 * i + 3];
          }
          ss0 += __shfl_xor_sync(0xffffffffu, ss0, 1);
          ss1 += __shfl_xor_sync(0xffffffffu, ss1, 1);
          ss0 += __shfl_xor_sync(0xffffffffu, ss0, 2);
          ss1 += __shfl_xor_sync(0xffffffffu, ss1, 2);
          rs[0] = rsqrtf(ss0 * (1.0f / 128.0f) + p.norm_eps);
          rs[1] = rsqrtf(ss1 * (1.0f / 128.0f) + p.norm_eps);
        }
        const float* w = (col0 < p.norm_seg) ? p.norm_w0 : p.norm_w1;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int pos = (valid[h] ? row[h] : 0) / p.rope_rows_per_pos;
          const float* cs = p.rope_cos + (long long)pos * 64;
          const float* sn = p.rope_sin + (long long)pos * 64;
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int lc = 8 * i + 2 * q;  // column inside the head
            float v0 = a[4 * i + 2 * h], v1 = a[4 * i + 2 * h + 1];
            if (do_norm) {
              const float2 ww = __ldg(reinterpret_cast<const float2*>(w + lc));
              v0 *= rs[h] * ww.x;
              v1 *= rs[h] * ww.y;
            }
            if (do_rope) {  // interleaved pair (lc, lc + 1) rotates by angle lc / 2 of the row's position
              const float c = __ldg(cs + (lc >> 1)), s = __ldg(sn + (lc >> 1));
              const float x = v0, y = v1;
              v0 = x * c - y * s;
              v1 = y * c + x * s;
            }
            if (valid[h]) store2(p.C, p.c_fp32, drow[h] * p.ldc + col0 + lc, v0, v1);
          }
        }
      }
      return;
    }
  }
#pragma unroll
  for (int i = 0; i < BN / 8; ++i) {
    const int col = n0 + 8 * i + 2 * q;
    finish_pair(p, acc[4 * i], acc[4 * i + 1], drow[0], col, valid[0]);
    finish_pair(p, acc[4 * i + 2], acc[4 * i + 3], drow[1], col, valid[1]);
  }
}

template <int BN>
__device__ __forceinline__ void wgmma_tile_k16(float* acc, uint64_t adesc, uint64_t bdesc) {
  if constexpr (BN == 256) wgmma_ss_n256(acc, adesc, bdesc, 1u);
  else if constexpr (BN == 128) wgmma_ss_n128(acc, adesc, bdesc, 1u);
  else wgmma_ss_n64(acc, adesc, bdesc, 1u);
}

template <int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
                 const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  using L = GemmSmem<BN>;
  constexpr int STAGES = L::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);  // warp-uniform role
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmA2);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int num_n_tiles = p.N / BN;
  const int m0 = (blockIdx.x / num_n_tiles) * BM;
  const int n0 = (blockIdx.x % num_n_tiles) * BN;
  const int num_kb = p.K / BK;

  if (wg == 0) {
    // ===================== TMA producer =====================
    reg_dealloc<40>();
    if (warp == 0) {
      int s = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&empty_bar[s], phase ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&full_bar[s], L::STAGE_BYTES);
          uint8_t* sa = smem + s * L::STAGE_BYTES;
          uint8_t* sb = sa + L::A_BYTES;
          if (kb < p.k_split_blocks) tma_load_2d(sa, &tmA, &full_bar[s], kb * BK, m0, kEvictNormal);
          else tma_load_2d(sa, &tmA2, &full_bar[s], (kb - p.k_split_blocks) * BK, m0, kEvictNormal);
          tma_load_2d(sb, &tmB, &full_bar[s], kb * BK, n0, kEvictLast);
        }
        __syncwarp();
        if (++s == STAGES) { s = 0; phase ^= 1; }
      }
    }
  } else {
    // ===================== consumers: warpgroup 1 rows [0, 64), warpgroup 2 rows [64, 128) of the tile =====================
    reg_alloc<232>();
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    const uint32_t a_row_off = (wg - 1) * 64 * 128;  // 64 rows of 128 B (a multiple of the 1024-B swizzle atom)
    int s = 0, s_prev = 0;
    uint32_t phase = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[s], phase);
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
        if (lane == 0) mbar_arrive(&empty_bar[s_prev]);
      }
      s_prev = s;
      if (++s == STAGES) { s = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);
    const int r0 = m0 + (wg - 1) * 64 + (warp & 3) * 16 + (lane >> 2);
    epilogue_tile<BN>(p, acc, n0, r0);
  }
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
    uint32_t box[2] = {BK, BN};
    int r = encode_tmap_bf16(&tmB, a->w, 2, dims, str, box);
    if (r) return r;
  }
  GemmParams p = make_params(a);
  auto kern = gemm_bf16_kernel<BN>;
  {
    int r = ensure_smem_optin(kern, L::TOTAL);
    if (r) return r;
  }
  const long long num_tiles = (long long)(a->n / BN) * ((a->m + BM - 1) / BM);
  AMB_CHECK_ARG(num_tiles < 0x7fffffffLL, "gemm: too many tiles (m=%d n=%d)", a->m, a->n);
  kern<<<(unsigned)num_tiles, GEMM_THREADS, L::TOTAL, stream>>>(tmA, tmA2, tmB, p);
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
  AMB_CHECK_ARG(a->act == 0 || a->act == 1, "gemm: unknown activation %d", a->act);
  AMB_CHECK_ARG(!a->c2 || a->ldc2 % 8 == 0, "gemm: ldc2 must be a multiple of 8");
  if (a->norm_cols > 0 || a->rope_cols > 0) {
    AMB_CHECK_ARG(a->n % 128 == 0 && a->norm_cols % 128 == 0 && a->rope_cols % 128 == 0,
                  "gemm: head epilogue needs n, norm_cols, rope_cols multiples of 128");
    AMB_CHECK_ARG(a->norm_cols == 0 || (a->norm_w0 && a->norm_seg % 128 == 0), "gemm: norm weights / norm_seg (multiple of 128) required");
    AMB_CHECK_ARG(a->rope_cols == 0 || (a->rope_cos && a->rope_sin), "gemm: rope tables required");
    AMB_CHECK_ARG(!a->residual && a->act == 0 && !a->col_scale && !a->c2, "gemm: head epilogue excludes residual/activation/col_scale/c2");
  }
  cudaStream_t s = (cudaStream_t)stream;
  if (a->n % 256 == 0) return launch_gemm<256>(a, s);
  if (a->n % 128 == 0) return launch_gemm<128>(a, s);
  return launch_gemm<64>(a, s);
}
