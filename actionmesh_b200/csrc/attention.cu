// wgmma flash-attention forward for sm_90a (non-causal, no mask):  O = softmax(scale · Q Kᵀ) V
// Replaces F.scaled_dot_product_attention at actionmesh/model/utils/attention_processor.py:133-139 (head_dim 128) and
// DinoV2's attention (head_dim 64).
//
// One CTA owns 128 query rows of one (batch, head); three warpgroups:
//   warpgroup 0     TMA producer: the Q tile once, then a STAGES-deep ring of 128-key K and V tiles (strided 4-D / 5-D tensor
//                   maps, so q/k/v are read in place from the fused QKV GEMM output; K and V on separate barriers so that
//                   Q·Kᵀ starts before V has landed)
//   warpgroups 1-2  consumers, 64 query rows each:  S = Q·Kᵀ (wgmma, both operands in shared memory) -> online softmax in
//                   registers (exp2 with the scale folded in; a row lives in one quad, so its max / sum are two shuffles) ->
//                   O += P·V (wgmma with P as the register A operand, V MN-major from shared memory).  The two consumer
//                   warpgroups interleave: one computes exponentials while the other's MMAs run.
#include "common.cuh"
#include "ptx.cuh"
#include "attention.cuh"

namespace amb {

constexpr int ATT_BQ = 128;   // query rows per CTA (64 per consumer warpgroup)
constexpr int ATT_BK = 128;   // keys per K/V tile
constexpr int ATT_THREADS = 384;
constexpr int ATT_STAGES = 2;

template <int D>
struct AttnSmem {
  static constexpr int BOX_BYTES = 128 * 128;                   // 128 rows x 64 columns of bf16 (one SWIZZLE_128B box)
  static constexpr int Q_BYTES = (D / 64) * BOX_BYTES;
  static constexpr int KV_BYTES = (D / 64) * BOX_BYTES;         // one K or V tile of 128 keys
  static constexpr int Q_OFF = 0;
  static constexpr int K_OFF = Q_BYTES;
  static constexpr int V_OFF = K_OFF + ATT_STAGES * KV_BYTES;
  static constexpr int BAR_OFF = V_OFF + ATT_STAGES * KV_BYTES;
  static constexpr int NUM_BARS = 1 + 3 * ATT_STAGES;            // q_full, k_full[], v_full[], kv_empty[]
  static constexpr int TOTAL = BAR_OFF + NUM_BARS * 8 + 1024;
};

template <int D>
__device__ __forceinline__ void pv_k16(float* o, const uint32_t* a, uint64_t vdesc) {
  if constexpr (D == 128) wgmma_rs_n128_tb(o, a, vdesc, 1u);
  else wgmma_rs_n64_tb(o, a, vdesc, 1u);
}

template <int D>
__global__ void __launch_bounds__(ATT_THREADS, 1)
flash_attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                      const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  using L = AttnSmem<D>;
  constexpr int DH = D / 64;  // 64-column boxes per row
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* k_full = q_full + 1;
  uint64_t* v_full = k_full + ATT_STAGES;
  uint64_t* kv_empty = v_full + ATT_STAGES;

  const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);  // warp-uniform role
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * ATT_BQ;
  const int head = blockIdx.y;
  const int batch = blockIdx.z;
  const int tiles_per_chunk = (p.sk_chunk + ATT_BK - 1) / ATT_BK;
  const int n_kv = p.kv_chunks * tiles_per_chunk;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int s = 0; s < ATT_STAGES; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&v_full[s], 1);
      mbar_init(&kv_empty[s], 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    reg_dealloc<24>();
    if (warp == 0) {
      if (elect_one()) {
        mbar_expect_tx(q_full, L::Q_BYTES);
        for (int c = 0; c < DH; ++c)
          tma_load_4d(smem + L::Q_OFF + c * L::BOX_BYTES, &tmQ, q_full, c * 64, q0, head, batch, kEvictFirst);
      }
      __syncwarp();
      int s = 0;
      uint32_t phase = 0;
      for (int j = 0; j < n_kv; ++j) {
        const int chunk = j / tiles_per_chunk;
        const int key0 = (j - chunk * tiles_per_chunk) * ATT_BK;
        mbar_wait(&kv_empty[s], phase ^ 1);
        if (elect_one()) {  // K/V maps are 5-D: (d, key, head, batch, chunk)
          uint8_t* sk = smem + L::K_OFF + s * L::KV_BYTES;
          uint8_t* sv = smem + L::V_OFF + s * L::KV_BYTES;
          mbar_expect_tx(&k_full[s], L::KV_BYTES);
          for (int c = 0; c < DH; ++c)
            tma_load_5d(sk + c * L::BOX_BYTES, &tmK, &k_full[s], c * 64, key0, head, batch, chunk, kEvictLast);
          mbar_expect_tx(&v_full[s], L::KV_BYTES);
          for (int c = 0; c < DH; ++c)
            tma_load_5d(sv + c * L::BOX_BYTES, &tmV, &v_full[s], c * 64, key0, head, batch, chunk, kEvictLast);
        }
        __syncwarp();
        if (++s == ATT_STAGES) { s = 0; phase ^= 1; }
      }
    }
  } else {
    // ===================== consumers =====================
    reg_alloc<240>();
    const int q = lane & 3;
    const int r_local = (wg - 1) * 64 + (warp & 3) * 16 + (lane >> 2);  // my rows: r_local and r_local + 8
    const uint32_t sq_addr = smem_u32(smem + L::Q_OFF) + (wg - 1) * 64 * 128;
    const uint32_t sk_addr = smem_u32(smem + L::K_OFF);
    const uint32_t sv_addr = smem_u32(smem + L::V_OFF);
    const float c = p.scale_log2;
    const int last_valid = p.sk_chunk - (tiles_per_chunk - 1) * ATT_BK;  // valid keys in the last tile of each chunk

    float o[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
    float m_a = -INFINITY, m_b = -INFINITY;  // running maxima (raw score units) of my two rows
    float l_a = 0.f, l_b = 0.f;              // partial row sums over my columns

    mbar_wait(q_full, 0);
    int s = 0, jj = 0;
    uint32_t phase = 0;
    for (int j = 0; j < n_kv; ++j) {
      // ---- S = Q Kᵀ (64 x 128 per warpgroup)
      float sc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) sc[i] = 0.f;
      mbar_wait(&k_full[s], phase);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < D / 16; ++k) {  // 16 columns of d per step: +32 B inside a 128-B row, next box after 4 steps
        const uint32_t off = (k >> 2) * L::BOX_BYTES + (k & 3) * 32;
        wgmma_ss_n128(sc, make_desc_kmajor_sw128(sq_addr + off), make_desc_kmajor_sw128(sk_addr + s * L::KV_BYTES + off), 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < 64; ++i) reg_fence(sc[i]);

      // ---- online softmax: sc[4i + {0,1}] = row a, keys 8i + 2q + {0,1}; sc[4i + {2,3}] = row b, same keys
      if (jj == tiles_per_chunk - 1 && last_valid < ATT_BK) {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int key = 8 * i + 2 * q;
          if (key >= last_valid) sc[4 * i] = sc[4 * i + 2] = -INFINITY;
          if (key + 1 >= last_valid) sc[4 * i + 1] = sc[4 * i + 3] = -INFINITY;
        }
      }
      if (++jj == tiles_per_chunk) jj = 0;
      float mx_a = m_a, mx_b = m_b;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        mx_a = fmaxf(mx_a, fmaxf(sc[4 * i], sc[4 * i + 1]));
        mx_b = fmaxf(mx_b, fmaxf(sc[4 * i + 2], sc[4 * i + 3]));
      }
      mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 1));
      mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 1));
      mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 2));
      mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 2));
      const float al_a = ex2_approx((m_a - mx_a) * c), al_b = ex2_approx((m_b - mx_b) * c);  // 0 on the first tile
      m_a = mx_a;
      m_b = mx_b;
      const float mb_a = m_a * c, mb_b = m_b * c;
      uint32_t pk[32];
      float ts_a = 0.f, ts_b = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float ea0 = ex2_approx(fmaf(sc[4 * i], c, -mb_a)), ea1 = ex2_approx(fmaf(sc[4 * i + 1], c, -mb_a));
        const float eb0 = ex2_approx(fmaf(sc[4 * i + 2], c, -mb_b)), eb1 = ex2_approx(fmaf(sc[4 * i + 3], c, -mb_b));
        ts_a += ea0 + ea1;
        ts_b += eb0 + eb1;
        pk[2 * i] = pack_bf16(ea0, ea1);      // A fragment of P·V: (row a, keys 2q, 2q+1) / (row b, ...) of 8-key group i
        pk[2 * i + 1] = pack_bf16(eb0, eb1);
      }
      l_a = l_a * al_a + ts_a;
      l_b = l_b * al_b + ts_b;
#pragma unroll
      for (int i = 0; i < D / 8; ++i) {
        o[4 * i] *= al_a;
        o[4 * i + 1] *= al_a;
        o[4 * i + 2] *= al_b;
        o[4 * i + 3] *= al_b;
      }

      // ---- O += P V: 16 keys per step = 2048 B of the MN-major V tile; the second 64-column box of d is BOX_BYTES further
      mbar_wait(&v_full[s], phase);
      wgmma_fence();
      const uint32_t vbase = sv_addr + s * L::KV_BYTES;
#pragma unroll
      for (int kk = 0; kk < ATT_BK / 16; ++kk)
        pv_k16<D>(o, pk + 4 * kk, make_desc_mnmajor_sw128(vbase + kk * 2048, L::BOX_BYTES));
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < D / 2; ++i) reg_fence(o[i]);
      __syncwarp();
      if (lane == 0) mbar_arrive(&kv_empty[s]);  // this warp is done with K_j and V_j
      if (++s == ATT_STAGES) { s = 0; phase ^= 1; }
    }

    // ---- epilogue: O / rowsum -> bf16 -> global (b, s, h, d)
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 1);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 1);
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
    const float inv_a = 1.0f / l_a, inv_b = 1.0f / l_b;
    const int qr_a = q0 + r_local, qr_b = qr_a + 8;
    __nv_bfloat16* obase = p.o + (long long)batch * p.o_stride_b + (long long)head * p.o_stride_h + 2 * q;
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      if (qr_a < p.sq)
        *reinterpret_cast<uint32_t*>(obase + (long long)qr_a * p.o_stride_s + 8 * i) = pack_bf16(o[4 * i] * inv_a, o[4 * i + 1] * inv_a);
      if (qr_b < p.sq)
        *reinterpret_cast<uint32_t*>(obase + (long long)qr_b * p.o_stride_s + 8 * i) = pack_bf16(o[4 * i + 2] * inv_b, o[4 * i + 3] * inv_b);
    }
  }
}

template <int D>
static int launch_attn(const amb_attn_args* a, cudaStream_t stream) {
  using L = AttnSmem<D>;
  CUtensorMap tmQ, tmK, tmV;
  int r = encode_attn_maps(a, D, ATT_BQ, ATT_BK, ATT_BK, &tmQ, &tmK, &tmV);
  if (r) return r;
  const AttnParams p = make_attn_params(a);
  dim3 grid((a->sq + ATT_BQ - 1) / ATT_BQ, a->heads, a->batch);
  auto kern = flash_attn_fwd_kernel<D>;
  r = ensure_smem_optin(kern, L::TOTAL);
  if (r) return r;
  kern<<<grid, ATT_THREADS, L::TOTAL, stream>>>(tmQ, tmK, tmV, p);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

}  // namespace amb

using namespace amb;

extern "C" int amb_flash_attn_fwd(const amb_attn_args* a, amb_stream_t stream) {
  AMB_CHECK_ARG(a && a->q && a->k && a->v && a->o, "flash_attn: null pointer");
  AMB_CHECK_ARG(a->batch > 0 && a->heads > 0 && a->sq > 0 && a->sk > 0, "flash_attn: bad shape b=%d h=%d sq=%d sk=%d",
                a->batch, a->heads, a->sq, a->sk);
  AMB_CHECK_ARG(a->head_dim == 128 || a->head_dim == 64, "flash_attn: head_dim %d unsupported (64 or 128)", a->head_dim);
  AMB_CHECK_ARG(a->q_stride_s % 8 == 0 && a->k_stride_s % 8 == 0 && a->v_stride_s % 8 == 0 && a->o_stride_s % 8 == 0 &&
                    a->q_stride_h % 8 == 0 && a->k_stride_h % 8 == 0 && a->v_stride_h % 8 == 0 && a->o_stride_h % 8 == 0 &&
                    a->q_stride_b % 8 == 0 && a->k_stride_b % 8 == 0 && a->v_stride_b % 8 == 0 && a->o_stride_b % 8 == 0,
                "flash_attn: strides must be multiples of 8 elements (16 bytes)");
  AMB_CHECK_ARG(a->kv_chunks <= 1 || (a->sk_chunk > 0 && (int64_t)a->sk_chunk * a->kv_chunks == a->sk),
                "flash_attn: kv_chunks * sk_chunk must equal sk");
  AMB_CHECK_ARG(a->batch <= 65535 && a->heads <= 65535, "flash_attn: grid limits");
  cudaStream_t s = (cudaStream_t)stream;
  if (a->head_dim == 64) return launch_attn<64>(a, s);
  return launch_attn<128>(a, s);
}
