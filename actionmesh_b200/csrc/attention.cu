// wgmma flash-attention forward for sm_90a (non-causal, no mask):  O = softmax(scale · Q Kᵀ) V
// Replaces F.scaled_dot_product_attention at actionmesh/model/utils/attention_processor.py:133-139 (head_dim 128) and
// DinoV2's attention (head_dim 64).
//
// One CTA owns 128 query rows of one (batch, head); three warpgroups:
//   warpgroup 0     TMA producer: the Q tile once, then a STAGES-deep ring of BK-key K and V tiles (strided 4-D / 5-D tensor
//                   maps, so q/k/v are read in place from the fused QKV GEMM output).  K and V have their own full and empty
//                   barriers: Q·Kᵀ starts before V has landed, and a K slot is refilled as soon as its S = Q·Kᵀ is done.
//                   It also watches the consumers for a stall (bounded wait and trap), since they hold 240 registers and
//                   ptxas allocates fewer to a warp that can trap.
//   warpgroups 1-2  consumers, 64 query rows each:  S = Q·Kᵀ (wgmma, both operands in shared memory) -> online softmax in
//                   registers (exp2 with the scale folded in; a row lives in one quad, so its max / sum are two shuffles) ->
//                   O += P·V (wgmma with P as the register A operand, V MN-major from shared memory).
// The consumers are software-pipelined: S_{j+1} = Q·K_{j+1}ᵀ and O += P_j·V_j are issued together, and the softmax of S_{j+1}
// runs while P_j·V_j is still on the tensor cores.  The two consumer warpgroups take turns issuing their MMAs (named
// barriers 1 and 2), so one warpgroup's softmax also overlaps the other's MMAs.
// Key tiles are BK = 128 or 176 keys wide: every tile costs each consumer the same barrier waits, turn handoff,
// wgmma commit/wait pairs and O rescale whatever its width, so long rows run on 176-key tiles, 27 % fewer of them.
#include "common.cuh"
#include "ptx.cuh"
#include "attention.cuh"

namespace amb {

constexpr int ATT_BQ = 128;   // query rows per CTA (64 per consumer warpgroup)
constexpr int ATT_THREADS = 384;
constexpr int ATT_STAGES = 2;
// Long rows (head_dim 128, at least this many keys per chunk) run on 176-key tiles; everything else on 128-key tiles.
constexpr int ATT_LONG_BK = 176;
constexpr int ATT_LONG_MIN_KEYS = 4096;

// Shared memory of one CTA.  Q and every K / V tile are stored as 64-column (128-B, SWIZZLE_128B) boxes, one box after the
// other along d; a box of R rows is R x 128 B, so with R a multiple of 8 every box starts on a 1024-B swizzle atom.
// BK = 176, D = 128: 32 KB of Q + 2 stages x (44 KB K + 44 KB V) = 208 KB.
template <int D, int BK>
struct AttnSmem {
  static_assert(BK == 128 || BK == 176, "qk_issue has Q·Kᵀ wrappers for N = 128 and 176 only");
  static constexpr int Q_BOX_BYTES = ATT_BQ * 128;              // 128 query rows x 64 columns of bf16
  static constexpr int KV_BOX_BYTES = BK * 128;                 // BK keys x 64 columns of bf16
  static constexpr int Q_BYTES = (D / 64) * Q_BOX_BYTES;
  static constexpr int KV_BYTES = (D / 64) * KV_BOX_BYTES;      // one K or V tile of BK keys
  static constexpr int Q_OFF = 0;
  static constexpr int K_OFF = Q_BYTES;
  static constexpr int V_OFF = K_OFF + ATT_STAGES * KV_BYTES;
  static constexpr int BAR_OFF = V_OFF + ATT_STAGES * KV_BYTES;
  static constexpr int NUM_BARS = 1 + 4 * ATT_STAGES;            // q_full, k_full[], v_full[], k_empty[], v_empty[]
  static constexpr int TOTAL = BAR_OFF + NUM_BARS * 8 + 1024;
};

// S = Q·K_sᵀ for one warpgroup (64 x BK): 16 columns of d per k16 step, +32 B inside a 128-B row, next box after 4 steps.
// The first step overwrites the accumulator (scale-d 0).
template <int D, int BK>
__device__ __forceinline__ void qk_issue(float* sc, uint32_t sq_addr, uint32_t sk_addr) {
  using L = AttnSmem<D, BK>;
#pragma unroll
  for (int k = 0; k < D / 16; ++k) {
    const uint64_t qdesc = make_desc_kmajor_sw128(sq_addr + (k >> 2) * L::Q_BOX_BYTES + (k & 3) * 32);
    const uint64_t kdesc = make_desc_kmajor_sw128(sk_addr + (k >> 2) * L::KV_BOX_BYTES + (k & 3) * 32);
    if constexpr (BK == 176) wgmma_ss_n176(sc, qdesc, kdesc, k > 0 ? 1u : 0u);
    else wgmma_ss_n128(sc, qdesc, kdesc, k > 0 ? 1u : 0u);
  }
  wgmma_commit();
}

// O += P·V_s: 16 keys per step = 2048 B of the MN-major V tile; the second 64-column box of d is KV_BOX_BYTES further
// (22 528 B at BK = 176: still a whole number of 1024-B swizzle atoms).
template <int D, int BK>
__device__ __forceinline__ void pv_issue(float* o, const uint32_t* pk, uint32_t sv_addr) {
#pragma unroll
  for (int kk = 0; kk < BK / 16; ++kk) {
    const uint64_t vdesc = make_desc_mnmajor_sw128(sv_addr + kk * 2048, AttnSmem<D, BK>::KV_BOX_BYTES);
    if constexpr (D == 128) wgmma_rs_n128_tb(o, pk + 4 * kk, vdesc, 1u);
    else wgmma_rs_n64_tb(o, pk + 4 * kk, vdesc, 1u);
  }
  wgmma_commit();
}

// Online-softmax update with one S tile (sc[4i + {0,1}] = row a, keys 8i + 2q + {0,1}; sc[4i + {2,3}] = row b, same keys):
// keys >= valid are masked, the running maxima m rise, sc becomes exp2((S - m)·c), its row sums are added to l, and al gets
// the factors exp2((m_old - m)·c) that rescale the older terms (0 on the first tile).
template <int BK>
__device__ __forceinline__ void softmax_tile(float* sc, int valid, int q, float c, float& m_a, float& m_b, float& l_a,
                                             float& l_b, float& al_a, float& al_b) {
  if (valid < BK) {
#pragma unroll
    for (int i = 0; i < BK / 8; ++i) {
      const int key = 8 * i + 2 * q;
      if (key >= valid) sc[4 * i] = sc[4 * i + 2] = -INFINITY;
      if (key + 1 >= valid) sc[4 * i + 1] = sc[4 * i + 3] = -INFINITY;
    }
  }
  float mx_a = m_a, mx_b = m_b;
#pragma unroll
  for (int i = 0; i < BK / 8; ++i) {
    mx_a = fmaxf(mx_a, fmaxf(sc[4 * i], sc[4 * i + 1]));
    mx_b = fmaxf(mx_b, fmaxf(sc[4 * i + 2], sc[4 * i + 3]));
  }
  mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 1));
  mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 1));
  mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 2));
  mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 2));
  al_a = ex2_approx((m_a - mx_a) * c);
  al_b = ex2_approx((m_b - mx_b) * c);
  m_a = mx_a;
  m_b = mx_b;
  const float mb_a = m_a * c, mb_b = m_b * c;
  float ts_a = 0.f, ts_b = 0.f;
#pragma unroll
  for (int i = 0; i < BK / 8; ++i) {
    sc[4 * i] = ex2_approx(fmaf(sc[4 * i], c, -mb_a));
    sc[4 * i + 1] = ex2_approx(fmaf(sc[4 * i + 1], c, -mb_a));
    sc[4 * i + 2] = ex2_approx(fmaf(sc[4 * i + 2], c, -mb_b));
    sc[4 * i + 3] = ex2_approx(fmaf(sc[4 * i + 3], c, -mb_b));
    ts_a += sc[4 * i] + sc[4 * i + 1];
    ts_b += sc[4 * i + 2] + sc[4 * i + 3];
  }
  l_a = l_a * al_a + ts_a;
  l_b = l_b * al_b + ts_b;
}

// A fragment of P·V from the exponentials: (row a, keys 2q, 2q+1) / (row b, ...) of 8-key group i.
template <int BK>
__device__ __forceinline__ void pack_p(uint32_t* pk, const float* sc) {
#pragma unroll
  for (int i = 0; i < BK / 8; ++i) {
    pk[2 * i] = pack_bf16(sc[4 * i], sc[4 * i + 1]);
    pk[2 * i + 1] = pack_bf16(sc[4 * i + 2], sc[4 * i + 3]);
  }
}

template <int D, int BK>
__global__ void __launch_bounds__(ATT_THREADS, 1)
flash_attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                      const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  using L = AttnSmem<D, BK>;
  constexpr int DH = D / 64;  // 64-column boxes per row
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* k_full = q_full + 1;
  uint64_t* v_full = k_full + ATT_STAGES;
  uint64_t* k_empty = v_full + ATT_STAGES;
  uint64_t* v_empty = k_empty + ATT_STAGES;

  const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);  // warp-uniform role
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * ATT_BQ;
  const int head = blockIdx.y;
  const int batch = blockIdx.z;
  const int tiles_per_chunk = (p.sk_chunk + BK - 1) / BK;
  const int n_kv = p.kv_chunks * tiles_per_chunk;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int s = 0; s < ATT_STAGES; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&v_full[s], 1);
      mbar_init(&k_empty[s], 8);  // one arrival per consumer warp
      mbar_init(&v_empty[s], 8);
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
          tma_load_4d(smem + L::Q_OFF + c * L::Q_BOX_BYTES, &tmQ, q_full, c * 64, q0, head, batch, kEvictFirst);
      }
      __syncwarp();
      int s = 0;
      uint32_t phase = 0;
      for (int j = 0; j < n_kv; ++j) {  // K/V maps are 5-D: (d, key, head, batch, chunk)
        const int chunk = j / tiles_per_chunk;
        const int key0 = (j - chunk * tiles_per_chunk) * BK;
        mbar_wait(&k_empty[s], phase ^ 1);  // K_j's slot frees before V_j's: load it first
        if (elect_one()) {
          uint8_t* sk = smem + L::K_OFF + s * L::KV_BYTES;
          mbar_expect_tx(&k_full[s], L::KV_BYTES);
          for (int c = 0; c < DH; ++c)
            tma_load_5d(sk + c * L::KV_BOX_BYTES, &tmK, &k_full[s], c * 64, key0, head, batch, chunk, kEvictLast);
        }
        __syncwarp();
        mbar_wait(&v_empty[s], phase ^ 1);
        if (elect_one()) {
          uint8_t* sv = smem + L::V_OFF + s * L::KV_BYTES;
          mbar_expect_tx(&v_full[s], L::KV_BYTES);
          for (int c = 0; c < DH; ++c)
            tma_load_5d(sv + c * L::KV_BOX_BYTES, &tmV, &v_full[s], c * 64, key0, head, batch, chunk, kEvictLast);
        }
        __syncwarp();
        if (++s == ATT_STAGES) { s = 0; phase ^= 1; }
      }
      // Watchdog: the consumers wait without a timeout (see mbar_wait_watched), so this warp waits, bounded, until they
      // have released the last STAGES tiles.  A stalled consumer makes that wait trap and the launch fail.
      for (int j = 0; j < ATT_STAGES; ++j) {
        mbar_wait(&k_empty[s], phase ^ 1);
        mbar_wait(&v_empty[s], phase ^ 1);
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
    const int last_valid = p.sk_chunk - (tiles_per_chunk - 1) * BK;  // valid keys in the last tile of each chunk
    // Issue turns: warpgroup w waits on named barrier w before issuing and then lets the other one go.  Warpgroup 1 takes the
    // first turn without waiting and warpgroup 2 gives no go-ahead after its last turn, so every arrival is matched by a wait.
    const uint32_t my_turn = wg, other_turn = 3 - wg;

    float o[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
    float m_a = -INFINITY, m_b = -INFINITY;  // running maxima (raw score units) of my two rows
    float l_a = 0.f, l_b = 0.f;              // partial row sums over my columns
    float al_a, al_b;
    float sc[BK / 2];
    uint32_t pk[BK / 4];

    // ---- prologue: S_0 and its softmax (O is still zero: nothing to rescale)
    mbar_wait_watched(q_full, 0);
    mbar_wait_watched(&k_full[0], 0);
    if (wg == 2) named_bar_sync(my_turn, 256);
    wgmma_fence();
    qk_issue<D, BK>(sc, sq_addr, sk_addr);
    named_bar_arrive(other_turn, 256);
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < BK / 2; ++i) reg_fence(sc[i]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&k_empty[0]);  // this warp is done with K_0
    int jn = tiles_per_chunk == 1 ? 0 : 1;    // tile index inside its chunk of the NEXT tile
    softmax_tile<BK>(sc, tiles_per_chunk == 1 ? last_valid : BK, q, c, m_a, m_b, l_a, l_b, al_a, al_b);
    pack_p<BK>(pk, sc);

    int s = 0;
    uint32_t phase = 0;
    for (int j = 0; j + 1 < n_kv; ++j) {
      int sn = s + 1;
      uint32_t phn = phase;
      if (sn == ATT_STAGES) { sn = 0; phn ^= 1; }
      // ---- issue S_{j+1} = Q·K_{j+1}ᵀ, then O += P_j·V_j
      mbar_wait_watched(&k_full[sn], phn);
      mbar_wait_watched(&v_full[s], phase);
      named_bar_sync(my_turn, 256);
      wgmma_fence();
      qk_issue<D, BK>(sc, sq_addr, sk_addr + sn * L::KV_BYTES);
      pv_issue<D, BK>(o, pk, sv_addr + s * L::KV_BYTES);
      named_bar_arrive(other_turn, 256);
      // ---- softmax of S_{j+1} while P_j·V_j runs
      wgmma_wait<1>();
#pragma unroll
      for (int i = 0; i < BK / 2; ++i) reg_fence(sc[i]);
      __syncwarp();
      if (lane == 0) mbar_arrive(&k_empty[sn]);
      softmax_tile<BK>(sc, jn == tiles_per_chunk - 1 ? last_valid : BK, q, c, m_a, m_b, l_a, l_b, al_a, al_b);
      if (++jn == tiles_per_chunk) jn = 0;
      // ---- P_j·V_j done: release V_j, rescale O for tile j+1 and pack P_{j+1}
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < D / 2; ++i) reg_fence(o[i]);
      __syncwarp();
      if (lane == 0) mbar_arrive(&v_empty[s]);
#pragma unroll
      for (int i = 0; i < D / 8; ++i) {
        o[4 * i] *= al_a;
        o[4 * i + 1] *= al_a;
        o[4 * i + 2] *= al_b;
        o[4 * i + 3] *= al_b;
      }
      pack_p<BK>(pk, sc);
      s = sn;
      phase = phn;
    }

    // ---- last tile: O += P·V
    mbar_wait_watched(&v_full[s], phase);
    named_bar_sync(my_turn, 256);
    wgmma_fence();
    pv_issue<D, BK>(o, pk, sv_addr + s * L::KV_BYTES);
    if (wg == 1) named_bar_arrive(other_turn, 256);
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < D / 2; ++i) reg_fence(o[i]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&v_empty[s]);

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

template <int D, int BK>
static int launch_attn(const amb_attn_args* a, cudaStream_t stream) {
  using L = AttnSmem<D, BK>;
  CUtensorMap tmQ, tmK, tmV;
  int r = encode_attn_maps(a, D, ATT_BQ, BK, BK, &tmQ, &tmK, &tmV);
  if (r) return r;
  const AttnParams p = make_attn_params(a);
  dim3 grid((a->sq + ATT_BQ - 1) / ATT_BQ, a->heads, a->batch);
  auto kern = flash_attn_fwd_kernel<D, BK>;
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
  if (a->head_dim == 64) return launch_attn<64, 128>(a, s);
  // The tile width depends on the shape alone, so chunks made of whole tiles of the width a call selects reproduce the
  // single call bit for bit (DESIGN 5).
  const int sk_chunk = a->kv_chunks > 1 ? a->sk_chunk : a->sk;
  if (sk_chunk >= ATT_LONG_MIN_KEYS) return launch_attn<128, ATT_LONG_BK>(a, s);
  return launch_attn<128, 128>(a, s);
}
