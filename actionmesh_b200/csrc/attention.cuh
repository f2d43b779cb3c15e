// Tensor maps and parameters of the flash-attention kernel (attention.cu).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include "common.cuh"
#include "../../include/actionmesh_b200.h"

namespace amb {

struct AttnParams {
  __nv_bfloat16* o;
  long long o_stride_b, o_stride_h, o_stride_s;
  int heads, sq, sk;
  int kv_chunks, sk_chunk;   // kv split into chunks along the outermost tensor-map coordinate
  float scale_log2;          // scale * log2(e)
};

// Q map is 4-D (d, s, head, batch); K/V maps are 5-D (d, key, head, batch, chunk) with free strides: one chunk per rank
// of a frame-sharded window (the all-gather output is chunk-major), a single chunk otherwise.  All boxes are 64 columns
// (128 bytes, SWIZZLE_128B) wide.
inline int encode_attn_maps(const amb_attn_args* a, int D, uint32_t q_rows, uint32_t k_rows, uint32_t v_rows,
                            CUtensorMap* tmQ, CUtensorMap* tmK, CUtensorMap* tmV) {
  const int chunks = a->kv_chunks > 0 ? a->kv_chunks : 1;
  const int sk_chunk = chunks > 1 ? a->sk_chunk : a->sk;
  {
    uint64_t dims[4] = {(uint64_t)D, (uint64_t)a->sq, (uint64_t)a->heads, (uint64_t)a->batch};
    uint64_t str[3] = {(uint64_t)a->q_stride_s * 2, (uint64_t)a->q_stride_h * 2, (uint64_t)a->q_stride_b * 2};
    uint32_t box[4] = {64, q_rows, 1, 1};
    int r = encode_tmap_bf16(tmQ, a->q, 4, dims, str, box);
    if (r) return r;
  }
  auto enc_kv = [&](CUtensorMap* tm, const void* base, int64_t ss, int64_t sh, int64_t sb, int64_t schunk,
                    uint32_t rows) -> int {
    if (chunks == 1) schunk = sb > 0 ? sb : 16;  // extent-1 dimension: any legal stride
    uint64_t dims[5] = {(uint64_t)D, (uint64_t)sk_chunk, (uint64_t)a->heads, (uint64_t)a->batch, (uint64_t)chunks};
    uint64_t str[4] = {(uint64_t)ss * 2, (uint64_t)sh * 2, (uint64_t)sb * 2, (uint64_t)schunk * 2};
    if (a->batch == 1 && str[2] == 0) str[2] = str[0] * sk_chunk;
    uint32_t box[5] = {64, rows, 1, 1, 1};
    return encode_tmap_bf16(tm, base, 5, dims, str, box);
  };
  int r = enc_kv(tmK, a->k, a->k_stride_s, a->k_stride_h, a->k_stride_b, a->k_chunk_stride, k_rows);
  if (r) return r;
  return enc_kv(tmV, a->v, a->v_stride_s, a->v_stride_h, a->v_stride_b, a->v_chunk_stride, v_rows);
}

inline AttnParams make_attn_params(const amb_attn_args* a) {
  AttnParams p;
  p.o = reinterpret_cast<__nv_bfloat16*>(a->o);
  p.o_stride_b = a->o_stride_b; p.o_stride_h = a->o_stride_h; p.o_stride_s = a->o_stride_s;
  p.heads = a->heads; p.sq = a->sq; p.sk = a->sk;
  p.kv_chunks = a->kv_chunks > 0 ? a->kv_chunks : 1;
  p.sk_chunk = p.kv_chunks > 1 ? a->sk_chunk : a->sk;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  return p;
}

}  // namespace amb
