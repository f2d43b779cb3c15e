// HBM-bound elementwise / row-reduction kernels of the denoising path (sm_90a).
//  - cfg_euler_step : CFG combine + Euler flow update + observed-frame mask   (scheduler.py:238-248, guidance.py:95-118)
//  - layernorm      : affine LayerNorm with fp32 statistics                    (block.py:64,83,98,107)
//  - cast / timestep embedding / bias-row add
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/actionmesh_b200.h"

namespace amb {

// ------------------------------------------------------------------------------------------------ K9
constexpr int kMaxBranches = 4;
struct CfgEulerParams {
  float* latents;
  const __nv_bfloat16* pred;
  const uint8_t* frame_update;
  float scales[kMaxBranches];
  float dt;
  int n_branches;
  int n_frames;
  long long n_per_frame;  // multiple of 8
  long long branch_stride, frame_stride, frame_offset;
};

// One thread = 8 consecutive latent elements: two 16 B fp32 reads + one 16 B read per bf16 branch + two 16 B writes, all
// coalesced; every load of an element group is issued before the first use (4 independent 16 B requests in flight).
__global__ void __launch_bounds__(256) cfg_euler_kernel(const CfgEulerParams p) {
  const long long vec_per_frame = p.n_per_frame >> 3;
  const long long total = vec_per_frame * p.n_frames;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int f = (int)(i / vec_per_frame);
    if (!p.frame_update[f]) continue;  // observed frame: bit-identical pass-through (scheduler.py:244-246)
    const long long e = (i - (long long)f * vec_per_frame) << 3;
    float4* xp = reinterpret_cast<float4*>(p.latents + (long long)f * p.n_per_frame + e);
    const __nv_bfloat16* pp = p.pred + (long long)f * p.frame_stride + p.frame_offset + e;
    uint4 raw[kMaxBranches];
#pragma unroll
    for (int k = 0; k < kMaxBranches; ++k)
      if (k < p.n_branches) raw[k] = __ldg(reinterpret_cast<const uint4*>(pp + (long long)k * p.branch_stride));
    float4 x0 = xp[0], x1 = xp[1];
    float v[8], q[8];
    {
      float2 a = unpack_bf16(raw[0].x), b = unpack_bf16(raw[0].y), c = unpack_bf16(raw[0].z), d = unpack_bf16(raw[0].w);
      v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
#pragma unroll
      for (int t = 0; t < 8; ++t) q[t] = v[t];
    }
#pragma unroll
    for (int k = 1; k < kMaxBranches; ++k) {
      if (k < p.n_branches) {
        float2 a = unpack_bf16(raw[k].x), b = unpack_bf16(raw[k].y), c = unpack_bf16(raw[k].z), d = unpack_bf16(raw[k].w);
        const float w[8] = {a.x, a.y, b.x, b.y, c.x, c.y, d.x, d.y};
        const float s = p.scales[k - 1];
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          v[t] += s * (w[t] - q[t]);
          q[t] = w[t];
        }
      }
    }
    x0.x += p.dt * v[0]; x0.y += p.dt * v[1]; x0.z += p.dt * v[2]; x0.w += p.dt * v[3];
    x1.x += p.dt * v[4]; x1.y += p.dt * v[5]; x1.z += p.dt * v[6]; x1.w += p.dt * v[7];
    xp[0] = x0;
    xp[1] = x1;
  }
}

// ------------------------------------------------------------------------------------------------ LayerNorm
// One warp per row; the row (<= 4096 elements) is held in registers between the statistics and the normalise pass, so
// HBM sees exactly one read and one write of the row.  Two-pass (mean, then centred variance) in fp32 like
// F.layer_norm on an fp32 upcast.
template <int COLS, bool XF32, bool YF32>
__global__ void __launch_bounds__(256) layernorm_kernel(const void* __restrict__ xv, long long ldx,
                                                        const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, void* __restrict__ yv,
                                                        long long ldy, long long rows, float eps) {
  constexpr int PER_LANE = COLS / 32;   // elements per lane
  constexpr int VEC = PER_LANE / 8;     // 8-element vectors per lane
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + warp;
  if (row >= rows) return;
  float v[PER_LANE];
  if constexpr (XF32) {
    const float* x = reinterpret_cast<const float*>(xv) + row * ldx;
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float4* p4 = reinterpret_cast<const float4*>(x + (j * 32 + lane) * 8);
      float4 a = __ldg(p4), b = __ldg(p4 + 1);
      v[j * 8 + 0] = a.x; v[j * 8 + 1] = a.y; v[j * 8 + 2] = a.z; v[j * 8 + 3] = a.w;
      v[j * 8 + 4] = b.x; v[j * 8 + 5] = b.y; v[j * 8 + 6] = b.z; v[j * 8 + 7] = b.w;
    }
  } else {
    const __nv_bfloat16* x = reinterpret_cast<const __nv_bfloat16*>(xv) + row * ldx;
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      uint4 r = __ldg(reinterpret_cast<const uint4*>(x + (j * 32 + lane) * 8));
      float2 f0 = unpack_bf16(r.x), f1 = unpack_bf16(r.y), f2 = unpack_bf16(r.z), f3 = unpack_bf16(r.w);
      v[j * 8 + 0] = f0.x; v[j * 8 + 1] = f0.y; v[j * 8 + 2] = f1.x; v[j * 8 + 3] = f1.y;
      v[j * 8 + 4] = f2.x; v[j * 8 + 5] = f2.y; v[j * 8 + 6] = f3.x; v[j * 8 + 7] = f3.y;
    }
  }
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < PER_LANE; ++j) s += v[j];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s * (1.0f / COLS);
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < PER_LANE; ++j) {
    const float d = v[j] - mean;
    q += d * d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q * (1.0f / COLS) + eps);
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    const int c = (j * 32 + lane) * 8;
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c)), b1 = __ldg(reinterpret_cast<const float4*>(beta + c + 4));
    if constexpr (YF32) {
      float* yr = reinterpret_cast<float*>(yv) + row * ldy + c;
      reinterpret_cast<float4*>(yr)[0] = make_float4((v[j * 8 + 0] - mean) * rstd * g0.x + b0.x, (v[j * 8 + 1] - mean) * rstd * g0.y + b0.y,
                                                     (v[j * 8 + 2] - mean) * rstd * g0.z + b0.z, (v[j * 8 + 3] - mean) * rstd * g0.w + b0.w);
      reinterpret_cast<float4*>(yr)[1] = make_float4((v[j * 8 + 4] - mean) * rstd * g1.x + b1.x, (v[j * 8 + 5] - mean) * rstd * g1.y + b1.y,
                                                     (v[j * 8 + 6] - mean) * rstd * g1.z + b1.z, (v[j * 8 + 7] - mean) * rstd * g1.w + b1.w);
      continue;
    }
    __nv_bfloat16* yr = reinterpret_cast<__nv_bfloat16*>(yv) + row * ldy;
    uint4 o;
    o.x = pack_bf16((v[j * 8 + 0] - mean) * rstd * g0.x + b0.x, (v[j * 8 + 1] - mean) * rstd * g0.y + b0.y);
    o.y = pack_bf16((v[j * 8 + 2] - mean) * rstd * g0.z + b0.z, (v[j * 8 + 3] - mean) * rstd * g0.w + b0.w);
    o.z = pack_bf16((v[j * 8 + 4] - mean) * rstd * g1.x + b1.x, (v[j * 8 + 5] - mean) * rstd * g1.y + b1.y);
    o.w = pack_bf16((v[j * 8 + 6] - mean) * rstd * g1.z + b1.z, (v[j * 8 + 7] - mean) * rstd * g1.w + b1.w);
    *reinterpret_cast<uint4*>(yr + c) = o;
  }
}

// ------------------------------------------------------------------------------------------------ helpers
__global__ void __launch_bounds__(256) cast_f32_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                                                            long long n) {
  const long long n4 = n >> 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 a = __ldg(reinterpret_cast<const float4*>(src) + i);
    uint2 o;
    o.x = pack_bf16(a.x, a.y);
    o.y = pack_bf16(a.z, a.w);
    reinterpret_cast<uint2*>(dst)[i] = o;
  }
  // tail (n % 4)
  const long long tail0 = n4 << 2;
  for (long long i = tail0 + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dst[i] = __float2bfloat16_rn(src[i]);
}

// diffusers Timesteps(flip_sin_to_cos=False, downscale_freq_shift=0): [sin(t w_j) | cos(t w_j)], w_j = exp(-ln(1e4) j / half)
// Row r uses t[r % n_t] * (1 - mask[r]): temporal_denoiser.py:209-212 (`diffusion_time.repeat(T) * (1 - mask)`, observed
// frames are conditioned on t = 0).
__global__ void timestep_embedding_kernel(const float* __restrict__ t, int n_t, const float* __restrict__ mask, int rows,
                                          int channels, __nv_bfloat16* __restrict__ out) {
  const int half = channels >> 1;
  const int r = blockIdx.x;
  const float tv = t[r % n_t] * (mask ? (1.0f - mask[r]) : 1.0f);
  for (int j = threadIdx.x; j < half; j += blockDim.x) {
    const float w = expf(-9.210340371976184f * (float)j / (float)half);
    const float a = tv * w;
    out[(long long)r * channels + j] = __float2bfloat16_rn(sinf(a));
    out[(long long)r * channels + half + j] = __float2bfloat16_rn(cosf(a));
  }
}

__global__ void __launch_bounds__(256) add_bias_rows_kernel(__nv_bfloat16* __restrict__ y, long long ldy,
                                                            const float* __restrict__ bias, long long rows, int cols) {
  const int vec_per_row = cols >> 3;
  const long long total = rows * vec_per_row;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / vec_per_row;
    const int c = (int)(i - r * vec_per_row) << 3;
    uint4* p = reinterpret_cast<uint4*>(y + r * ldy + c);
    uint4 raw = *p;
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + c)), b1 = __ldg(reinterpret_cast<const float4*>(bias + c + 4));
    float2 f0 = unpack_bf16(raw.x), f1 = unpack_bf16(raw.y), f2 = unpack_bf16(raw.z), f3 = unpack_bf16(raw.w);
    raw.x = pack_bf16(f0.x + b0.x, f0.y + b0.y);
    raw.y = pack_bf16(f1.x + b0.z, f1.y + b0.w);
    raw.z = pack_bf16(f2.x + b1.x, f2.y + b1.y);
    raw.w = pack_bf16(f3.x + b1.z, f3.y + b1.w);
    *p = raw;
  }
}

__global__ void __launch_bounds__(256) add_bias_rows_f32_kernel(float* __restrict__ y, long long ldy,
                                                                const float* __restrict__ bias, long long rows, int cols) {
  const int vec_per_row = cols >> 2;
  const long long total = rows * vec_per_row;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / vec_per_row;
    const int c = (int)(i - r * vec_per_row) << 2;
    float4* p = reinterpret_cast<float4*>(y + r * ldy + c);
    float4 v = *p;
    const float4 b = __ldg(reinterpret_cast<const float4*>(bias + c));
    v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
    *p = v;
  }
}

// DinoV2 patch embedding as a GEMM: im2col of (T,3,H,W) fp32 pixels into bf16 rows (t, py, px) x cols (c, ky, kx),
// zero-padded from 3*P*P to `kpad` columns (HF Dinov2PatchEmbeddings is Conv2d(3, D, P, stride P)).
__global__ void __launch_bounds__(256) patchify_kernel(const float* __restrict__ pix, __nv_bfloat16* __restrict__ out,
                                                       int T, int H, int W, int P, int kpad) {
  const int gw = W / P, gh = H / P;
  const long long total = (long long)T * gh * gw * kpad;
  const int kreal = 3 * P * P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(i % kpad);
    const long long row = i / kpad;
    float v = 0.f;
    if (col < kreal) {
      const int c = col / (P * P), r = col % (P * P), ky = r / P, kx = r % P;
      const int px = (int)(row % gw), py = (int)((row / gw) % gh), t = (int)(row / ((long long)gw * gh));
      v = pix[(((long long)t * 3 + c) * H + (py * P + ky)) * W + (px * P + kx)];
    }
    out[i] = __float2bfloat16_rn(v);
  }
}

// Stage II (temporal_autoencoder.py): (source_alpha, target_alpha) token, embeddings.py:56-132 TimestepEmbedder with
// frequency_embedding_size = size: [cos(s w) | sin(s w) | cos(t w) | sin(t w)], w_i = exp(-ln(1e4) i / (size/2)).
// The same 2*size vector is written to n_rows rows (one alpha token per frame).
__global__ void alpha_rows_kernel(float src, float tgt, int size, float* __restrict__ out, long long row_stride, int n_rows) {
  const int half = size >> 1;
  for (int i = threadIdx.x; i < 2 * size; i += blockDim.x) {
    const int which = i / size, j = i % size;
    const float t = which ? tgt : src;
    const int f = j % half;
    const float a = t * expf(-9.210340371976184f * (float)f / (float)half);
    const float v = (j < half) ? cosf(a) : sinf(a);
    out[(long long)blockIdx.x * row_stride + i] = v;
  }
}

// Stage II query embedding, embeddings.py:15-53 FrequencyPositionalEmbedding(logspace, include_input) + extra features:
// [x (3) | sin(x_c 2^f) (3*F) | cos(x_c 2^f) (3*F) | extra (E) | 0 ...] padded to `kpad` fp32 columns (the reference keeps
// the whole query path in fp32, temporal_autoencoder.py:240-243,264-266).
__global__ void __launch_bounds__(256) point_embedding_kernel(const float* __restrict__ q, int n_points, int in_dim, int extra,
                                                              int num_freqs, int include_pi, float* __restrict__ out, int kpad) {
  const long long total = (long long)n_points * kpad;
  const int nf3 = 3 * num_freqs;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(i % kpad);
    const long long pt = i / kpad;
    const float* x = q + pt * in_dim;
    float v = 0.f;
    if (col < 3) {
      v = x[col];
    } else if (col < 3 + 2 * nf3) {
      const int k = (col - 3) % nf3, c = k / num_freqs, f = k % num_freqs;
      float fr = (float)(1 << f);
      if (include_pi) fr *= 3.14159265358979323846f;
      const float a = x[c] * fr;
      v = (col < 3 + nf3) ? sinf(a) : cosf(a);
    } else if (col < 3 + 2 * nf3 + extra) {
      v = x[3 + (col - 3 - 2 * nf3)];
    }
    out[i] = v;
  }
}

// ---- split-bf16 ("3x bf16") operands for the fp32-grade GEMMs of the Stage-II query path ------------------------------
// x = hi + lo with hi = bf16(x), lo = bf16(x - hi) (|x - hi - lo| <= 2^-17 |x|).  A product a*w is evaluated on the tensor
// cores as a_hi*w_hi + a_lo*w_hi + a_hi*w_lo by concatenating along K: A-pattern [hi | lo | hi], W-pattern [hi | hi | lo].
// The source is cut in segments of `seg` columns; each becomes 3*seg destination columns (seg = cols for a plain GEMM
// operand, seg = head_dim for per-head attention operands).
__global__ void __launch_bounds__(256) split3_kernel(const float* __restrict__ src, long long ld_src, long long rows, int cols,
                                                     int seg, int w_pattern, __nv_bfloat16* __restrict__ dst, long long ld_dst) {
  const int c4 = cols >> 2;
  const long long total = rows * c4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / c4;
    const int c = (int)(i % c4) << 2;
    const float4 x = *reinterpret_cast<const float4*>(src + r * ld_src + c);
    const float xs[4] = {x.x, x.y, x.z, x.w};
    __nv_bfloat16 hi[4], lo[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      hi[j] = __float2bfloat16_rn(xs[j]);
      lo[j] = __float2bfloat16_rn(xs[j] - __bfloat162float(hi[j]));
    }
    const int s = c / seg, j0 = c % seg;
    __nv_bfloat16* d = dst + r * ld_dst + (long long)s * 3 * seg + j0;
    const uint2 vh = *reinterpret_cast<const uint2*>(hi), vl = *reinterpret_cast<const uint2*>(lo);
    *reinterpret_cast<uint2*>(d) = vh;
    *reinterpret_cast<uint2*>(d + seg) = w_pattern ? vh : vl;
    *reinterpret_cast<uint2*>(d + 2 * seg) = w_pattern ? vl : vh;
  }
}

// Row softmax of fp32 scores, written as the A-pattern split [P_hi | P_lo | P_hi] with each part n_pad wide and zeros in
// the padding columns [n, n_pad).  One 512-thread CTA per row, two sweeps and no shared-memory staging of the row (an
// earlier version staged the 131 KB row in shared memory, which capped occupancy at one CTA per SM): sweep 1 keeps a
// per-thread online (max, sum) pair, sweep 2 re-reads the row (4 CTAs/SM x 132 SMs x 131 KB = 69 MB of rows in flight
// against the 50 MB L2) and writes exp(x - max) / sum.
__global__ void __launch_bounds__(512, 4) softmax_split3_kernel(const float* __restrict__ s, long long ld_s, int n, int n_pad,
                                                                float scale, __nv_bfloat16* __restrict__ dst, long long ld_dst) {
  __shared__ float red_m[16], red_l[16];
  const float* src = s + (long long)blockIdx.x * ld_s;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float m = -INFINITY, l = 0.f;
  for (int c = tid * 4; c < n; c += blockDim.x * 4) {  // columns >= n (padding / ragged tail) never enter the statistics
    float4 x = *reinterpret_cast<const float4*>(src + c);
    x.x = x.x * scale;
    x.y = (c + 1 < n) ? x.y * scale : -INFINITY;
    x.z = (c + 2 < n) ? x.z * scale : -INFINITY;
    x.w = (c + 3 < n) ? x.w * scale : -INFINITY;
    const float m4 = fmaxf(fmaxf(x.x, x.y), fmaxf(x.z, x.w));
    if (m4 > m) {
      l *= expf(m - m4);  // m == -inf on the first visit: exp(-inf) == 0 and l == 0
      m = m4;
    }
    l += (expf(x.x - m) + expf(x.y - m)) + (expf(x.z - m) + expf(x.w - m));
  }
  // combine the (m, l) pairs of the CTA
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float mo = __shfl_xor_sync(0xffffffffu, m, o), lo = __shfl_xor_sync(0xffffffffu, l, o);
    const float mn = fmaxf(m, mo);
    l = (mn == -INFINITY) ? 0.f : l * expf(m - mn) + lo * expf(mo - mn);
    m = mn;
  }
  if (lane == 0) { red_m[warp] = m; red_l[warp] = l; }
  __syncthreads();
  float M = red_m[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) M = fmaxf(M, red_m[w]);
  float L = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) L += (red_m[w] == -INFINITY) ? 0.f : red_l[w] * expf(red_m[w] - M);
  const float inv = 1.0f / L;
  __nv_bfloat16* d = dst + (long long)blockIdx.x * ld_dst;
  for (int c = tid * 4; c < n_pad; c += blockDim.x * 4) {
    const float4 x = *reinterpret_cast<const float4*>(src + c);
    const float xs[4] = {x.x, x.y, x.z, x.w};
    __nv_bfloat16 hi[4], lo[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float p = (c + j < n) ? expf(xs[j] * scale - M) * inv : 0.f;
      hi[j] = __float2bfloat16_rn(p);
      lo[j] = __float2bfloat16_rn(p - __bfloat162float(hi[j]));
    }
    const uint2 vh = *reinterpret_cast<const uint2*>(hi), vl = *reinterpret_cast<const uint2*>(lo);
    *reinterpret_cast<uint2*>(d + c) = vh;
    *reinterpret_cast<uint2*>(d + n_pad + c) = vl;
    *reinterpret_cast<uint2*>(d + 2 * n_pad + c) = vh;
  }
}

// Stage II output head: displacement = 2 * sigmoid(-logit) - 1 on the first `out_dim` columns (temporal_autoencoder.py:160,269)
__global__ void __launch_bounds__(256) displacement_out_kernel(const float* __restrict__ logits, long long ld, int n_points,
                                                               int out_dim, float* __restrict__ out) {
  const long long total = (long long)n_points * out_dim;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long pt = i / out_dim;
    const int c = (int)(i % out_dim);
    const float x = -logits[pt * ld + c];
    out[i] = 2.0f / (1.0f + expf(-x)) - 1.0f;
  }
}

static int grid_for(long long work_items, int block) {
  long long g = (work_items + block - 1) / block;
  const long long cap = (long long)num_sms() * 16;  // grid-stride loops; a few waves of resident CTAs
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace amb

using namespace amb;

extern "C" {

int amb_cfg_euler_step(float* latents, const void* pred_bf16, int n_branches, const float* scales_host,
                       float dt_signed, const uint8_t* frame_update, int n_frames, int64_t n_per_frame,
                       int64_t branch_stride, int64_t frame_stride, int64_t frame_offset, amb_stream_t stream) {
  AMB_CHECK_ARG(latents && pred_bf16 && frame_update, "cfg_euler_step: null pointer");
  AMB_CHECK_ARG(n_branches >= 1 && n_branches <= kMaxBranches, "cfg_euler_step: n_branches %d not in [1,%d]", n_branches, kMaxBranches);
  AMB_CHECK_ARG(n_branches == 1 || scales_host, "cfg_euler_step: scales required");
  AMB_CHECK_ARG(n_per_frame % 8 == 0 && frame_stride % 8 == 0 && frame_offset % 8 == 0 && branch_stride % 8 == 0,
                "cfg_euler_step: sizes/strides must be multiples of 8 elements");
  AMB_CHECK_ARG((reinterpret_cast<uintptr_t>(latents) & 15) == 0 && (reinterpret_cast<uintptr_t>(pred_bf16) & 15) == 0,
                "cfg_euler_step: pointers must be 16-byte aligned");
  if (n_frames <= 0 || n_per_frame <= 0) return AMB_OK;
  CfgEulerParams p;
  p.latents = latents;
  p.pred = reinterpret_cast<const __nv_bfloat16*>(pred_bf16);
  p.frame_update = frame_update;
  for (int i = 0; i < kMaxBranches; ++i) p.scales[i] = (i < n_branches - 1) ? scales_host[i] : 0.f;
  p.dt = dt_signed;
  p.n_branches = n_branches;
  p.n_frames = n_frames;
  p.n_per_frame = n_per_frame;
  p.branch_stride = branch_stride;
  p.frame_stride = frame_stride;
  p.frame_offset = frame_offset;
  const long long vecs = (n_per_frame >> 3) * (long long)n_frames;
  cfg_euler_kernel<<<grid_for(vecs, 256), 256, 0, (cudaStream_t)stream>>>(p);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_layernorm(const void* x, int x_fp32, int64_t ldx, const float* gamma, const float* beta, void* y, int y_fp32,
                  int64_t ldy, int64_t rows, int cols, float eps, amb_stream_t stream) {
  AMB_CHECK_ARG(x && gamma && beta && y, "layernorm: null pointer");
  AMB_CHECK_ARG(ldx % 8 == 0 && ldy % 8 == 0, "layernorm: row strides must be multiples of 8 elements");
  if (rows <= 0) return AMB_OK;
  const int wpb = 8;
  dim3 grid((unsigned)((rows + wpb - 1) / wpb)), block(wpb * 32);
  cudaStream_t s = (cudaStream_t)stream;
#define AMB_LN_CASE(C)                                                                                                   \
  case C:                                                                                                                \
    if (x_fp32 && y_fp32) layernorm_kernel<C, true, true><<<grid, block, 0, s>>>(x, ldx, gamma, beta, y, ldy, rows, eps);  \
    else if (x_fp32) layernorm_kernel<C, true, false><<<grid, block, 0, s>>>(x, ldx, gamma, beta, y, ldy, rows, eps);      \
    else if (y_fp32) layernorm_kernel<C, false, true><<<grid, block, 0, s>>>(x, ldx, gamma, beta, y, ldy, rows, eps);      \
    else layernorm_kernel<C, false, false><<<grid, block, 0, s>>>(x, ldx, gamma, beta, y, ldy, rows, eps);                 \
    break;
  switch (cols) {
    AMB_LN_CASE(256)
    AMB_LN_CASE(512)
    AMB_LN_CASE(1024)
    AMB_LN_CASE(2048)
    AMB_LN_CASE(4096)
    default:
      set_last_error("layernorm: unsupported cols %d (256/512/1024/2048/4096)", cols);
      return AMB_ERR_UNSUPPORTED;
  }
#undef AMB_LN_CASE
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_patchify(const float* pixels, void* out_bf16, int n_images, int height, int width, int patch, int kpad,
                 amb_stream_t stream) {
  AMB_CHECK_ARG(pixels && out_bf16, "patchify: null pointer");
  AMB_CHECK_ARG(patch > 0 && height % patch == 0 && width % patch == 0 && kpad >= 3 * patch * patch && kpad % 64 == 0,
                "patchify: bad geometry h=%d w=%d p=%d kpad=%d", height, width, patch, kpad);
  if (n_images <= 0) return AMB_OK;
  const long long total = (long long)n_images * (height / patch) * (width / patch) * kpad;
  patchify_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(pixels, reinterpret_cast<__nv_bfloat16*>(out_bf16),
                                                                           n_images, height, width, patch, kpad);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_alpha_rows(float source_alpha, float target_alpha, int size, float* out, int64_t row_stride, int n_rows,
                   amb_stream_t stream) {
  AMB_CHECK_ARG(out && size > 0 && size % 2 == 0, "alpha_rows: bad arguments");
  if (n_rows <= 0) return AMB_OK;
  alpha_rows_kernel<<<n_rows, 256, 0, (cudaStream_t)stream>>>(source_alpha, target_alpha, size, out, row_stride, n_rows);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_split3_bf16(const float* src, int64_t ld_src, int64_t rows, int cols, int seg, int w_pattern, void* dst_bf16,
                    int64_t ld_dst, amb_stream_t stream) {
  AMB_CHECK_ARG(src && dst_bf16, "split3: null pointer");
  AMB_CHECK_ARG(cols > 0 && seg > 0 && cols % seg == 0 && seg % 4 == 0 && ld_src % 4 == 0 && ld_dst % 4 == 0 &&
                    ld_dst >= 3LL * cols && ld_src >= cols,
                "split3: bad geometry cols=%d seg=%d ld_src=%lld ld_dst=%lld", cols, seg, (long long)ld_src, (long long)ld_dst);
  // the kernel reads float4 and writes 4-element bf16 vectors (uint2)
  AMB_CHECK_ARG((reinterpret_cast<uintptr_t>(src) & 15) == 0, "split3: src must be 16-byte aligned");
  AMB_CHECK_ARG((reinterpret_cast<uintptr_t>(dst_bf16) & 7) == 0, "split3: dst must be 8-byte aligned");
  if (rows <= 0) return AMB_OK;
  split3_kernel<<<grid_for(rows * (cols / 4), 256), 256, 0, (cudaStream_t)stream>>>(
      src, ld_src, rows, cols, seg, w_pattern, reinterpret_cast<__nv_bfloat16*>(dst_bf16), ld_dst);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_softmax_split3(const float* scores, int64_t ld_s, int rows, int n, int n_pad, float scale, void* dst_bf16,
                       int64_t ld_dst, amb_stream_t stream) {
  AMB_CHECK_ARG(scores && dst_bf16, "softmax_split3: null pointer");
  AMB_CHECK_ARG(n > 0 && n_pad >= n && n_pad % 4 == 0 && ld_s % 4 == 0 && ld_s >= n_pad && ld_dst % 4 == 0 && ld_dst >= 3LL * n_pad,
                "softmax_split3: bad geometry n=%d n_pad=%d", n, n_pad);
  AMB_CHECK_ARG((reinterpret_cast<uintptr_t>(scores) & 15) == 0, "softmax_split3: scores must be 16-byte aligned");
  AMB_CHECK_ARG((reinterpret_cast<uintptr_t>(dst_bf16) & 7) == 0, "softmax_split3: dst must be 8-byte aligned");
  if (rows <= 0) return AMB_OK;
  softmax_split3_kernel<<<rows, 512, 0, (cudaStream_t)stream>>>(scores, ld_s, n, n_pad, scale,
                                                                  reinterpret_cast<__nv_bfloat16*>(dst_bf16), ld_dst);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_point_embedding(const float* points, int n_points, int in_dim, int extra, int num_freqs, int include_pi,
                        float* out, int kpad, amb_stream_t stream) {
  AMB_CHECK_ARG(points && out, "point_embedding: null pointer");
  AMB_CHECK_ARG(in_dim == 3 + extra && kpad % 64 == 0 && kpad >= 3 + 6 * num_freqs + extra && num_freqs >= 0 && num_freqs < 24,
                "point_embedding: bad geometry in_dim=%d extra=%d freqs=%d kpad=%d", in_dim, extra, num_freqs, kpad);
  if (n_points <= 0) return AMB_OK;
  point_embedding_kernel<<<grid_for((long long)n_points * kpad, 256), 256, 0, (cudaStream_t)stream>>>(
      points, n_points, in_dim, extra, num_freqs, include_pi, out, kpad);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_displacement_out(const float* logits, int64_t ld, int n_points, int out_dim, float* out, amb_stream_t stream) {
  AMB_CHECK_ARG(logits && out && out_dim > 0 && ld >= out_dim, "displacement_out: bad arguments");
  if (n_points <= 0) return AMB_OK;
  displacement_out_kernel<<<grid_for((long long)n_points * out_dim, 256), 256, 0, (cudaStream_t)stream>>>(logits, ld, n_points,
                                                                                                        out_dim, out);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_cast_f32_bf16(const float* src, void* dst_bf16, int64_t n, amb_stream_t stream) {
  AMB_CHECK_ARG(src && dst_bf16, "cast: null pointer");
  AMB_CHECK_ARG((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst_bf16) & 7) == 0, "cast: misaligned");
  if (n <= 0) return AMB_OK;
  cast_f32_bf16_kernel<<<grid_for((n + 3) / 4, 256), 256, 0, (cudaStream_t)stream>>>(src, reinterpret_cast<__nv_bfloat16*>(dst_bf16), n);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_timestep_embedding(const float* t, int n_t, const float* mask, int rows, int channels, void* out_bf16,
                           amb_stream_t stream) {
  AMB_CHECK_ARG(t && out_bf16 && n_t > 0, "timestep_embedding: null pointer");
  AMB_CHECK_ARG(channels % 2 == 0 && channels > 0, "timestep_embedding: channels must be even");
  if (rows <= 0) return AMB_OK;
  timestep_embedding_kernel<<<rows, 256, 0, (cudaStream_t)stream>>>(t, n_t, mask, rows, channels, reinterpret_cast<__nv_bfloat16*>(out_bf16));
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_add_bias_rows(void* y, int y_fp32, int64_t ldy, const float* bias, int64_t rows, int cols, amb_stream_t stream) {
  AMB_CHECK_ARG(y && bias, "add_bias_rows: null pointer");
  AMB_CHECK_ARG(cols % 8 == 0 && ldy % 8 == 0, "add_bias_rows: cols/ldy must be multiples of 8");
  if (rows <= 0) return AMB_OK;
  if (y_fp32)
    add_bias_rows_f32_kernel<<<grid_for(rows * (cols >> 2), 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<float*>(y), ldy, bias, rows, cols);
  else
    add_bias_rows_kernel<<<grid_for(rows * (cols >> 3), 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<__nv_bfloat16*>(y), ldy, bias, rows, cols);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

}  // extern "C"
