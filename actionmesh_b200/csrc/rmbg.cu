// Background removal (RMBG-1.4, actionmesh/preprocessing/background_removal.py): every kernel of the network except the
// convolutions' tensor-core work, which runs on amb_gemm_bf16 with split-bf16 operands (DESIGN §17).
//  - resize_input   : uint8 RGB frame -> bilinear to the model input size, /255, -0.5 (fp32 NHWC)     (:57-69)
//  - im2col_split   : 3x3 patches of up to two fp32 NHWC sources (the decoder's torch.cat) written as split3's
//                     activation layout [hi | lo | hi] (briarmbg.py REBNCONV / conv_in)
//  - maxpool2       : MaxPool2d(2, 2, ceil_mode=True)
//  - upsample       : F.interpolate(bilinear, align_corners=False) to any size (_upsample_like)
//  - mask head      : side1 (3x3, 64 -> 1) in fp32, upsample + sigmoid, resize to the frame, min-max, uint8 (:71-82, :104-106)
//  - refine + rgba  : Otsu as OpenCV computes it, 8-connected labelling, remove_small_objects, alpha write (:20-38, :111)
// Activations are fp32 NHWC with a pixel stride that may exceed the channel count (GEMM outputs padded to 64 columns).
// The bilinear kernels round every fp32 operation on its own (no FMA contraction), in the order tests/rmbg_ref.py restates.
#include "common.cuh"
#include "../../include/actionmesh_b200.h"

#include <cuda_bf16.h>
#include <cfloat>

namespace amb {
namespace rmbg {

int rmbg_grid(long long items, int block) {
  long long g = (items + block - 1) / block;
  const long long cap = (long long)num_sms() * 32;  // grid-stride loops
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

// ---- bilinear, align_corners=False (PyTorch's upsample_bilinear2d: scale = in / out in fp32) ---------------------------
struct Tap {
  int i0, i1;   // source indices (i1 = i0 + 1, or i0 at the last row / column)
  float l0, l1; // weights 1 - lambda, lambda
};

__device__ __forceinline__ Tap bilinear_tap(float scale, int dst, int in_size) {
  float src = __fsub_rn(__fmul_rn(scale, __fadd_rn((float)dst, 0.5f)), 0.5f);
  if (src < 0.f) src = 0.f;
  Tap t;
  t.i0 = (int)src;
  t.i1 = t.i0 + (t.i0 < in_size - 1 ? 1 : 0);
  t.l1 = __fsub_rn(src, (float)t.i0);
  t.l0 = __fsub_rn(1.0f, t.l1);
  return t;
}

// h0 (w0 x00 + w1 x01) + h1 (w0 x10 + w1 x11), each product and sum rounded on its own
__device__ __forceinline__ float bilinear_mix(const Tap& ty, const Tap& tx, float x00, float x01, float x10, float x11) {
  const float top = __fadd_rn(__fmul_rn(tx.l0, x00), __fmul_rn(tx.l1, x01));
  const float bot = __fadd_rn(__fmul_rn(tx.l0, x10), __fmul_rn(tx.l1, x11));
  return __fadd_rn(__fmul_rn(ty.l0, top), __fmul_rn(ty.l1, bot));
}

__device__ __forceinline__ float sigmoidf_rn(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }

__global__ void __launch_bounds__(256) resize_input_kernel(const uint8_t* __restrict__ rgb, int h, int w, float* __restrict__ out,
                                                           int oh, int ow, float sy, float sx) {
  const long long total = (long long)oh * ow;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int oy = (int)(i / ow), ox = (int)(i % ow);
    const Tap ty = bilinear_tap(sy, oy, h), tx = bilinear_tap(sx, ox, w);
    const uint8_t* r0 = rgb + (long long)ty.i0 * w * 3;
    const uint8_t* r1 = rgb + (long long)ty.i1 * w * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = bilinear_mix(ty, tx, (float)r0[tx.i0 * 3 + c], (float)r0[tx.i1 * 3 + c], (float)r1[tx.i0 * 3 + c],
                                   (float)r1[tx.i1 * 3 + c]);
      out[i * 3 + c] = __fsub_rn(__fdiv_rn(v, 255.0f), 0.5f);
    }
  }
}

__global__ void __launch_bounds__(256) upsample_kernel(const float* __restrict__ src, long long ps_src, int h, int w, int c,
                                                       float* __restrict__ dst, long long ps_dst, int oh, int ow, float sy,
                                                       float sx) {
  const long long total = (long long)oh * ow * c;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long px = i / c;
    const int ch = (int)(i - px * c);
    const int oy = (int)(px / ow), ox = (int)(px % ow);
    const Tap ty = bilinear_tap(sy, oy, h), tx = bilinear_tap(sx, ox, w);
    const float* r0 = src + (long long)ty.i0 * w * ps_src + ch;
    const float* r1 = src + (long long)ty.i1 * w * ps_src + ch;
    dst[px * ps_dst + ch] = bilinear_mix(ty, tx, r0[tx.i0 * ps_src], r0[tx.i1 * ps_src], r1[tx.i0 * ps_src], r1[tx.i1 * ps_src]);
  }
}

// ---- im2col -> split operand -------------------------------------------------------------------------------------------
// Row (oy, ox), column k = (ky * 3 + kx) * (c0 + c1) + c with c < c0 from src0 and the rest from src1; columns >= 9 (c0 + c1)
// are zero.  Each value x is written as hi = bf16(x) at k, lo = bf16(x - hi) at k_pad + k and hi again at 2 k_pad + k,
// which is ops.split3(im2col, seg=k_pad) element for element.
__global__ void __launch_bounds__(256) im2col_split_kernel(const float* __restrict__ src0, int c0, long long ps0,
                                                           const float* __restrict__ src1, int c1, long long ps1, int h, int w,
                                                           int oh, int ow, int stride, int pad, int dil, int k_pad,
                                                           __nv_bfloat16* __restrict__ dst, long long ld_dst) {
  const int ct = c0 + c1, k = 9 * ct;
  const long long total = (long long)oh * ow * k_pad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / k_pad;
    const int col = (int)(i - row * k_pad);
    float x = 0.f;
    if (col < k) {
      const int tap = col / ct, c = col - tap * ct;
      const int oy = (int)(row / ow), ox = (int)(row - (long long)oy * ow);
      const int iy = oy * stride - pad + (tap / 3) * dil, ix = ox * stride - pad + (tap % 3) * dil;
      if (iy >= 0 && iy < h && ix >= 0 && ix < w) {
        const long long p = (long long)iy * w + ix;
        x = c < c0 ? src0[p * ps0 + c] : src1[p * ps1 + (c - c0)];
      }
    }
    const __nv_bfloat16 hi = __float2bfloat16_rn(x);
    const __nv_bfloat16 lo = __float2bfloat16_rn(x - __bfloat162float(hi));
    __nv_bfloat16* d = dst + row * ld_dst + col;
    d[0] = hi;
    d[k_pad] = lo;
    d[2 * k_pad] = hi;
  }
}

// ---- MaxPool2d(2, stride 2, ceil_mode=True): a partial last window takes the max of its valid elements; NaN propagates --
__global__ void __launch_bounds__(256) maxpool2_kernel(const float* __restrict__ src, long long ps_src, int h, int w, int c,
                                                       float* __restrict__ dst, long long ps_dst, int oh, int ow) {
  const long long total = (long long)oh * ow * c;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long px = i / c;
    const int ch = (int)(i - px * c);
    const int oy = (int)(px / ow), ox = (int)(px % ow);
    float m = -INFINITY;
    for (int dy = 0; dy < 2; ++dy) {
      const int y = 2 * oy + dy;
      if (y >= h) break;
      for (int dx = 0; dx < 2; ++dx) {
        const int x = 2 * ox + dx;
        if (x >= w) break;
        const float v = src[((long long)y * w + x) * ps_src + ch];
        if (v > m || isnan(v)) m = v;
      }
    }
    dst[px * ps_dst + ch] = m;
  }
}

// ---- mask head ------------------------------------------------------------------------------------------------------------
// side1: 3x3, 64 -> 1, padding 1, bias; weight = 576 fp32 in (ky, kx, c) order followed by the bias.  fp32 sum in that order.
__global__ void __launch_bounds__(256) side1_kernel(const float* __restrict__ feat, long long ps, int h, int w,
                                                   const float* __restrict__ weight, float* __restrict__ logits) {
  __shared__ float sw[577];
  for (int j = threadIdx.x; j < 577; j += blockDim.x) sw[j] = weight[j];
  __syncthreads();
  const long long total = (long long)h * w;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(i / w), x = (int)(i % w);
    float acc = 0.f;
    for (int t = 0; t < 9; ++t) {
      const int iy = y - 1 + t / 3, ix = x - 1 + t % 3;
      if (iy < 0 || iy >= h || ix < 0 || ix >= w) continue;
      const float4* f = reinterpret_cast<const float4*>(feat + ((long long)iy * w + ix) * ps);
      const float* wt = sw + t * 64;
#pragma unroll 4
      for (int c4 = 0; c4 < 16; ++c4) {
        const float4 v = f[c4];
        acc = fmaf(v.x, wt[4 * c4 + 0], acc);
        acc = fmaf(v.y, wt[4 * c4 + 1], acc);
        acc = fmaf(v.z, wt[4 * c4 + 2], acc);
        acc = fmaf(v.w, wt[4 * c4 + 3], acc);
      }
    }
    logits[i] = acc + sw[576];
  }
}

__global__ void __launch_bounds__(256) upsample_sigmoid_kernel(const float* __restrict__ logits, int h, int w,
                                                               float* __restrict__ soft, int oh, int ow, float sy, float sx) {
  const long long total = (long long)oh * ow;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int oy = (int)(i / ow), ox = (int)(i % ow);
    const Tap ty = bilinear_tap(sy, oy, h), tx = bilinear_tap(sx, ox, w);
    const float* r0 = logits + (long long)ty.i0 * w;
    const float* r1 = logits + (long long)ty.i1 * w;
    soft[i] = sigmoidf_rn(bilinear_mix(ty, tx, r0[tx.i0], r0[tx.i1], r1[tx.i0], r1[tx.i1]));
  }
}

// order-preserving uint32 key of a float: larger float, larger key
__device__ __forceinline__ uint32_t float_key(float v) {
  const uint32_t b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// resized = bilinear(soft) at the frame size; minmax[0] = ~key(min), minmax[1] = key(max) (both zeroed before the launch)
__global__ void __launch_bounds__(256) resize_minmax_kernel(const float* __restrict__ soft, int h, int w,
                                                            float* __restrict__ resized, int oh, int ow, float sy, float sx,
                                                            uint32_t* __restrict__ minmax) {
  uint32_t kmin = 0xffffffffu, kmax = 0u;
  const long long total = (long long)oh * ow;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int oy = (int)(i / ow), ox = (int)(i % ow);
    const Tap ty = bilinear_tap(sy, oy, h), tx = bilinear_tap(sx, ox, w);
    const float* r0 = soft + (long long)ty.i0 * w;
    const float* r1 = soft + (long long)ty.i1 * w;
    const float v = bilinear_mix(ty, tx, r0[tx.i0], r0[tx.i1], r1[tx.i0], r1[tx.i1]);
    resized[i] = v;
    const uint32_t k = float_key(v);
    kmin = min(kmin, k);
    kmax = max(kmax, k);
  }
  for (int o = 16; o; o >>= 1) {
    kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, o));
    kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMax(&minmax[0], ~kmin);
    atomicMax(&minmax[1], kmax);
  }
}

// uint8((r - mi) / (ma - mi) * 255), truncated as numpy's astype(uint8) does; all zero when ma == mi (the reference
// divides by zero there)
__global__ void __launch_bounds__(256) mask_u8_kernel(const float* __restrict__ resized, long long n,
                                                      const uint32_t* __restrict__ minmax, uint8_t* __restrict__ mask) {
  const float mi = key_float(~minmax[0]), ma = key_float(minmax[1]);
  const float range = __fsub_rn(ma, mi);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    uint8_t u = 0;
    if (ma != mi) {
      const float v = __fmul_rn(__fdiv_rn(__fsub_rn(resized[i], mi), range), 255.0f);
      u = (uint8_t)__float2int_rz(v);
    }
    mask[i] = u;
  }
}

// ---- refinement --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) histogram_kernel(const uint8_t* __restrict__ mask, long long n, int32_t* __restrict__ hist) {
  __shared__ int32_t sh[256];
  sh[threadIdx.x] = 0;
  __syncthreads();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    atomicAdd(&sh[mask[i]], 1);
  __syncthreads();
  if (sh[threadIdx.x]) atomicAdd(&hist[threadIdx.x], sh[threadIdx.x]);
}

// cv2.threshold(THRESH_OTSU)'s threshold in double precision (DESIGN §17); hist[256] = t
__global__ void otsu_kernel(int32_t* hist, long long n) {
  if (threadIdx.x != 0) return;
  const double scale = 1.0 / (double)n;
  double mu = 0.0;
  for (int i = 0; i < 256; ++i) mu += i * (double)hist[i];
  mu *= scale;
  double q1 = 0.0, mu1 = 0.0, max_sigma = 0.0;
  int t = 0;
  for (int i = 0; i < 256; ++i) {
    const double p = hist[i] * scale;
    mu1 *= q1;
    q1 += p;
    const double q2 = 1.0 - q1;
    if (fmin(q1, q2) < FLT_EPSILON || fmax(q1, q2) > 1.0 - FLT_EPSILON) continue;
    mu1 = (mu1 + i * p) / q1;
    const double mu2 = (mu - q1 * mu1) / q2;
    const double sigma = q1 * q2 * (mu1 - mu2) * (mu1 - mu2);
    if (sigma > max_sigma) {
      max_sigma = sigma;
      t = i;
    }
  }
  hist[256] = t;
}

// foreground (mask > t) pixels start as their own root; sizes are cleared for the count
__global__ void __launch_bounds__(256) label_init_kernel(const uint8_t* __restrict__ mask, long long n, const int32_t* __restrict__ hist,
                                                         int32_t* __restrict__ labels, int32_t* __restrict__ sizes) {
  const int t = hist[256];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    labels[i] = mask[i] > t ? (int32_t)i : -1;
    sizes[i] = 0;
  }
}

__device__ __forceinline__ int find_root(const int32_t* labels, int x) {
  const volatile int32_t* l = labels;
  int p = l[x];
  while (p != x) {
    x = p;
    p = l[x];
  }
  return x;
}

// hook the larger root under the smaller with atomicMin; when the larger one stopped being a root in the meantime, its new
// parent still has to be joined with the smaller root, so go round again.  Labels only decrease, so every root is the
// smallest pixel index of its tree and the final forest does not depend on scheduling.
__device__ __forceinline__ void unite(int32_t* labels, int a, int b) {
  while (true) {
    a = find_root(labels, a);
    b = find_root(labels, b);
    if (a == b) return;
    if (a < b) {
      const int t = a;
      a = b;
      b = t;
    }
    const int old = atomicMin(&labels[a], b);
    if (old == a) return;
    a = old;
  }
}

// 8-connectivity: each foreground pixel joins its W, NW, N and NE foreground neighbours
__global__ void __launch_bounds__(256) label_union_kernel(int h, int w, int32_t* labels) {
  const long long n = (long long)h * w;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (labels[i] < 0) continue;
    const int y = (int)(i / w), x = (int)(i % w);
    if (x > 0 && labels[i - 1] >= 0) unite(labels, (int)i, (int)i - 1);
    if (y > 0) {
      const long long up = i - w;
      if (x > 0 && labels[up - 1] >= 0) unite(labels, (int)i, (int)up - 1);
      if (labels[up] >= 0) unite(labels, (int)i, (int)up);
      if (x + 1 < w && labels[up + 1] >= 0) unite(labels, (int)i, (int)up + 1);
    }
  }
}

__global__ void __launch_bounds__(256) label_count_kernel(long long n, int32_t* labels, int32_t* __restrict__ sizes) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (labels[i] < 0) continue;
    const int r = find_root(labels, (int)i);
    labels[i] = r;
    atomicAdd(&sizes[r], 1);
  }
}

// RGB copy + alpha: refined (a component of >= min_size pixels) or the uint8 soft mask as is
__global__ void __launch_bounds__(256) rgba_kernel(const uint8_t* __restrict__ rgb, const uint8_t* __restrict__ mask, long long n,
                                                   const int32_t* __restrict__ labels, const int32_t* __restrict__ sizes,
                                                   int min_size, uint8_t* __restrict__ rgba) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    uint8_t a;
    if (labels) {
      const int r = labels[i];
      a = (r >= 0 && sizes[r] >= min_size) ? 255 : 0;
    } else {
      a = mask[i];
    }
    const uchar4 v = make_uchar4(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2], a);
    *reinterpret_cast<uchar4*>(rgba + 4 * i) = v;
  }
}

bool aligned(const void* p, int bytes) { return (reinterpret_cast<uintptr_t>(p) % bytes) == 0; }

// output size of a 3x3 convolution / the largest image side the kernels index with int
int conv_out(int in, int stride, int pad, int dil) { return (in + 2 * pad - 2 * dil - 1) / stride + 1; }
constexpr long long kMaxPixels = 1LL << 30;

}  // namespace rmbg
}  // namespace amb

using namespace amb;
using namespace amb::rmbg;

extern "C" {

int amb_rmbg_resize_input(const uint8_t* rgb, int height, int width, float* out, int out_height, int out_width,
                          amb_stream_t stream) {
  AMB_CHECK_ARG(rgb && out, "rmbg_resize_input: null pointer");
  AMB_CHECK_ARG(aligned(out, 4), "rmbg_resize_input: out must be 4-byte aligned");
  AMB_CHECK_ARG(height > 0 && width > 0 && out_height > 0 && out_width > 0 && (long long)height * width <= kMaxPixels &&
                    (long long)out_height * out_width <= kMaxPixels,
                "rmbg_resize_input: bad sizes %dx%d -> %dx%d", height, width, out_height, out_width);
  const long long total = (long long)out_height * out_width;
  resize_input_kernel<<<rmbg_grid(total, 256), 256, 0, (cudaStream_t)stream>>>(
      rgb, height, width, out, out_height, out_width, (float)height / (float)out_height, (float)width / (float)out_width);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_rmbg_im2col_split(const float* src0, int c0, int64_t ps0, const float* src1, int c1, int64_t ps1, int height, int width,
                          int stride, int pad, int dilation, int k_pad, void* dst_bf16, int64_t ld_dst, amb_stream_t stream) {
  AMB_CHECK_ARG(src0 && dst_bf16 && (c1 == 0 || src1), "rmbg_im2col_split: null pointer");
  AMB_CHECK_ARG(aligned(src0, 4) && aligned(src1, 4) && aligned(dst_bf16, 2), "rmbg_im2col_split: misaligned pointer");
  AMB_CHECK_ARG(c0 > 0 && c1 >= 0 && ps0 >= c0 && (c1 == 0 || ps1 >= c1), "rmbg_im2col_split: bad channels c0=%d (stride %lld) c1=%d (stride %lld)",
                c0, (long long)ps0, c1, (long long)ps1);
  AMB_CHECK_ARG(height > 0 && width > 0 && (long long)height * width <= kMaxPixels, "rmbg_im2col_split: bad size %dx%d", height, width);
  AMB_CHECK_ARG((stride == 1 || stride == 2) && dilation >= 1 && pad >= 0 && pad <= dilation,
                "rmbg_im2col_split: bad stride %d / padding %d / dilation %d", stride, pad, dilation);
  AMB_CHECK_ARG(k_pad > 0 && k_pad % 64 == 0 && 9LL * (c0 + c1) <= k_pad && ld_dst >= 3LL * k_pad,
                "rmbg_im2col_split: bad k_pad %d for %d channels (ld_dst %lld)", k_pad, c0 + c1, (long long)ld_dst);
  const int oh = conv_out(height, stride, pad, dilation), ow = conv_out(width, stride, pad, dilation);
  AMB_CHECK_ARG(oh > 0 && ow > 0, "rmbg_im2col_split: %dx%d is too small for dilation %d", height, width, dilation);
  const long long total = (long long)oh * ow * k_pad;
  im2col_split_kernel<<<rmbg_grid(total, 256), 256, 0, (cudaStream_t)stream>>>(
      src0, c0, ps0, src1, c1, ps1, height, width, oh, ow, stride, pad, dilation, k_pad,
      reinterpret_cast<__nv_bfloat16*>(dst_bf16), ld_dst);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_rmbg_maxpool2(const float* src, int64_t ps_src, int height, int width, int channels, float* dst, int64_t ps_dst,
                      amb_stream_t stream) {
  AMB_CHECK_ARG(src && dst, "rmbg_maxpool2: null pointer");
  AMB_CHECK_ARG(aligned(src, 4) && aligned(dst, 4), "rmbg_maxpool2: misaligned pointer");
  AMB_CHECK_ARG(height > 0 && width > 0 && (long long)height * width <= kMaxPixels && channels > 0 && ps_src >= channels &&
                    ps_dst >= channels,
                "rmbg_maxpool2: bad geometry %dx%dx%d (strides %lld, %lld)", height, width, channels, (long long)ps_src,
                (long long)ps_dst);
  const int oh = (height + 1) / 2, ow = (width + 1) / 2;
  const long long total = (long long)oh * ow * channels;
  maxpool2_kernel<<<rmbg_grid(total, 256), 256, 0, (cudaStream_t)stream>>>(src, ps_src, height, width, channels, dst, ps_dst, oh, ow);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_rmbg_upsample(const float* src, int64_t ps_src, int height, int width, int channels, float* dst, int64_t ps_dst,
                      int out_height, int out_width, amb_stream_t stream) {
  AMB_CHECK_ARG(src && dst, "rmbg_upsample: null pointer");
  AMB_CHECK_ARG(aligned(src, 4) && aligned(dst, 4), "rmbg_upsample: misaligned pointer");
  AMB_CHECK_ARG(height > 0 && width > 0 && out_height > 0 && out_width > 0 && (long long)height * width <= kMaxPixels &&
                    (long long)out_height * out_width <= kMaxPixels && channels > 0 && ps_src >= channels && ps_dst >= channels,
                "rmbg_upsample: bad geometry %dx%dx%d -> %dx%d (strides %lld, %lld)", height, width, channels, out_height,
                out_width, (long long)ps_src, (long long)ps_dst);
  const long long total = (long long)out_height * out_width * channels;
  upsample_kernel<<<rmbg_grid(total, 256), 256, 0, (cudaStream_t)stream>>>(
      src, ps_src, height, width, channels, dst, ps_dst, out_height, out_width, (float)height / (float)out_height,
      (float)width / (float)out_width);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_rmbg_mask_head(const float* feat, int64_t ps, int height, int width, const float* weight, float* logits, int model_height,
                       int model_width, float* soft, int out_height, int out_width, float* resized, int32_t* minmax,
                       uint8_t* mask, amb_stream_t stream) {
  AMB_CHECK_ARG(feat && weight && logits && soft && resized && minmax && mask, "rmbg_mask_head: null pointer");
  AMB_CHECK_ARG(aligned(feat, 16) && aligned(weight, 4) && aligned(logits, 4) && aligned(soft, 4) && aligned(resized, 4) &&
                    aligned(minmax, 4),
                "rmbg_mask_head: misaligned pointer (feat needs 16 bytes, the rest 4)");
  AMB_CHECK_ARG(ps >= 64 && ps % 4 == 0, "rmbg_mask_head: the 64-channel features need a pixel stride >= 64, multiple of 4 (got %lld)",
                (long long)ps);
  AMB_CHECK_ARG(height > 0 && width > 0 && model_height > 0 && model_width > 0 && out_height > 0 && out_width > 0 &&
                    (long long)height * width <= kMaxPixels && (long long)model_height * model_width <= kMaxPixels &&
                    (long long)out_height * out_width <= kMaxPixels,
                "rmbg_mask_head: bad sizes %dx%d -> %dx%d -> %dx%d", height, width, model_height, model_width, out_height, out_width);
  cudaStream_t s = (cudaStream_t)stream;
  const long long n_feat = (long long)height * width, n_model = (long long)model_height * model_width;
  const long long n_out = (long long)out_height * out_width;
  side1_kernel<<<rmbg_grid(n_feat, 256), 256, 0, s>>>(feat, ps, height, width, weight, logits);
  AMB_CHECK_CUDA(cudaGetLastError());
  upsample_sigmoid_kernel<<<rmbg_grid(n_model, 256), 256, 0, s>>>(logits, height, width, soft, model_height, model_width,
                                                                  (float)height / (float)model_height,
                                                                  (float)width / (float)model_width);
  AMB_CHECK_CUDA(cudaGetLastError());
  AMB_CHECK_CUDA(cudaMemsetAsync(minmax, 0, 2 * sizeof(uint32_t), s));
  resize_minmax_kernel<<<rmbg_grid(n_out, 256), 256, 0, s>>>(soft, model_height, model_width, resized, out_height, out_width,
                                                             (float)model_height / (float)out_height,
                                                             (float)model_width / (float)out_width, reinterpret_cast<uint32_t*>(minmax));
  AMB_CHECK_CUDA(cudaGetLastError());
  mask_u8_kernel<<<rmbg_grid(n_out, 256), 256, 0, s>>>(resized, n_out, reinterpret_cast<const uint32_t*>(minmax), mask);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_rmbg_refine_rgba(const uint8_t* rgb, const uint8_t* mask, int height, int width, int refine, int min_size,
                         int32_t* hist, int32_t* labels, int32_t* sizes, uint8_t* rgba, amb_stream_t stream) {
  AMB_CHECK_ARG(rgb && mask && rgba && (!refine || (hist && labels && sizes)), "rmbg_refine_rgba: null pointer");
  AMB_CHECK_ARG(aligned(rgba, 4) && aligned(hist, 4) && aligned(labels, 4) && aligned(sizes, 4),
                "rmbg_refine_rgba: misaligned pointer (rgba, hist, labels and sizes need 4 bytes)");
  AMB_CHECK_ARG(height > 0 && width > 0 && (long long)height * width <= kMaxPixels, "rmbg_refine_rgba: bad size %dx%d", height, width);
  AMB_CHECK_ARG(refine == 0 || refine == 1, "rmbg_refine_rgba: refine must be 0 or 1");
  cudaStream_t s = (cudaStream_t)stream;
  const long long n = (long long)height * width;
  const int g = rmbg_grid(n, 256);
  if (refine) {
    AMB_CHECK_CUDA(cudaMemsetAsync(hist, 0, 257 * sizeof(int32_t), s));
    histogram_kernel<<<g, 256, 0, s>>>(mask, n, hist);
    AMB_CHECK_CUDA(cudaGetLastError());
    otsu_kernel<<<1, 32, 0, s>>>(hist, n);
    AMB_CHECK_CUDA(cudaGetLastError());
    label_init_kernel<<<g, 256, 0, s>>>(mask, n, hist, labels, sizes);
    AMB_CHECK_CUDA(cudaGetLastError());
    label_union_kernel<<<g, 256, 0, s>>>(height, width, labels);
    AMB_CHECK_CUDA(cudaGetLastError());
    label_count_kernel<<<g, 256, 0, s>>>(n, labels, sizes);
    AMB_CHECK_CUDA(cudaGetLastError());
  }
  rgba_kernel<<<g, 256, 0, s>>>(rgb, mask, n, refine ? labels : nullptr, sizes, min_size, rgba);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

}  // extern "C"
