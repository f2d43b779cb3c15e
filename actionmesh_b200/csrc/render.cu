// Multi-view normal rendering of a mesh: vertex normals, a binned z-buffer rasterizer and the normal-image compositor behind
// actionmesh_b200/render.py's B200MeshVisualizer.
//
// Replaces the reference's ActionMeshVisualizer (actionmesh/render/{visualizer,renderer,cameras,utils}.py), which runs
// PyTorch3D's naive rasterizer (bin_size=0, faces_per_pixel=1, blur_radius=0, perspective_correct, clip_barycentric_coords,
// no culling, no z clip) and soft_normal_shading.  DESIGN.md §16 states the contract; tests/render_ref.py restates it in
// numpy float32.  Every fp32 product, sum, difference, quotient and square root below is an explicit round-to-nearest
// intrinsic in the written order (the build does not pass --fmad=false, and an FMA would change the last bit), so the
// kernels reproduce the restatement bit for bit.
//
// Rasterization: each (camera, face) pair is set up by one thread: project, cull, and take the rectangle of samples its
// projected bounding box can reach.  A small rectangle is tested by that thread; a larger one, or any face that is not safely
// in front of the camera (it can then cover samples outside its projected box), goes to a list that whole CTAs work through.
// Both paths fold every covered sample into one 64-bit key (bits(depth) << 32 | face) with atomicMin, so the surviving face is
// the nearest one, ties go to the lower face index, and the result depends on neither the path nor the order.
#include <cuda_runtime.h>
#include <cstdint>
#include "common.cuh"
#include "scan.cuh"
#include "../../include/actionmesh_b200.h"

namespace amb {
namespace {

constexpr float kAreaEps = 1e-8f;      // zero-area test and denominator offsets (PyTorch3D kEpsilon)
constexpr float kClipEps = 1e-5f;      // clipped-barycentric normaliser floor
constexpr float kNormalEps = 1e-6f;    // vertex-normal normalisation floor (verts_normals_packed)
constexpr float kShadeEps = 1e-12f;    // F.normalize's default floor
constexpr float kBoxLimit = 64.0f;     // a face set up in front of the camera has every projected |x|, |y| below this
constexpr float kBoxPad = 1.0f / 1024; // NDC slack around a box: far above the rounding noise of the edge functions there
constexpr int kSmallSamples = 64;      // faces whose box holds at most this many samples are tested by their own thread
constexpr unsigned long long kEmpty = ~0ull;

__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fs(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fd(float a, float b) { return __fdiv_rn(a, b); }

struct P3 {
  float x, y, z;
};

__device__ __forceinline__ P3 load3(const float* p, long long i) { return {p[3 * i], p[3 * i + 1], p[3 * i + 2]}; }

// row vector times R (row-major 3x3) plus t: ((p.x R0j + p.y R1j) + p.z R2j) + t_j
__device__ __forceinline__ P3 transform(P3 p, const float* r, float t0, float t1, float t2) {
  return {fa(fa(fa(fm(p.x, r[0]), fm(p.y, r[3])), fm(p.z, r[6])), t0),
          fa(fa(fa(fm(p.x, r[1]), fm(p.y, r[4])), fm(p.z, r[7])), t1),
          fa(fa(fa(fm(p.x, r[2]), fm(p.y, r[5])), fm(p.z, r[8])), t2)};
}

// view space -> (f X / Z', f Y / Z', Z) with Z' = sign(Z) max(|Z|, 1e-8)
__device__ __forceinline__ P3 project(const float* cam, float focal, P3 w) {
  const P3 v = transform(w, cam, cam[9], cam[10], cam[11]);
  const float az = fabsf(v.z) > kAreaEps ? fabsf(v.z) : kAreaEps;
  const float zd = v.z < 0.0f ? -az : az;
  return {fd(fm(focal, v.x), zd), fd(fm(focal, v.y), zd), v.z};
}

// E(p, a, b) = (p.x - a.x)(b.y - a.y) - (p.y - a.y)(b.x - a.x)
__device__ __forceinline__ float edge(float px, float py, P3 a, P3 b) {
  return fs(fm(fs(px, a.x), fs(b.y, a.y)), fm(fs(py, a.y), fs(b.x, a.x)));
}

// NDC centre of sample index i on a side of n2 = 2S samples: 1 - (2i + 1) / 2S (+X left, +Y up, index 0 at +1)
__device__ __forceinline__ float sample_ndc(int i, int n2) { return fs(1.0f, fd((float)(2 * i + 1), (float)n2)); }

struct Face {
  P3 v0, v1, v2;
  bool live;     // not culled
  bool bounded;  // every depth > 0 and every |x|, |y| < kBoxLimit: only samples in [c0, c1] x [r0, r1] can be inside
  int c0, c1, r0, r1;
};

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// samples i with ndc(i) in [lo - pad, hi + pad]: ndc(i) = 1 - (2i+1)/2S, so i = (1 - ndc) S - 1/2, widened by floor/ceil
__device__ __forceinline__ void sample_range(float lo, float hi, int n2, int* i0, int* i1) {
  const float s = 0.5f * (float)n2;
  const float a = floorf((1.0f - (hi + kBoxPad)) * s - 0.5f), b = ceilf((1.0f - (lo - kBoxPad)) * s - 0.5f);
  *i0 = clampi((int)a, 0, n2 - 1);
  *i1 = clampi((int)b, -1, n2 - 1);
}

__device__ __forceinline__ Face face_setup(const float* verts, const int32_t* faces, int f, const float* cam, float focal, int n2) {
  Face s;
  s.v0 = project(cam, focal, load3(verts, faces[3LL * f]));
  s.v1 = project(cam, focal, load3(verts, faces[3LL * f + 1]));
  s.v2 = project(cam, focal, load3(verts, faces[3LL * f + 2]));
  const float area = edge(s.v0.x, s.v0.y, s.v1, s.v2);
  s.live = !(fabsf(area) <= kAreaEps) && !(s.v0.z < 0.0f && s.v1.z < 0.0f && s.v2.z < 0.0f);
  const float xmin = fminf(fminf(s.v0.x, s.v1.x), s.v2.x), xmax = fmaxf(fmaxf(s.v0.x, s.v1.x), s.v2.x);
  const float ymin = fminf(fminf(s.v0.y, s.v1.y), s.v2.y), ymax = fmaxf(fmaxf(s.v0.y, s.v1.y), s.v2.y);
  s.bounded = s.v0.z > 0.0f && s.v1.z > 0.0f && s.v2.z > 0.0f && xmin > -kBoxLimit && xmax < kBoxLimit &&
              ymin > -kBoxLimit && ymax < kBoxLimit;
  if (s.bounded) {
    sample_range(xmin, xmax, n2, &s.c0, &s.c1);
    sample_range(ymin, ymax, n2, &s.r0, &s.r1);
  } else {
    s.c0 = s.r0 = 0;
    s.c1 = s.r1 = n2 - 1;
  }
  return s;
}

struct Bary {
  float b0, b1, b2;
};

// perspective-corrected, clipped barycentrics of (px, py); false when the sample is not strictly inside
__device__ __forceinline__ bool barycentrics(const Face& s, float px, float py, Bary* out) {
  const float den = fa(edge(s.v2.x, s.v2.y, s.v0, s.v1), kAreaEps);
  const float w0 = fd(edge(px, py, s.v1, s.v2), den);
  const float w1 = fd(edge(px, py, s.v2, s.v0), den);
  const float w2 = fd(edge(px, py, s.v0, s.v1), den);
  const float t0 = fm(fm(w0, s.v1.z), s.v2.z), t1 = fm(fm(s.v0.z, w1), s.v2.z), t2 = fm(fm(s.v0.z, s.v1.z), w2);
  const float st = fa(fa(t0, t1), t2);
  const float dn = st > kAreaEps ? st : kAreaEps;
  const float p0 = fd(t0, dn), p1 = fd(t1, dn), p2 = fd(t2, dn);
  if (!(p0 > 0.0f && p1 > 0.0f && p2 > 0.0f)) return false;
  const float c0 = fmaxf(p0, 0.0f), c1 = fmaxf(p1, 0.0f), c2 = fmaxf(p2, 0.0f);
  const float sc = fa(fa(c0, c1), c2);
  const float dc = sc > kClipEps ? sc : kClipEps;
  *out = {fd(c0, dc), fd(c1, dc), fd(c2, dc)};
  return true;
}

// fold sample (r, c) into the z-buffer when the face covers it at a non-negative depth
__device__ __forceinline__ void test_sample(const Face& s, int f, int r, int c, int n2, unsigned long long* zbuf) {
  Bary b;
  if (!barycentrics(s, sample_ndc(c, n2), sample_ndc(r, n2), &b)) return;
  float pz = fa(fa(fm(b.b0, s.v0.z), fm(b.b1, s.v1.z)), fm(b.b2, s.v2.z));
  if (!(pz >= 0.0f)) return;  // behind the camera (or NaN)
  pz = pz == 0.0f ? 0.0f : pz;  // -0 -> +0
  const unsigned long long key = ((unsigned long long)__float_as_uint(pz) << 32) | (unsigned int)f;
  if (key < zbuf[(long long)r * n2 + c]) atomicMin(zbuf + (long long)r * n2 + c, key);
}

// one thread per (camera, face): set up, test a small box in place, queue anything larger as camera * F + face
__global__ void __launch_bounds__(256) raster_small_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces,
                                                           int n_faces, const float* __restrict__ cams, int n_cams, float focal,
                                                           int n2, unsigned long long* __restrict__ zbuf,
                                                           int32_t* __restrict__ queue) {
  const long long n = (long long)n_cams * n_faces;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int cam = (int)(i / n_faces), f = (int)(i % n_faces);
    const Face s = face_setup(verts, faces, f, cams + 12 * cam, focal, n2);
    if (!s.live || s.c1 < s.c0 || s.r1 < s.r0) continue;
    if (s.bounded && (s.c1 - s.c0 + 1) * (s.r1 - s.r0 + 1) <= kSmallSamples) {
      unsigned long long* zb = zbuf + (long long)cam * n2 * n2;
      for (int r = s.r0; r <= s.r1; ++r)
        for (int c = s.c0; c <= s.c1; ++c) test_sample(s, f, r, c, n2, zb);
    } else {
      queue[1 + atomicAdd(queue, 1)] = (int32_t)i;
    }
  }
}

// one CTA per queued (camera, face) at a time: each warp takes every eighth row of the face's box, its lanes the columns
__global__ void __launch_bounds__(256) raster_large_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces,
                                                           int n_faces, const float* __restrict__ cams, float focal, int n2,
                                                           unsigned long long* __restrict__ zbuf,
                                                           const int32_t* __restrict__ queue) {
  const int n = queue[0];
  for (int q = blockIdx.x; q < n; q += gridDim.x) {
    const int i = queue[1 + q];
    const int cam = i / n_faces, f = i % n_faces;
    const Face s = face_setup(verts, faces, f, cams + 12 * cam, focal, n2);
    unsigned long long* zb = zbuf + (long long)cam * n2 * n2;
    for (int r = s.r0 + (int)(threadIdx.x >> 5); r <= s.r1; r += (int)(blockDim.x >> 5))
      for (int c = s.c0 + (int)(threadIdx.x & 31); c <= s.c1; c += 32) test_sample(s, f, r, c, n2, zb);
  }
}

__global__ void resolve_kernel(const unsigned long long* __restrict__ zbuf, long long n, int32_t* __restrict__ pix_to_face) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = zbuf[i];
    pix_to_face[i] = k == kEmpty ? -1 : (int32_t)(unsigned int)(k & 0xffffffffu);
  }
}

// ---- vertex normals --------------------------------------------------------------------------------------------------------

// sum of cross(v1 - v0, v2 - v0) over the vertex's faces in ascending face order, then n / max(|n|, 1e-6)
__global__ void vertex_normals_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces, int n_vertices,
                                      const int32_t* __restrict__ off, const int32_t* __restrict__ vf,
                                      float* __restrict__ normals) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n_vertices; v += gridDim.x * blockDim.x) {
    float nx = 0.0f, ny = 0.0f, nz = 0.0f;
    for (int t = off[v]; t < off[v + 1]; ++t) {
      const int f = vf[t];
      const P3 p0 = load3(verts, faces[3LL * f]), p1 = load3(verts, faces[3LL * f + 1]), p2 = load3(verts, faces[3LL * f + 2]);
      const P3 a = {fs(p1.x, p0.x), fs(p1.y, p0.y), fs(p1.z, p0.z)}, b = {fs(p2.x, p0.x), fs(p2.y, p0.y), fs(p2.z, p0.z)};
      nx = fa(nx, fs(fm(a.y, b.z), fm(a.z, b.y)));
      ny = fa(ny, fs(fm(a.z, b.x), fm(a.x, b.z)));
      nz = fa(nz, fs(fm(a.x, b.y), fm(a.y, b.x)));
    }
    const float len = __fsqrt_rn(fa(fa(fm(nx, nx), fm(ny, ny)), fm(nz, nz)));
    const float d = len > kNormalEps ? len : kNormalEps;
    normals[3LL * v] = fd(nx, d);
    normals[3LL * v + 1] = fd(ny, d);
    normals[3LL * v + 2] = fd(nz, d);
  }
}

// ---- shading and compositing -----------------------------------------------------------------------------------------------

// one thread per output pixel (view, i, j): 2x2 coverage, the normal of sample (2i, 2j), composite on white, truncate to u8
__global__ void shade_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces,
                             const float* __restrict__ normals, const float* __restrict__ cams, int n_cams, float focal, int S,
                             const int32_t* __restrict__ pix_to_face, uint8_t* __restrict__ out, long long row_stride,
                             int view_stride) {
  const int n2 = 2 * S;
  const long long n = (long long)n_cams * S * S;
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < n; p += (long long)gridDim.x * blockDim.x) {
    const int cam = (int)(p / ((long long)S * S)), i = (int)(p / S % S), j = (int)(p % S);
    const float* cp = cams + 12 * cam;
    const int32_t* pf = pix_to_face + (long long)cam * n2 * n2 + (2LL * i) * n2 + 2 * j;
    const int f = pf[0];
    const int covered = (f >= 0) + (pf[1] >= 0) + (pf[n2] >= 0) + (pf[n2 + 1] >= 0);
    const float mask = fm((float)covered, 0.25f);
    P3 nrm = {0.0f, 0.0f, 0.0f};
    if (f >= 0) {
      const Face s = face_setup(verts, faces, f, cp, focal, n2);
      Bary b;
      barycentrics(s, sample_ndc(2 * j, n2), sample_ndc(2 * i, n2), &b);  // inside: pix_to_face came from this test
      const P3 a0 = load3(normals, faces[3LL * f]), a1 = load3(normals, faces[3LL * f + 1]),
               a2 = load3(normals, faces[3LL * f + 2]);
      nrm = {fa(fa(fm(b.b0, a0.x), fm(b.b1, a1.x)), fm(b.b2, a2.x)), fa(fa(fm(b.b0, a0.y), fm(b.b1, a1.y)), fm(b.b2, a2.y)),
             fa(fa(fm(b.b0, a0.z), fm(b.b1, a1.z)), fm(b.b2, a2.z))};
    }
    // the reference's "camera sphere": the normal mapped as a point with the translation halved
    const P3 t = transform(nrm, cp, fm(cp[9], 0.5f), fm(cp[10], 0.5f), fm(cp[11], 0.5f));
    const float len = __fsqrt_rn(fa(fa(fm(t.x, t.x), fm(t.y, t.y)), fm(t.z, t.z)));
    const float d = len > kShadeEps ? len : kShadeEps;
    const float ch[3] = {fd(t.x, d), fd(t.y, d), fd(t.z, d)};
    uint8_t* o = out + (long long)i * row_stride + (long long)cam * view_stride + 3LL * j;
    const float inv = fs(1.0f, mask);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float c = fminf(fmaxf(fm(fa(ch[k], 1.0f), 0.5f), 0.0f), 1.0f);
      o[k] = (uint8_t)(int)fm(fa(fm(c, mask), inv), 255.0f);
    }
  }
}

// ---- texture shading -------------------------------------------------------------------------------------------------------

constexpr int kMaxTexSide = 16384;
constexpr int kMaxLevels = 15;  // 16384 -> 1 in 14 halvings
constexpr float kUvLimit = 32768.0f;
constexpr int kMaxRecords = 65536;

enum : int {
  kNearest = 9728,
  kLinear = 9729,
  kNearestMipNearest = 9984,
  kLinearMipNearest = 9985,
  kNearestMipLinear = 9986,
  kLinearMipLinear = 9987,
  kRepeat = 10497,
  kClampToEdge = 33071,
  kMirroredRepeat = 33648,
};

// a shading record (the header's amb_shade_record): the mip chain, level l being level_height[l] rows of level_width[l] RGB
// texels at byte offset level_offset[l] of the level buffer (n_levels = 0: no texture), the sampler's enums and the base
// colour factor.  amb_render_shade_texture passes one by value, amb_render_shade_materials reads one per face.
using Record = amb_shade_record;
static_assert(sizeof(((Record*)nullptr)->level_offset) / sizeof(int64_t) == kMaxLevels, "one slot per level");

// level l + 1 texel (x, y) = floor((a + b + c + d + 2) / 4) per channel over level-l texels (min(2x+dx, w-1), min(2y+dy, h-1))
__global__ void texture_level_kernel(uint8_t* __restrict__ levels, long long src_off, int sw, int sh, long long dst_off,
                                     int dw, int dh) {
  const long long n = (long long)dw * dh;
  const uint8_t* src = levels + src_off;
  uint8_t* dst = levels + dst_off;
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < n; p += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(p % dw), y = (int)(p / dw);
    const int x0 = min(2 * x, sw - 1), x1 = min(2 * x + 1, sw - 1), y0 = min(2 * y, sh - 1), y1 = min(2 * y + 1, sh - 1);
    const uint8_t* r0 = src + 3LL * y0 * sw;
    const uint8_t* r1 = src + 3LL * y1 * sw;
#pragma unroll
    for (int k = 0; k < 3; ++k)
      dst[3 * p + k] = (uint8_t)((r0[3 * x0 + k] + r0[3 * x1 + k] + r1[3 * x0 + k] + r1[3 * x1 + k] + 2) >> 2);
  }
}

__device__ __forceinline__ int wrap_index(int i, int n, int mode) {
  if (mode == kClampToEdge) return clampi(i, 0, n - 1);
  if (mode == kMirroredRepeat) {
    const int m = ((i % (2 * n)) + 2 * n) % (2 * n);
    return m < n ? m : 2 * n - 1 - m;
  }
  return ((i % n) + n) % n;  // REPEAT
}

// filtered RGB (0..255, not rounded) of level `l` at (u, v): NEAREST texel (floor(u w), floor(v h)), or LINEAR around
// (u w - 1/2, v h - 1/2) with weights ((t00 (1-fx) + t10 fx) (1-fy)) + ((t01 (1-fx) + t11 fx) fy)
__device__ __forceinline__ void sample_level(const uint8_t* __restrict__ levels, const Record& rec, int l, bool linear,
                                             int wrap_s, int wrap_t, float u, float v, float* rgb) {
  const int w = rec.level_width[l], h = rec.level_height[l];
  const uint8_t* base = levels + rec.level_offset[l];
  u = fminf(fmaxf(u, -kUvLimit), kUvLimit);
  v = fminf(fmaxf(v, -kUvLimit), kUvLimit);
  if (!linear) {
    const int x = wrap_index((int)floorf(fm(u, (float)w)), w, wrap_s), y = wrap_index((int)floorf(fm(v, (float)h)), h, wrap_t);
    const uint8_t* t = base + 3LL * ((long long)y * w + x);
    rgb[0] = (float)t[0];
    rgb[1] = (float)t[1];
    rgb[2] = (float)t[2];
    return;
  }
  const float x = fs(fm(u, (float)w), 0.5f), y = fs(fm(v, (float)h), 0.5f);
  const float xf = floorf(x), yf = floorf(y);
  const float fx = fs(x, xf), fy = fs(y, yf), gx = fs(1.0f, fx), gy = fs(1.0f, fy);
  const int xi = (int)xf, yi = (int)yf;
  const int xa = wrap_index(xi, w, wrap_s), xb = wrap_index(xi + 1, w, wrap_s);
  const int ya = wrap_index(yi, h, wrap_t), yb = wrap_index(yi + 1, h, wrap_t);
  const uint8_t* r0 = base + 3LL * ya * w;
  const uint8_t* r1 = base + 3LL * yb * w;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float t00 = r0[3 * xa + k], t10 = r0[3 * xb + k], t01 = r1[3 * xa + k], t11 = r1[3 * xb + k];
    rgb[k] = fa(fm(fa(fm(t00, gx), fm(t10, fx)), gy), fm(fa(fm(t01, gx), fm(t11, fx)), fy));
  }
}

// the shaded colour of one sample covered by face f (DESIGN §16, texture shading)
__device__ __forceinline__ void texture_sample(const float* __restrict__ verts, const int32_t* __restrict__ faces,
                                               const float* __restrict__ normals, const float* __restrict__ uv,
                                               const float* cp, float focal, int S, int f, int r, int c,
                                               const uint8_t* __restrict__ levels, const Record& rec, float* col) {
  const int n2 = 2 * S;
  const Face s = face_setup(verts, faces, f, cp, focal, n2);
  Bary b;
  barycentrics(s, sample_ndc(c, n2), sample_ndc(r, n2), &b);  // inside: pix_to_face came from this test
  const int i0 = faces[3LL * f], i1 = faces[3LL * f + 1], i2 = faces[3LL * f + 2];
  const P3 a0 = load3(normals, i0), a1 = load3(normals, i1), a2 = load3(normals, i2);
  const P3 n = {fa(fa(fm(b.b0, a0.x), fm(b.b1, a1.x)), fm(b.b2, a2.x)), fa(fa(fm(b.b0, a0.y), fm(b.b1, a1.y)), fm(b.b2, a2.y)),
                fa(fa(fm(b.b0, a0.z), fm(b.b1, a1.z)), fm(b.b2, a2.z))};
  // n R (rotation only), normalised; two-sided headlight
  const float vx = fa(fa(fm(n.x, cp[0]), fm(n.y, cp[3])), fm(n.z, cp[6]));
  const float vy = fa(fa(fm(n.x, cp[1]), fm(n.y, cp[4])), fm(n.z, cp[7]));
  const float vz = fa(fa(fm(n.x, cp[2]), fm(n.y, cp[5])), fm(n.z, cp[8]));
  const float len = __fsqrt_rn(fa(fa(fm(vx, vx), fm(vy, vy)), fm(vz, vz)));
  const float shade = fa(0.35f, fm(0.65f, fabsf(fd(vz, len > kShadeEps ? len : kShadeEps))));
  float base[3] = {rec.base_color[0], rec.base_color[1], rec.base_color[2]};
  if (rec.n_levels) {
    const float u0 = uv[2LL * i0], w0 = uv[2LL * i0 + 1], u1 = uv[2LL * i1], w1 = uv[2LL * i1 + 1];
    const float u2 = uv[2LL * i2], w2 = uv[2LL * i2 + 1];
    const float u = fa(fa(fm(b.b0, u0), fm(b.b1, u1)), fm(b.b2, u2)), v = fa(fa(fm(b.b0, w0), fm(b.b1, w1)), fm(b.b2, w2));
    // level of detail of (face, view): projected area A_s in samples against the uv area A_t in level-0 texels
    const float a_s = fm(fm(0.5f, fabsf(edge(s.v0.x, s.v0.y, s.v1, s.v2))), (float)(S * S));
    const float a_t = fm(fm(0.5f, fabsf(fs(fm(fs(u0, u1), fs(w2, w1)), fm(fs(w0, w1), fs(u2, u1))))),
                         (float)((long long)rec.level_width[0] * rec.level_height[0]));
    int level = 0, filter = rec.mag_filter;  // magnified, or a face with a depth <= 0
    if (s.v0.z > 0.0f && s.v1.z > 0.0f && s.v2.z > 0.0f && !(a_t <= a_s)) {
      filter = rec.min_filter;
      if (rec.min_filter >= kNearestMipNearest) {
        float lim = a_s;
        while (level < rec.n_levels - 1 && !(a_t <= lim)) {
          lim = fm(lim, 4.0f);
          ++level;
        }
      }
    }
    const bool linear = filter == kLinear || filter == kLinearMipNearest || filter == kLinearMipLinear;
    float t[3];
    sample_level(levels, rec, level, linear, rec.wrap_s, rec.wrap_t, u, v, t);
#pragma unroll
    for (int k = 0; k < 3; ++k) base[k] = fm(base[k], fd(t[k], 255.0f));
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) col[k] = fm(base[k], shade);
}

// one thread per output pixel (view, i, j): the mean of its four samples' shaded colours (white where no face), truncated.
// Each covered sample shades with `rec` when face_record is null (amb_render_shade_texture), else with
// records[face_record[f]] (amb_render_shade_materials).
__device__ __forceinline__ void shade_texture_pixels(const float* __restrict__ verts, const int32_t* __restrict__ faces,
                                                     const float* __restrict__ normals, const float* __restrict__ uv,
                                                     const float* __restrict__ cams, int n_cams, float focal, int S,
                                                     const int32_t* __restrict__ pix_to_face,
                                                     const int32_t* __restrict__ face_record, const Record* __restrict__ records,
                                                     const uint8_t* __restrict__ levels, const Record& rec,
                                                     uint8_t* __restrict__ out, long long row_stride, int view_stride) {
  const int n2 = 2 * S;
  const long long n = (long long)n_cams * S * S;
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < n; p += (long long)gridDim.x * blockDim.x) {
    const int cam = (int)(p / ((long long)S * S)), i = (int)(p / S % S), j = (int)(p % S);
    const float* cp = cams + 12 * cam;
    const int32_t* pf = pix_to_face + (long long)cam * n2 * n2;
    float acc[3];
#pragma unroll 1
    for (int q = 0; q < 4; ++q) {
      const int r = 2 * i + (q >> 1), c = 2 * j + (q & 1);
      const int f = pf[(long long)r * n2 + c];
      float col[3] = {1.0f, 1.0f, 1.0f};
      if (f >= 0)
        texture_sample(verts, faces, normals, uv, cp, focal, S, f, r, c, levels, face_record ? records[face_record[f]] : rec,
                       col);
#pragma unroll
      for (int k = 0; k < 3; ++k) acc[k] = q ? fa(acc[k], col[k]) : col[k];
    }
    uint8_t* o = out + (long long)i * row_stride + (long long)cam * view_stride + 3LL * j;
#pragma unroll
    for (int k = 0; k < 3; ++k) o[k] = (uint8_t)(int)fm(fminf(fmaxf(fm(acc[k], 0.25f), 0.0f), 1.0f), 255.0f);
  }
}

__global__ void __launch_bounds__(256) shade_texture_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces,
                                                            const float* __restrict__ normals, const float* __restrict__ uv,
                                                            const float* __restrict__ cams, int n_cams, float focal, int S,
                                                            const int32_t* __restrict__ pix_to_face,
                                                            const uint8_t* __restrict__ levels, const Record rec,
                                                            uint8_t* __restrict__ out, long long row_stride, int view_stride) {
  shade_texture_pixels(verts, faces, normals, uv, cams, n_cams, focal, S, pix_to_face, nullptr, nullptr, levels, rec, out,
                       row_stride, view_stride);
}

__global__ void __launch_bounds__(256) shade_materials_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces,
                                                              const float* __restrict__ normals, const float* __restrict__ uv,
                                                              const float* __restrict__ cams, int n_cams, float focal, int S,
                                                              const int32_t* __restrict__ pix_to_face,
                                                              const int32_t* __restrict__ face_record,
                                                              const Record* __restrict__ records,
                                                              const uint8_t* __restrict__ levels, uint8_t* __restrict__ out,
                                                              long long row_stride, int view_stride) {
  shade_texture_pixels(verts, faces, normals, uv, cams, n_cams, focal, S, pix_to_face, face_record, records, levels,
                       records[0], out, row_stride, view_stride);
}

constexpr int kThreads = 256;

bool render_sizes_ok(int64_t n_vertices, int64_t n_faces) {
  return n_vertices >= 0 && n_faces >= 0 && n_vertices < (1LL << 31) - 1 && 6 * n_faces < (1LL << 31);
}

// a full mip chain: level 0 of 1..16384 texels a side, each next level halved (at least 1), down to 1 x 1, in ascending
// non-overlapping byte ranges; false with the reason in *why
bool level_table_ok(const int64_t* table, int n_levels, Record* rec, const char** why) {
  *why = "";
  if (n_levels < 1 || n_levels > kMaxLevels) return *why = "n_levels outside [1, 15]", false;
  long long end = 0;
  for (int l = 0; l < n_levels; ++l) {
    const int64_t off = table[3 * l], w = table[3 * l + 1], h = table[3 * l + 2];
    if (l == 0 && (w < 1 || h < 1 || w > kMaxTexSide || h > kMaxTexSide)) return *why = "level 0 size outside [1, 16384]", false;
    if (l > 0 && (w != (rec->level_width[l - 1] > 1 ? rec->level_width[l - 1] >> 1 : 1) ||
                  h != (rec->level_height[l - 1] > 1 ? rec->level_height[l - 1] >> 1 : 1)))
      return *why = "a level is not the previous one halved", false;
    if (off < end) return *why = "level byte ranges overlap or descend", false;
    rec->level_offset[l] = off;
    rec->level_width[l] = (int)w;
    rec->level_height[l] = (int)h;
    end = off + 3 * w * h;
  }
  if (rec->level_width[n_levels - 1] != 1 || rec->level_height[n_levels - 1] != 1)
    return *why = "the chain does not end at 1 x 1", false;
  rec->n_levels = n_levels;
  return true;
}

}  // namespace
}  // namespace amb

using namespace amb;

extern "C" {

int amb_render_vertex_normals(const float* vertices, int64_t n_vertices, const int32_t* faces, const int32_t* vf_offsets,
                              const int32_t* vf_faces, float* normals, amb_stream_t stream) {
  AMB_CHECK_ARG(vertices && faces && vf_offsets && vf_faces && normals, "render_vertex_normals: null pointer");
  AMB_CHECK_ARG(render_sizes_ok(n_vertices, 0), "render_vertex_normals: bad vertex count %lld", (long long)n_vertices);
  if (!n_vertices) return AMB_OK;
  vertex_normals_kernel<<<blocks_for(n_vertices, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      vertices, faces, (int)n_vertices, vf_offsets, vf_faces, normals);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_render_rasterize(const float* vertices, int64_t n_vertices, const int32_t* faces, int64_t n_faces,
                         const float* cameras, int n_cameras, float focal, int image_size, uint64_t* depth_keys,
                         int32_t* queue, int32_t* pix_to_face, amb_stream_t stream) {
  AMB_CHECK_ARG((!n_faces || (vertices && faces)) && cameras && depth_keys && queue && pix_to_face,
                "render_rasterize: null pointer");
  AMB_CHECK_ARG(render_sizes_ok(n_vertices, n_faces), "render_rasterize: bad mesh size (%lld vertices, %lld faces)",
                (long long)n_vertices, (long long)n_faces);
  AMB_CHECK_ARG(n_cameras >= 1 && image_size >= 1, "render_rasterize: need n_cameras >= 1 and image_size >= 1 (got %d, %d)",
                n_cameras, image_size);
  const long long n2 = 2LL * image_size, samples = (long long)n_cameras * n2 * n2;
  AMB_CHECK_ARG(samples < (1LL << 31) && (long long)n_cameras * n_faces < (1LL << 31) - 1,
                "render_rasterize: %d cameras x %lld samples or x %lld faces overflow int32 indices", n_cameras, n2 * n2,
                (long long)n_faces);
  cudaStream_t st = (cudaStream_t)stream;
  AMB_CHECK_CUDA(cudaMemsetAsync(depth_keys, 0xff, sizeof(uint64_t) * samples, st));
  if (n_faces) {
    AMB_CHECK_CUDA(cudaMemsetAsync(queue, 0, sizeof(int32_t), st));
    const int nf = (int)n_faces;
    raster_small_kernel<<<blocks_for((long long)n_cameras * nf, kThreads), kThreads, 0, st>>>(
        vertices, faces, nf, cameras, n_cameras, focal, (int)n2, reinterpret_cast<unsigned long long*>(depth_keys), queue);
    raster_large_kernel<<<4 * num_sms(), kThreads, 0, st>>>(vertices, faces, nf, cameras, focal, (int)n2,
                                                            reinterpret_cast<unsigned long long*>(depth_keys), queue);
    AMB_CHECK_CUDA(cudaGetLastError());
  }
  resolve_kernel<<<blocks_for(samples, kThreads), kThreads, 0, st>>>(reinterpret_cast<const unsigned long long*>(depth_keys),
                                                                    samples, pix_to_face);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_render_shade_normals(const float* vertices, int64_t n_vertices, const int32_t* faces, int64_t n_faces,
                             const float* normals, const float* cameras, int n_cameras, float focal, int image_size,
                             const int32_t* pix_to_face, uint8_t* out, int64_t row_stride, int64_t view_stride,
                             amb_stream_t stream) {
  AMB_CHECK_ARG((!n_faces || (vertices && faces && normals)) && cameras && pix_to_face && out,
                "render_shade_normals: null pointer");
  AMB_CHECK_ARG(render_sizes_ok(n_vertices, n_faces), "render_shade_normals: bad mesh size (%lld vertices, %lld faces)",
                (long long)n_vertices, (long long)n_faces);
  AMB_CHECK_ARG(n_cameras >= 1 && image_size >= 1,
                "render_shade_normals: need n_cameras >= 1 and image_size >= 1 (got %d, %d)", n_cameras, image_size);
  const long long n2 = 2LL * image_size;
  AMB_CHECK_ARG((long long)n_cameras * n2 * n2 < (1LL << 31), "render_shade_normals: %d cameras x %lld samples overflow int32",
                n_cameras, n2 * n2);
  AMB_CHECK_ARG(row_stride >= 3LL * image_size && view_stride >= 0 && view_stride < (1LL << 31) &&
                    (n_cameras == 1 || view_stride >= 3LL * image_size),
                "render_shade_normals: bad strides (row %lld, view %lld)", (long long)row_stride, (long long)view_stride);
  const long long n = (long long)n_cameras * image_size * image_size;
  shade_kernel<<<blocks_for(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      vertices, faces, normals, cameras, n_cameras, focal, image_size, pix_to_face, out, row_stride, (int)view_stride);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_render_texture_levels(uint8_t* levels, const int64_t* level_table, int n_levels, amb_stream_t stream) {
  AMB_CHECK_ARG(levels && level_table, "render_texture_levels: null pointer");
  Record tl;
  const char* why;
  AMB_CHECK_ARG(level_table_ok(level_table, n_levels, &tl, &why), "render_texture_levels: bad level table (%s)", why);
  for (int l = 1; l < n_levels; ++l) {
    texture_level_kernel<<<blocks_for((long long)tl.level_width[l] * tl.level_height[l], kThreads), kThreads, 0,
                           (cudaStream_t)stream>>>(levels, tl.level_offset[l - 1], tl.level_width[l - 1],
                                                   tl.level_height[l - 1], tl.level_offset[l], tl.level_width[l],
                                                   tl.level_height[l]);
    AMB_CHECK_CUDA(cudaGetLastError());
  }
  return AMB_OK;
}

int amb_render_shade_texture(const float* vertices, int64_t n_vertices, const int32_t* faces, int64_t n_faces,
                             const float* normals, const float* uv, const float* cameras, int n_cameras, float focal,
                             int image_size, const int32_t* pix_to_face, const uint8_t* levels, const int64_t* level_table,
                             int n_levels, int mag_filter, int min_filter, int wrap_s, int wrap_t, float base_r,
                             float base_g, float base_b, uint8_t* out, int64_t row_stride, int64_t view_stride,
                             amb_stream_t stream) {
  AMB_CHECK_ARG((!n_faces || (vertices && faces && normals && (!n_levels || uv))) && (!n_levels || (levels && level_table)) &&
                    cameras && pix_to_face && out,
                "render_shade_texture: null pointer");
  AMB_CHECK_ARG(render_sizes_ok(n_vertices, n_faces), "render_shade_texture: bad mesh size (%lld vertices, %lld faces)",
                (long long)n_vertices, (long long)n_faces);
  AMB_CHECK_ARG(n_cameras >= 1 && image_size >= 1,
                "render_shade_texture: need n_cameras >= 1 and image_size >= 1 (got %d, %d)", n_cameras, image_size);
  const long long n2 = 2LL * image_size;
  AMB_CHECK_ARG((long long)n_cameras * n2 * n2 < (1LL << 31), "render_shade_texture: %d cameras x %lld samples overflow int32",
                n_cameras, n2 * n2);
  AMB_CHECK_ARG(row_stride >= 3LL * image_size && view_stride >= 0 && view_stride < (1LL << 31) &&
                    (n_cameras == 1 || view_stride >= 3LL * image_size),
                "render_shade_texture: bad strides (row %lld, view %lld)", (long long)row_stride, (long long)view_stride);
  AMB_CHECK_ARG(mag_filter == kNearest || mag_filter == kLinear, "render_shade_texture: bad mag_filter %d", mag_filter);
  AMB_CHECK_ARG(min_filter == kNearest || min_filter == kLinear || (min_filter >= kNearestMipNearest && min_filter <= kLinearMipLinear),
                "render_shade_texture: bad min_filter %d", min_filter);
  for (int wrap : {wrap_s, wrap_t})
    AMB_CHECK_ARG(wrap == kRepeat || wrap == kClampToEdge || wrap == kMirroredRepeat, "render_shade_texture: bad wrap mode %d",
                  wrap);
  Record rec = {};
  if (n_levels) {
    const char* why;
    AMB_CHECK_ARG(level_table_ok(level_table, n_levels, &rec, &why), "render_shade_texture: bad level table (%s)", why);
  }
  rec.mag_filter = mag_filter;
  rec.min_filter = min_filter;
  rec.wrap_s = wrap_s;
  rec.wrap_t = wrap_t;
  rec.base_color[0] = base_r;
  rec.base_color[1] = base_g;
  rec.base_color[2] = base_b;
  const long long n = (long long)n_cameras * image_size * image_size;
  shade_texture_kernel<<<blocks_for(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      vertices, faces, normals, uv, cameras, n_cameras, focal, image_size, pix_to_face, levels, rec, out, row_stride,
      (int)view_stride);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

int amb_render_shade_materials(const float* vertices, int64_t n_vertices, const int32_t* faces, int64_t n_faces,
                               const float* normals, const float* uv, const float* cameras, int n_cameras, float focal,
                               int image_size, const int32_t* pix_to_face, const int32_t* face_record,
                               const void* records, int n_records, const uint8_t* levels, uint8_t* out,
                               int64_t row_stride, int64_t view_stride, amb_stream_t stream) {
  AMB_CHECK_ARG((!n_faces || (vertices && faces && normals && face_record)) && records && cameras && pix_to_face && out,
                "render_shade_materials: null pointer");
  AMB_CHECK_ARG(render_sizes_ok(n_vertices, n_faces), "render_shade_materials: bad mesh size (%lld vertices, %lld faces)",
                (long long)n_vertices, (long long)n_faces);
  AMB_CHECK_ARG(n_cameras >= 1 && image_size >= 1,
                "render_shade_materials: need n_cameras >= 1 and image_size >= 1 (got %d, %d)", n_cameras, image_size);
  const long long n2 = 2LL * image_size;
  AMB_CHECK_ARG((long long)n_cameras * n2 * n2 < (1LL << 31),
                "render_shade_materials: %d cameras x %lld samples overflow int32", n_cameras, n2 * n2);
  AMB_CHECK_ARG(row_stride >= 3LL * image_size && view_stride >= 0 && view_stride < (1LL << 31) &&
                    (n_cameras == 1 || view_stride >= 3LL * image_size),
                "render_shade_materials: bad strides (row %lld, view %lld)", (long long)row_stride, (long long)view_stride);
  AMB_CHECK_ARG(n_records >= 1 && n_records <= kMaxRecords, "render_shade_materials: n_records %d outside [1, %d]", n_records,
                kMaxRecords);
  const long long n = (long long)n_cameras * image_size * image_size;
  shade_materials_kernel<<<blocks_for(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      vertices, faces, normals, uv, cameras, n_cameras, focal, image_size, pix_to_face, face_record,
      static_cast<const Record*>(records), levels, out, row_stride, (int)view_stride);
  AMB_CHECK_CUDA(cudaGetLastError());
  return AMB_OK;
}

}  // extern "C"
