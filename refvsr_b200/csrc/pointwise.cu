// HBM/L2-bound kernels of the RefVSR hot path: image prep, SPyNet pyramid glue, flow warp,
// reference gather / affine resampling, confidence-map glue and the reconstruction tail.
// Every kernel is NHWC with 16-byte vector accesses where the channel count allows it.
// Arithmetic follows SURVEY.md appendix A (verified against torch 2.11 by oracle/refvsr_oracle.py).
#include <cstdlib>
#include <type_traits>

#include "common.cuh"
#include "frame_u8.cuh"

namespace rv {

// ---------------------------------------------------------------------------------------------
// small vector helpers: V elements of T moved as one 16/8/4-byte access
// ---------------------------------------------------------------------------------------------
template <typename T, int V>
struct Vec {
  T v[V];
};
template <typename T, int V>
__device__ __forceinline__ Vec<T, V> ldv(const T* p) {
  Vec<T, V> r;
  if constexpr (sizeof(T) * V == 16) {
    *reinterpret_cast<uint4*>(&r) = __ldg(reinterpret_cast<const uint4*>(p));
  } else if constexpr (sizeof(T) * V == 8) {
    *reinterpret_cast<uint2*>(&r) = __ldg(reinterpret_cast<const uint2*>(p));
  } else {
#pragma unroll
    for (int i = 0; i < V; ++i) r.v[i] = p[i];
  }
  return r;
}
template <typename T, int V>
__device__ __forceinline__ void stv(T* p, const Vec<T, V>& r) {
  if constexpr (sizeof(T) * V == 16) {
    *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(&r);
  } else if constexpr (sizeof(T) * V == 8) {
    *reinterpret_cast<uint2*>(p) = *reinterpret_cast<const uint2*>(&r);
  } else {
#pragma unroll
    for (int i = 0; i < V; ++i) p[i] = r.v[i];
  }
}

// 16-byte vector number i of a map (i = pixel * vectors-per-pixel + vector, 32-bit): one IMAD.WIDE per address
template <typename T, int V>
__device__ __forceinline__ Vec<T, V> ldvi(const T* base, int i) {
  static_assert(sizeof(T) * V == 16, "16-byte vectors");
  Vec<T, V> r;
  *reinterpret_cast<uint4*>(&r) = __ldg(reinterpret_cast<const uint4*>(base) + (unsigned)i);
  return r;
}
template <typename T, int V>
__device__ __forceinline__ void stvi(T* base, int i, const Vec<T, V>& r) {
  static_assert(sizeof(T) * V == 16, "16-byte vectors");
  reinterpret_cast<uint4*>(base)[(unsigned)i] = *reinterpret_cast<const uint4*>(&r);
}

// ---------------------------------------------------------------------------------------------
// 4-tap blend of one channel vector: r = a * w.x + b * w.y + c * w.z + d * w.w in fp32, evaluated for every element as
// fma(d, w.w, fma(c, w.z, fma(b, w.y, a * w.x))).  The gather kernels spend many issue slots per byte, so the 16-bit <-> fp32 conversions are done on packed words.  sm_90 has no packed fp32 FMA: each pair is
// two round-to-nearest FFMAs, the same values a packed instruction gives.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
template <typename T>
__device__ __forceinline__ float2 unpack2(const T* p);
template <>
__device__ __forceinline__ float2 unpack2<float>(const float* p) { return make_float2(p[0], p[1]); }
template <>
__device__ __forceinline__ float2 unpack2<__half>(const __half* p) { return __half22float2(*reinterpret_cast<const __half2*>(p)); }
template <>
__device__ __forceinline__ float2 unpack2<__nv_bfloat16>(const __nv_bfloat16* p) {
  const uint32_t u = *reinterpret_cast<const uint32_t*>(p);
  return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}
template <typename T>
__device__ __forceinline__ void pack2(T* p, float2 v);
template <>
__device__ __forceinline__ void pack2<float>(float* p, float2 v) { p[0] = v.x; p[1] = v.y; }
template <>
__device__ __forceinline__ void pack2<__half>(__half* p, float2 v) { *reinterpret_cast<__half2*>(p) = __floats2half2_rn(v.x, v.y); }
template <>
__device__ __forceinline__ void pack2<__nv_bfloat16>(__nv_bfloat16* p, float2 v) {
  *reinterpret_cast<__nv_bfloat162*>(p) = __floats2bfloat162_rn(v.x, v.y);
}

template <typename T, int V>
__device__ __forceinline__ Vec<T, V> blend4(const Vec<T, V>& a, const Vec<T, V>& b, const Vec<T, V>& c, const Vec<T, V>& d, float4 w) {
  static_assert(V % 2 == 0, "blend4 works on pairs");
  const float2 wx = make_float2(w.x, w.x), wy = make_float2(w.y, w.y), wz = make_float2(w.z, w.z), ww = make_float2(w.w, w.w);
  Vec<T, V> r;
#pragma unroll
  for (int k = 0; k < V; k += 2) {
    float2 acc = fmul2(unpack2<T>(&a.v[k]), wx);
    acc = ffma2(unpack2<T>(&b.v[k]), wy, acc);
    acc = ffma2(unpack2<T>(&c.v[k]), wz, acc);
    acc = ffma2(unpack2<T>(&d.v[k]), ww, acc);
    pack2<T>(&r.v[k], acc);
  }
  return r;
}

// The same blend in the order the compiler contracts aligned_sample_kernel's `lt * a + rb * b + lb * c + rt * d`:
// fma(d, w.w, fma(c, w.z, fma(a, w.x, b * w.y))) - for the fast paths that must reproduce that kernel bit for bit.
template <typename T, int V>
__device__ __forceinline__ Vec<T, V> blend4_as_generic(const Vec<T, V>& a, const Vec<T, V>& b, const Vec<T, V>& c, const Vec<T, V>& d,
                                                       float4 w) {
  static_assert(V % 2 == 0, "blend4 works on pairs");
  const float2 wx = make_float2(w.x, w.x), wy = make_float2(w.y, w.y), wz = make_float2(w.z, w.z), ww = make_float2(w.w, w.w);
  Vec<T, V> r;
#pragma unroll
  for (int k = 0; k < V; k += 2) {
    float2 acc = fmul2(unpack2<T>(&b.v[k]), wy);
    acc = ffma2(unpack2<T>(&a.v[k]), wx, acc);
    acc = ffma2(unpack2<T>(&c.v[k]), wz, acc);
    acc = ffma2(unpack2<T>(&d.v[k]), ww, acc);
    pack2<T>(&r.v[k], acc);
  }
  return r;
}

// torch.linspace(-1, 1, n)[i]  (symmetric evaluation, aten RangeFactories)
__device__ __forceinline__ float linspace_m1_1(int i, int n) {
  if (n == 1) return -1.f;
  float step = 2.0f / (float)(n - 1);
  return (i < n / 2) ? (-1.0f + step * (float)i) : (1.0f - step * (float)(n - 1 - i));
}

// aten area_pixel_compute_source_index for bilinear, align_corners=False
__device__ __forceinline__ void bilin_src(int X, float scale, int in_size, int& i0, int& i1,
                                          float& l1) {
  float s = scale * ((float)X + 0.5f) - 0.5f;
  if (s < 0.f) s = 0.f;
  i0 = (int)s;
  if (i0 > in_size - 1) i0 = in_size - 1;
  i1 = i0 + ((i0 < in_size - 1) ? 1 : 0);
  l1 = s - (float)i0;
}
// align_corners=True variant: src = X * (in-1)/(out-1)
__device__ __forceinline__ void bilin_src_ac(int X, float scale, int in_size, int& i0, int& i1,
                                             float& l1) {
  float s = scale * (float)X;
  i0 = (int)s;
  if (i0 > in_size - 1) i0 = in_size - 1;
  i1 = i0 + ((i0 < in_size - 1) ? 1 : 0);
  l1 = s - (float)i0;
}

// ---------------------------------------------------------------------------------------------
// rv_prep_image
// ---------------------------------------------------------------------------------------------
struct Mat12 {
  float m[12];
  int use;
};

template <typename T>
__global__ void prep_image_kernel(const float* __restrict__ src, int H, int W, Mat12 mat, int pool2,
                                  T* __restrict__ out, int out_c) {
  int Ho = pool2 ? H / 2 : H, Wo = pool2 ? W / 2 : W;
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Ho * Wo) return;
  int y = p / Wo, x = p % Wo;
  float acc[3] = {0.f, 0.f, 0.f};
  int n = pool2 ? 2 : 1;
  for (int dy = 0; dy < n; ++dy)
    for (int dx = 0; dx < n; ++dx) {
      int sy = pool2 ? 2 * y + dy : y, sx = pool2 ? 2 * x + dx : x;
      float r = src[(0 * H + sy) * W + sx], g = src[(1 * H + sy) * W + sx],
            b = src[(2 * H + sy) * W + sx];
      if (mat.use) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
          acc[c] += mat.m[c * 4 + 0] * r + mat.m[c * 4 + 1] * g + mat.m[c * 4 + 2] * b +
                    mat.m[c * 4 + 3];
      } else {
        acc[0] += r;
        acc[1] += g;
        acc[2] += b;
      }
    }
  float inv = pool2 ? 0.25f : 1.f;
  T* o = out + (size_t)p * out_c;
  for (int c = 0; c < out_c; ++c) o[c] = from_f<T>(c < 3 ? acc[c] * inv : 0.f);
}

// ---------------------------------------------------------------------------------------------
// SPyNet glue
// ---------------------------------------------------------------------------------------------
__global__ void spynet_resize_norm_kernel(const float* __restrict__ src, int H, int W,
                                          float* __restrict__ out, int Ho, int Wo) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Ho * Wo) return;
  int y = p / Wo, x = p % Wo;
  const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
  int y0, y1, x0, x1;
  float ly, lx;
  bilin_src(y, (float)H / (float)Ho, H, y0, y1, ly);
  bilin_src(x, (float)W / (float)Wo, W, x0, x1, lx);
  float hy = 1.f - ly, hx = 1.f - lx;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float* s = src + (size_t)c * H * W;
    float v = hy * (hx * s[y0 * W + x0] + lx * s[y0 * W + x1]) +
              ly * (hx * s[y1 * W + x0] + lx * s[y1 * W + x1]);
    out[(size_t)p * 3 + c] = (v - mean[c]) / stdv[c];
  }
}

__global__ void avgpool2_kernel(const float* __restrict__ src, int H, int W, int C,
                                float* __restrict__ out) {
  int Ho = H / 2, Wo = W / 2;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Ho * Wo * C) return;
  int c = i % C, p = i / C;
  int y = p / Wo, x = p % Wo;
  const float* s = src + ((size_t)(2 * y) * W + 2 * x) * C + c;
  float v = s[0] + s[C] + s[(size_t)W * C] + s[(size_t)W * C + C];
  out[i] = v * 0.25f;
}

template <typename T>
__global__ void spynet_level_input_kernel(const float* __restrict__ ref,
                                          const float* __restrict__ supp,
                                          const float* __restrict__ flow_prev, int H, int W,
                                          T* __restrict__ out8, float* __restrict__ flow_up) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= H * W) return;
  int y = p / W, x = p % W;
  float fx = 0.f, fy = 0.f;
  if (flow_prev != nullptr) {
    int Hp = H / 2, Wp = W / 2;
    int y0, y1, x0, x1;
    float ly, lx;
    float sy = (H > 1) ? (float)(Hp - 1) / (float)(H - 1) : 0.f;
    float sx = (W > 1) ? (float)(Wp - 1) / (float)(W - 1) : 0.f;
    bilin_src_ac(y, sy, Hp, y0, y1, ly);
    bilin_src_ac(x, sx, Wp, x0, x1, lx);
    float hy = 1.f - ly, hx = 1.f - lx;
    const float* f = flow_prev;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      float v = hy * (hx * f[(y0 * Wp + x0) * 2 + c] + lx * f[(y0 * Wp + x1) * 2 + c]) +
                ly * (hx * f[(y1 * Wp + x0) * 2 + c] + lx * f[(y1 * Wp + x1) * 2 + c]);
      if (c == 0) fx = v * 2.0f; else fy = v * 2.0f;
    }
  }
  flow_up[(size_t)p * 2 + 0] = fx;
  flow_up[(size_t)p * 2 + 1] = fy;
  // flow_warp(..., padding_mode='border', align_corners=True): flow_warp.py:36-46
  float gx = 2.0f * ((float)x + fx) / (float)max(W - 1, 1) - 1.0f;
  float gy = 2.0f * ((float)y + fy) / (float)max(H - 1, 1) - 1.0f;
  float px = (gx + 1.f) * 0.5f * (float)(W - 1);
  float py = (gy + 1.f) * 0.5f * (float)(H - 1);
  px = fminf(fmaxf(px, 0.f), (float)(W - 1));
  py = fminf(fmaxf(py, 0.f), (float)(H - 1));
  float x0f = floorf(px), y0f = floorf(py);
  int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
  float wx1 = px - x0f, wx0 = 1.f - wx1, wy1 = py - y0f, wy0 = 1.f - wy1;
  T* o = out8 + (size_t)p * 8;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    o[c] = from_f<T>(ref[(size_t)p * 3 + c]);
    float v = 0.f;
    // nw, ne, sw, se (aten grid_sampler order)
    v += supp[((size_t)y0 * W + x0) * 3 + c] * (wx0 * wy0);
    if (x1 <= W - 1) v += supp[((size_t)y0 * W + x1) * 3 + c] * (wx1 * wy0);
    if (y1 <= H - 1) v += supp[((size_t)y1 * W + x0) * 3 + c] * (wx0 * wy1);
    if (x1 <= W - 1 && y1 <= H - 1) v += supp[((size_t)y1 * W + x1) * 3 + c] * (wx1 * wy1);
    o[3 + c] = from_f<T>(v);
  }
  o[6] = from_f<T>(fx);
  o[7] = from_f<T>(fy);
}

__global__ void flow_resize_kernel(const float* __restrict__ flow, int H, int W,
                                   float* __restrict__ out, int h, int w) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= h * w) return;
  int y = p / w, x = p % w;
  int y0, y1, x0, x1;
  float ly, lx;
  bilin_src(y, (float)H / (float)h, H, y0, y1, ly);
  bilin_src(x, (float)W / (float)w, W, x0, x1, lx);
  float hy = 1.f - ly, hx = 1.f - lx;
  float sc[2] = {(float)w / (float)W, (float)h / (float)H};
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    float v = hy * (hx * flow[((size_t)y0 * W + x0) * 2 + c] + lx * flow[((size_t)y0 * W + x1) * 2 + c]) +
              ly * (hx * flow[((size_t)y1 * W + x0) * 2 + c] + lx * flow[((size_t)y1 * W + x1) * 2 + c]);
    out[(size_t)p * 2 + c] = v * sc[c];
  }
}

// ---------------------------------------------------------------------------------------------
// rv_warp : grid_sample(bilinear, zeros, align_corners=False) with the reference grid
// ---------------------------------------------------------------------------------------------
// F.interpolate(flow, x2, bilinear, align_corners=True) * 2 at pixel (Y, X) of the Ho x Wo = 2 hf x 2 wf grid; at(y, x) reads
// the hf x wf flow (global memory, or warp3_kernel's shared flow tile)
template <typename F>
__device__ __forceinline__ float2 flow_up2_at(int Y, int X, int Ho, int Wo, int hf, int wf, F at) {
  int y0, y1, x0, x1;
  float ly, lx;
  const float sy = (Ho > 1) ? (float)(hf - 1) / (float)(Ho - 1) : 0.f;
  const float sx = (Wo > 1) ? (float)(wf - 1) / (float)(Wo - 1) : 0.f;
  bilin_src_ac(Y, sy, hf, y0, y1, ly);
  bilin_src_ac(X, sx, wf, x0, x1, lx);
  const float hy = 1.f - ly, hx = 1.f - lx;
  const float2 a = at(y0, x0), b = at(y0, x1), c = at(y1, x0), d = at(y1, x1);
  return make_float2((hy * (hx * a.x + lx * b.x) + ly * (hx * c.x + lx * d.x)) * 2.0f,
                     (hy * (hx * a.y + lx * b.y) + ly * (hx * c.y + lx * d.y)) * 2.0f);
}

// the reference grid (models/utils.py:36-43) at pixel (Xi, Yi) of a Wo x Ho map moved by (fx, fy), unnormalised for a Wi x Hi
// source (aten grid_sampler_unnormalize, align_corners=False): top-left corner (ix, iy) and the weights of nw, ne, sw, se
__device__ __forceinline__ void warp_pos(float fx, float fy, int Wo, int Ho, int Wi, int Hi, int Xi, int Yi, int& ix, int& iy,
                                         float4& wq) {
  float gx = linspace_m1_1(Xi, Wo) + fx / (((float)Wi - 1.0f) / 2.0f);
  float gy = linspace_m1_1(Yi, Ho) + fy / (((float)Hi - 1.0f) / 2.0f);
  float px = ((gx + 1.f) * (float)Wi - 1.f) / 2.f;
  float py = ((gy + 1.f) * (float)Hi - 1.f) / 2.f;
  float xw = floorf(px), yn = floorf(py);
  ix = (int)xw;
  iy = (int)yn;
  float xe = xw + 1.f, ys = yn + 1.f;
  wq = make_float4((xe - px) * (ys - py), (px - xw) * (ys - py), (xe - px) * (py - yn), (px - xw) * (py - yn));
}

// warp_pos for the branch-free gathers: weights of corners outside the source zeroed, corner pixel offsets clamped into it
__device__ __forceinline__ void warp_corner(float fx, float fy, int Wo, int Ho, int Wi, int Hi, int Xi, int Yi, float4& wq, int4& off) {
  int ix, iy;
  warp_pos(fx, fy, Wo, Ho, Wi, Hi, Xi, Yi, ix, iy, wq);
  const bool x0ok = ix >= 0 && ix < Wi, x1ok = ix + 1 >= 0 && ix + 1 < Wi;
  const bool y0ok = iy >= 0 && iy < Hi, y1ok = iy + 1 >= 0 && iy + 1 < Hi;
  if (!(y0ok && x0ok)) wq.x = 0.f;
  if (!(y0ok && x1ok)) wq.y = 0.f;
  if (!(y1ok && x0ok)) wq.z = 0.f;
  if (!(y1ok && x1ok)) wq.w = 0.f;
  const int cx0 = clampi(ix, 0, Wi - 1), cx1 = clampi(ix + 1, 0, Wi - 1);
  const int cy0 = clampi(iy, 0, Hi - 1), cy1 = clampi(iy + 1, 0, Hi - 1);
  off = make_int4(cy0 * Wi + cx0, cy0 * Wi + cx1, cy1 * Wi + cx0, cy1 * Wi + cx1);
}

// generic path: one thread = one output pixel x one channel vector
template <typename T, int V>
__global__ void warp_kernel(const T* __restrict__ src, int Hi, int Wi, int C,
                            const float* __restrict__ flow, int hf, int wf, int flow_up2,
                            T* __restrict__ out) {
  const int Ho = flow_up2 ? 2 * hf : hf, Wo = flow_up2 ? 2 * wf : wf;
  const int cv = C / V;
  src += (size_t)blockIdx.z * Hi * Wi * C;           // image blockIdx.z of a batch (rv_warp_batched)
  flow += (size_t)blockIdx.z * hf * wf * 2;
  out += (size_t)blockIdx.z * Ho * Wo * C;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)Ho * Wo * cv) return;
  int vc = (int)(i % cv);
  int p = (int)(i / cv);
  int Y = p / Wo, X = p % Wo;
  const float2* f2 = reinterpret_cast<const float2*>(flow);
  float2 f;
  if (flow_up2) f = flow_up2_at(Y, X, Ho, Wo, hf, wf, [&](int y, int x) { return __ldg(f2 + y * wf + x); });
  else f = __ldg(f2 + p);
  int ix, iy;
  float4 wq;
  warp_pos(f.x, f.y, Wo, Ho, Wi, Hi, X, Y, ix, iy, wq);
  float acc[V];
#pragma unroll
  for (int k = 0; k < V; ++k) acc[k] = 0.f;
  const bool x0ok = ix >= 0 && ix < Wi, x1ok = ix + 1 >= 0 && ix + 1 < Wi;
  const bool y0ok = iy >= 0 && iy < Hi, y1ok = iy + 1 >= 0 && iy + 1 < Hi;
  const T* base = src + (size_t)vc * V;
  if (y0ok && x0ok) {
    Vec<T, V> t = ldv<T, V>(base + ((size_t)iy * Wi + ix) * C);
#pragma unroll
    for (int k = 0; k < V; ++k) acc[k] += to_f(t.v[k]) * wq.x;
  }
  if (y0ok && x1ok) {
    Vec<T, V> t = ldv<T, V>(base + ((size_t)iy * Wi + ix + 1) * C);
#pragma unroll
    for (int k = 0; k < V; ++k) acc[k] += to_f(t.v[k]) * wq.y;
  }
  if (y1ok && x0ok) {
    Vec<T, V> t = ldv<T, V>(base + ((size_t)(iy + 1) * Wi + ix) * C);
#pragma unroll
    for (int k = 0; k < V; ++k) acc[k] += to_f(t.v[k]) * wq.z;
  }
  if (y1ok && x1ok) {
    Vec<T, V> t = ldv<T, V>(base + ((size_t)(iy + 1) * Wi + ix + 1) * C);
#pragma unroll
    for (int k = 0; k < V; ++k) acc[k] += to_f(t.v[k]) * wq.w;
  }
  Vec<T, V> o;
#pragma unroll
  for (int k = 0; k < V; ++k) o.v[k] = from_f<T>(acc[k]);
  stv<T, V>(out + (size_t)p * C + (size_t)vc * V, o);
}

// Vector variant used for feature maps: phase 1 computes, once per output pixel, the four corner
// offsets (clamped) and weights (zeroed when the corner is outside the image) into shared memory;
// phase 2 is a branch-free 4-tap gather with one thread per (pixel, 16-byte channel vector), so global
// loads and stores stay fully coalesced along the NHWC channel axis.
template <typename T, int V>
__global__ void __launch_bounds__(256) warp_vec_kernel(const T* __restrict__ src, int Hi, int Wi, int C,
                                                       const float* __restrict__ flow, int hf, int wf,
                                                       int flow_up2, T* __restrict__ out, int ppb) {
  __shared__ float4 s_w[256];
  __shared__ int4 s_o[256];
  const int Ho = flow_up2 ? 2 * hf : hf, Wo = flow_up2 ? 2 * wf : wf;
  const int cv = C / V;             // threads per pixel
  src += (size_t)blockIdx.z * Hi * Wi * C;           // image blockIdx.z of a batch (rv_warp_batched)
  flow += (size_t)blockIdx.z * hf * wf * 2;
  out += (size_t)blockIdx.z * Ho * Wo * C;
  const int npix = Ho * Wo;
  const int p0 = blockIdx.x * ppb;
  if (threadIdx.x < ppb && p0 + threadIdx.x < npix) {
    const int p = p0 + threadIdx.x;
    const int Y = p / Wo, X = p - Y * Wo;
    const float2* f2 = reinterpret_cast<const float2*>(flow);
    float2 f;
    if (flow_up2) f = flow_up2_at(Y, X, Ho, Wo, hf, wf, [&](int y, int x) { return __ldg(f2 + y * wf + x); });
    else f = __ldg(f2 + p);
    float4 wq;
    int4 off;
    warp_corner(f.x, f.y, Wo, Ho, Wi, Hi, X, Y, wq, off);
    s_w[threadIdx.x] = wq;
    s_o[threadIdx.x] = off;
  }
  __syncthreads();
  const int pl = threadIdx.x / cv, vc = threadIdx.x - pl * cv;
  if (pl >= ppb || p0 + pl >= npix) return;
  const float4 wq = s_w[pl];
  const int4 o = s_o[pl];
  const T* base = src + (size_t)vc * V;
  const Vec<T, V> t0 = ldv<T, V>(base + (size_t)o.x * C), t1 = ldv<T, V>(base + (size_t)o.y * C),
                  t2 = ldv<T, V>(base + (size_t)o.z * C), t3 = ldv<T, V>(base + (size_t)o.w * C);
  stv<T, V>(out + (size_t)(p0 + pl) * C + (size_t)vc * V, blend4<T, V>(t0, t1, t2, t3, wq));
}


// ---------------------------------------------------------------------------------------------
// rv_warp3 : the three warps of one propagation step in ONE launch (RefVSR.py:216-220,256-260):
//   feat (h,w,C), conf (h,w) with the LR flow, feat_UP (2h,2w,C) with the x2 bilinear (align_corners=True) * 2 flow.
// One CTA = one 8 x 16 LR tile = 16 x 32 pixels of the 2x grid.  Phase 0 stages the LR flow tile (+1 halo) in shared
// memory (one coalesced read of the flow for all three warps), phase 1 computes for every output pixel of the tile the four
// corner offsets (clamped) and weights (zero outside the image) into shared memory, phase 2 is the branch-free 4-tap gather
// with one thread per (pixel, 16-byte channel vector): coalesced along the NHWC channel axis, and - because the tile is 2-D -
// the corner rows shared by vertically adjacent output pixels are fetched from L2 once per CTA (L1 hits), not once per row.
// Same arithmetic as warp_kernel / warp_vec_kernel (bit-identical results).  Measured at 270x480x48 bf16 on an H100 80GB HBM3
// at a 400 W limit (tools/pointwise_bench.py): 52.7 us for 8 x 16 and 4 x 16 tiles, 57.3 us for 2 x 16 - every CTA pays the
// flow-tile load and two barriers before its first gather, so the smallest tiles lose.
// ---------------------------------------------------------------------------------------------
constexpr int W3_TH = 8, W3_TW = 16;

template <typename T, int CV>      // CV = C / V (16-byte vectors per pixel) when known at compile time, 0 = run-time
__global__ void __launch_bounds__(256) warp3_kernel(const T* __restrict__ feat, const T* __restrict__ featUP,
                                                    const float* __restrict__ conf, const float* __restrict__ flow, int h, int w,
                                                    int C, T* __restrict__ o_feat, T* __restrict__ o_featUP,
                                                    float* __restrict__ o_conf) {
  constexpr int V = 16 / (int)sizeof(T);
  constexpr int NLR = W3_TH * W3_TW, NUP = 4 * NLR;
  __shared__ float2 s_flow[(W3_TH + 2) * (W3_TW + 2)];
  __shared__ float4 s_w[NLR + NUP];
  __shared__ int4 s_o[NLR + NUP];
  const int tiles_x = (w + W3_TW - 1) / W3_TW;
  const int ty0 = (blockIdx.x / tiles_x) * W3_TH, tx0 = (blockIdx.x % tiles_x) * W3_TW;
  const int H2 = 2 * h, W2 = 2 * w;
  {                                                  // image blockIdx.z of a batch (rv_warp3_batched)
    const size_t px = (size_t)blockIdx.z * h * w;
    feat += px * C; o_feat += px * C; featUP += 4 * px * C; o_featUP += 4 * px * C;
    conf += px; o_conf += px; flow += 2 * px;
  }
  // ---- phase 0: LR flow tile with a one-pixel halo (the x2 flow of a tile reads rows / columns ty0 - 1 .. ty0 + TH)
  for (int i = threadIdx.x; i < (W3_TH + 2) * (W3_TW + 2); i += blockDim.x) {
    const int yy = clampi(ty0 - 1 + i / (W3_TW + 2), 0, h - 1), xx = clampi(tx0 - 1 + i % (W3_TW + 2), 0, w - 1);
    s_flow[i] = __ldg(reinterpret_cast<const float2*>(flow) + (size_t)yy * w + xx);
  }
  __syncthreads();
  auto flow_at = [&](int yy, int xx) -> float2 {      // (yy, xx) within [ty0 - 1, ty0 + TH] x [tx0 - 1, tx0 + TW] after clamping
    return s_flow[(clampi(yy, 0, h - 1) - (ty0 - 1)) * (W3_TW + 2) + (clampi(xx, 0, w - 1) - (tx0 - 1))];
  };
  // ---- phase 1: corner offsets + weights
  for (int i = threadIdx.x; i < NLR + NUP; i += blockDim.x) {
    float4 wq = make_float4(0.f, 0.f, 0.f, 0.f);
    int4 off = make_int4(0, 0, 0, 0);
    if (i < NLR) {
      const int Y = ty0 + i / W3_TW, X = tx0 + i % W3_TW;
      if (Y < h && X < w) {
        const float2 f = flow_at(Y, X);
        warp_corner(f.x, f.y, w, h, w, h, X, Y, wq, off);
      }
    } else {
      const int j = i - NLR;
      const int Y = 2 * ty0 + j / (2 * W3_TW), X = 2 * tx0 + j % (2 * W3_TW);
      if (Y < H2 && X < W2) {
        const float2 f = flow_up2_at(Y, X, H2, W2, h, w, flow_at);
        warp_corner(f.x, f.y, W2, H2, W2, H2, X, Y, wq, off);
      }
    }
    s_w[i] = wq;
    s_o[i] = off;
  }
  __syncthreads();
  // ---- phase 2: gathers.  item = (pixel, vector); the 2x feature first (largest), then the LR feature, then conf.
  const int cv = CV > 0 ? CV : C / V;          // (compile-time constant for the shipped widths: no integer divisions below)
  auto gather = [&](const T* __restrict__ src, T* __restrict__ dst, int pl0, int npl, int tw, int Y0, int X0, int Hh, int Ww) {
    // two (pixel, vector) items per thread and iteration: all eight 16-byte loads are issued before the first use
    const int nit = npl * cv;
    for (int it = threadIdx.x; it < nit; it += 2 * blockDim.x) {
      const int itb = it + blockDim.x;
      const int pla = it / cv, vca = it - pla * cv;
      const int plb = (itb < nit) ? itb / cv : pla, vcb = (itb < nit) ? itb - plb * cv : vca;
      const int Ya = Y0 + pla / tw, Xa = X0 + pla % tw, Yb = Y0 + plb / tw, Xb = X0 + plb % tw;
      const bool oka = Ya < Hh && Xa < Ww, okb = itb < nit && Yb < Hh && Xb < Ww;
      const float4 wa = s_w[pl0 + pla], wb = s_w[pl0 + plb];
      const int4 oa = s_o[pl0 + pla], ob = s_o[pl0 + plb];            // (offsets of out-of-image pixels are 0: safe to read)
      // addresses as 32-bit indices of 16-byte vectors (pixel * cv + vector; the launcher checks that they fit)
      const Vec<T, V> a0 = ldvi<T, V>(src, oa.x * cv + vca), a1 = ldvi<T, V>(src, oa.y * cv + vca),
                      a2 = ldvi<T, V>(src, oa.z * cv + vca), a3 = ldvi<T, V>(src, oa.w * cv + vca);
      const Vec<T, V> b0 = ldvi<T, V>(src, ob.x * cv + vcb), b1 = ldvi<T, V>(src, ob.y * cv + vcb),
                      b2 = ldvi<T, V>(src, ob.z * cv + vcb), b3 = ldvi<T, V>(src, ob.w * cv + vcb);
      if (oka) stvi<T, V>(dst, (Ya * Ww + Xa) * cv + vca, blend4<T, V>(a0, a1, a2, a3, wa));
      if (okb) stvi<T, V>(dst, (Yb * Ww + Xb) * cv + vcb, blend4<T, V>(b0, b1, b2, b3, wb));
    }
  };
  gather(featUP, o_featUP, NLR, NUP, 2 * W3_TW, 2 * ty0, 2 * tx0, H2, W2);
  gather(feat, o_feat, 0, NLR, W3_TW, ty0, tx0, h, w);
  for (int i = threadIdx.x; i < NLR; i += blockDim.x) {
    const int Y = ty0 + i / W3_TW, X = tx0 + i % W3_TW;
    if (Y < h && X < w) {
      const float4 wq = s_w[i];
      const int4 o = s_o[i];
      // same accumulation order as warp_kernel<float, 1> (taps nw, ne, sw, se added one by one)
      float acc = 0.f;
      acc += __ldg(conf + o.x) * wq.x;
      acc += __ldg(conf + o.y) * wq.y;
      acc += __ldg(conf + o.z) * wq.z;
      acc += __ldg(conf + o.w) * wq.w;
      o_conf[(size_t)Y * w + X] = acc;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// rv_patch_pack : one warp per pixel
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int reflect1(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

template <typename T>
__global__ void patch_pack_kernel(const T* __restrict__ feat, int H, int W, int C, int mode,
                                  __half* __restrict__ out, int kpad) {
  const int K = C * 9;
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (warp >= H * W) return;
  int y = warp / W, x = warp % W;
  float vals[8];  // K <= 256
  float ss = 0.f;
  int nk = 0;
  for (int k = lane; k < K; k += 32, ++nk) {
    int c = k / 9, t = k % 9, ky = t / 3, kx = t % 3;
    int sy = reflect1(y + ky - 1, H), sx = reflect1(x + kx - 1, W);
    float v = to_f(feat[((size_t)sy * W + sx) * C + c]);
    vals[nk] = v;
    ss += v * v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  float denom = fmaxf(sqrtf(ss), 1e-12f);
  __half* row = out + (size_t)warp * kpad;
  // zero the padding columns
  int used = (mode == 0) ? K : 3 * K;
  for (int k = used + lane; k < kpad; k += 32) row[k] = __float2half_rn(0.f);
  nk = 0;
  for (int k = lane; k < K; k += 32, ++nk) {
    float v = vals[nk] / denom * 64.0f;
    __half hi = __float2half_rn(v);
    __half lo = __float2half_rn(v - __half2float(hi));
    if (mode == 0) {
      row[k] = hi;
    } else if (mode == 1) {
      row[k] = hi; row[K + k] = lo; row[2 * K + k] = hi;
    } else {
      row[k] = hi; row[K + k] = hi; row[2 * K + k] = lo;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// rv_gather_blocks / rv_aligned_sample
// ---------------------------------------------------------------------------------------------
template <int BYTES>
__global__ void gather_blocks_kernel(const uint8_t* __restrict__ value, int Hv, int Wv, int rowbytes,
                                     const int32_t* __restrict__ idx, int hq, int wq, int ks,
                                     uint8_t* __restrict__ out) {
  const int Ho = ks * hq, Wo = ks * wq;
  const int nv = rowbytes / BYTES;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)Ho * Wo * nv) return;
  int v = (int)(i % nv);
  int p = (int)(i / nv);
  int Y = p / Wo, X = p % Wo;
  int ci = Y / ks, a = Y % ks, cj = X / ks, b = X % ks;
  int r = __ldg(idx + ci * wq + cj);
  int wvk = Wv / ks;
  int ry = r / wvk, rx = r % wvk;
  const uint8_t* s = value + ((size_t)(ks * ry + a) * Wv + (ks * rx + b)) * rowbytes + (size_t)v * BYTES;
  uint8_t* d = out + (size_t)p * rowbytes + (size_t)v * BYTES;
  if constexpr (BYTES == 16) *reinterpret_cast<uint4*>(d) = __ldg(reinterpret_cast<const uint4*>(s));
  else if constexpr (BYTES == 8) *reinterpret_cast<uint2*>(d) = __ldg(reinterpret_cast<const uint2*>(s));
  else if constexpr (BYTES == 4) *reinterpret_cast<uint32_t*>(d) = __ldg(reinterpret_cast<const uint32_t*>(s));
  else *reinterpret_cast<uint16_t*>(d) = *reinterpret_cast<const uint16_t*>(s);
}

// 16-byte rows, ks = 1 / 2 / 4: one thread = one (cell, 16-byte vector) - the index lookup and its division are done once per
// cell and the thread then moves the ks * ks pixels of the cell (the per-output-vector version above spends ~190 instructions,
// six integer divisions among them, on every 16 bytes).  blockIdx.y = cell row.  Pure copies: bit-identical.
template <int KS, int NVC>
__global__ void __launch_bounds__(256) gather_cells_kernel(const uint4* __restrict__ value, int Wv, int nv_rt,
                                                           const int32_t* __restrict__ idx, int wq, uint4* __restrict__ out) {
  const int nv = NVC > 0 ? NVC : nv_rt;
  const int j = blockIdx.x * 256 + threadIdx.x;
  const int cj = j / nv, v = j - cj * nv;
  if (cj >= wq) return;
  const int ci = blockIdx.y;
  const int r = __ldg(idx + ci * wq + cj);
  const int wvk = Wv / KS;
  const int ry = r / wvk, rx = r - ry * wvk;
  const int Wo = KS * wq;
  const uint4* s = value + ((size_t)(KS * ry) * Wv + KS * rx) * nv + v;
  uint4* d = out + ((size_t)(KS * ci) * Wo + KS * cj) * nv + v;
  uint4 t[KS * KS];
#pragma unroll
  for (int a = 0; a < KS; ++a)
#pragma unroll
    for (int b = 0; b < KS; ++b) t[a * KS + b] = __ldg(s + ((size_t)a * Wv + b) * nv);
#pragma unroll
  for (int a = 0; a < KS; ++a)
#pragma unroll
    for (int b = 0; b < KS; ++b) d[((size_t)a * Wo + b) * nv] = t[a * KS + b];
}

// space-to-depth (factor 2): out[(Y,X)][(ry*2+rx)*C + c] = in[(2Y+ry, 2X+rx)][c]; 16-byte vectors
__global__ void space_to_depth2_kernel(const uint4* __restrict__ src, int H, int W, int cv,
                                       uint4* __restrict__ out) {
  const int Ho = H / 2, Wo = W / 2;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)Ho * Wo * 4 * cv) return;
  int v = (int)(i % cv);
  long long r = i / cv;
  int sub = (int)(r % 4);
  int p = (int)(r / 4);
  int Y = p / Wo, X = p % Wo;
  int ry = sub >> 1, rx = sub & 1;
  out[((size_t)p * 4 + sub) * cv + v] = __ldg(src + ((size_t)(2 * Y + ry) * W + (2 * X + rx)) * cv + v);
}

// AlignedConv2d's sample of cell (ci, cj) of a ks x ks block grid over the H x W map, at offset (u, v) from the cell's centre
// (half = ks / 2) before the cell's rotation (cs, sn): the position, clamped into the reflection-padded map, gives the weights of
// the corners (lt, rb, lb, rt) and their source rows r0, r1 and columns c0, c1 (ReflectionPad2d(1)).  FMA_AS_GENERIC spells out
// the contraction the compiler picks for the rotation in aligned_sample_kernel, where the offsets are run-time values: with them
// known at compile time it would fuse the other product of each pair (its products of v are shared across rows).
template <bool FMA_AS_GENERIC>
__device__ __forceinline__ void aligned_tap(float u, float v, float cs, float sn, float half, int ci, int cj, int ks, int H, int W,
                                            float4& g, int& r0, int& r1, int& c0, int& c1) {
  const int Hp = H + 2, Wp = W + 2;
  float rr, cc;
  if constexpr (FMA_AS_GENERIC) {
    rr = __fmaf_rn(u, cs, -__fmul_rn(v, sn));
    cc = __fmaf_rn(v, cs, __fmul_rn(u, sn));
  } else {
    rr = u * cs - v * sn;
    cc = u * sn + v * cs;
  }
  float pr = rr + half + (float)(1 + ci * ks);
  float pc = cc + half + (float)(1 + cj * ks);
  float ltr = floorf(pr), ltc = floorf(pc);
  float rbr = ltr + 1.f, rbc = ltc + 1.f;
  const float Hm = (float)(Hp - 1), Wm = (float)(Wp - 1);
  ltr = fminf(fmaxf(ltr, 0.f), Hm); rbr = fminf(fmaxf(rbr, 0.f), Hm);
  ltc = fminf(fmaxf(ltc, 0.f), Wm); rbc = fminf(fmaxf(rbc, 0.f), Wm);
  pr = fminf(fmaxf(pr, 0.f), Hm); pc = fminf(fmaxf(pc, 0.f), Wm);
  g = make_float4((1.f + (ltr - pr)) * (1.f + (ltc - pc)), (1.f - (rbr - pr)) * (1.f - (rbc - pc)),
                  (1.f + (ltr - pr)) * (1.f - (rbc - pc)), (1.f - (rbr - pr)) * (1.f + (ltc - pc)));
  // padded index -> source index
  r0 = reflect1((int)ltr - 1, H); r1 = reflect1((int)rbr - 1, H);
  c0 = reflect1((int)ltc - 1, W); c1 = reflect1((int)rbc - 1, W);
}

template <typename T, int V>
__global__ void aligned_sample_kernel(const T* __restrict__ x, int h, int w, int ks, int C,
                                      const float* __restrict__ affine, T* __restrict__ out) {
  const int H = ks * h, W = ks * w;
  const int cv = C / V;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)H * W * cv) return;
  int vc = (int)(i % cv);
  int p = (int)(i / cv);
  int Y = p / W, X = p % W;
  int ci = Y / ks, a = Y % ks, cj = X / ks, b = X % ks;
  const float* af = affine + ((size_t)ci * w + cj) * 3;
  float s_x = af[0], s_y = af[1], th = (af[2] - 1.0f) * 1.0472f;
  float half = (float)((ks - 1) / 2) + 0.5f;  // -(ks-1)//2 - 0.5 + a  ==  a - half
  float u = ((float)a - half) * s_x, v = ((float)b - half) * s_y;
  float cs = cosf(th), sn = sinf(th);
  float4 g;
  int r0, r1, c0, c1;
  aligned_tap<false>(u, v, cs, sn, half, ci, cj, ks, H, W, g, r0, r1, c0, c1);
  const T* base = x + (size_t)vc * V;
  Vec<T, V> t_lt = ldv<T, V>(base + ((size_t)r0 * W + c0) * C);
  Vec<T, V> t_rb = ldv<T, V>(base + ((size_t)r1 * W + c1) * C);
  Vec<T, V> t_lb = ldv<T, V>(base + ((size_t)r0 * W + c1) * C);
  Vec<T, V> t_rt = ldv<T, V>(base + ((size_t)r1 * W + c0) * C);
  Vec<T, V> o;
#pragma unroll
  for (int k = 0; k < V; ++k)
    o.v[k] = from_f<T>(g.x * to_f(t_lt.v[k]) + g.y * to_f(t_rb.v[k]) + g.z * to_f(t_lb.v[k]) +
                       g.w * to_f(t_rt.v[k]));
  stv<T, V>(out + (size_t)p * C + (size_t)vc * V, o);
}

// ks = 2 (every x4 model) and ks = 4 (aa2 of the x2 models, aa1 of the flag_HD_in models) on 2-D tiles of cells: 4 x 16 cells =
// 8 x 32 output pixels at ks 2 (41.2 us vs 43.0 us for 8 x 16 cells at 270x480x48 bf16, H100 80GB HBM3 at a 400 W limit), 8 x 8
// cells = 32 x 32 pixels at ks 4.  Phase 1 evaluates the ks * ks sampling positions of a cell once (sin / cos once per cell
// instead of once per channel vector of every pixel) into shared memory, phase 2 is the same branch-free 4-tap gather as
// warp3_kernel.  At ks 4 the result is bit-identical to aligned_sample_kernel: the rotation and the blend are written out in the
// order the compiler contracts that kernel's expressions; at ks 2 the compiler contracts them.
template <int KS, typename T, int CV>
__device__ __forceinline__ void aligned_sample_tiled(const T* __restrict__ x, int h, int w, int C, const float* __restrict__ affine,
                                                     T* __restrict__ out) {
  constexpr int V = 16 / (int)sizeof(T);
  constexpr int AS_TH = KS == 2 ? 4 : 8, AS_TW = KS == 2 ? 16 : 8, NC = AS_TH * AS_TW, NP = KS * KS * NC, PW = KS * AS_TW;
  __shared__ float4 s_w[NP];
  __shared__ int4 s_o[NP];
  const int H = KS * h, W = KS * w;
  const int tiles_x = (w + AS_TW - 1) / AS_TW;
  const int ci0 = (blockIdx.x / tiles_x) * AS_TH, cj0 = (blockIdx.x % tiles_x) * AS_TW;
  const int Y0 = KS * ci0, X0 = KS * cj0;
  for (int c = threadIdx.x; c < NC; c += blockDim.x) {
    const int li = c / AS_TW, lj = c % AS_TW;
    const int ci = ci0 + li, cj = cj0 + lj;
    if (ci >= h || cj >= w) continue;                       // (entries of cells outside the image are never read)
    const float* af = affine + ((size_t)ci * w + cj) * 3;
    const float s_x = af[0], s_y = af[1], th = (af[2] - 1.0f) * 1.0472f;
    const float half = (float)((KS - 1) / 2) + 0.5f;
    const float cs = cosf(th), sn = sinf(th);
#pragma unroll
    for (int a = 0; a < KS; ++a)
#pragma unroll
      for (int b = 0; b < KS; ++b) {
        const float u = ((float)a - half) * s_x, v = ((float)b - half) * s_y;
        float4 g;
        int r0, r1, c0, c1;
        aligned_tap<KS == 4>(u, v, cs, sn, half, ci, cj, KS, H, W, g, r0, r1, c0, c1);
        const int e = (KS * li + a) * PW + KS * lj + b;
        s_w[e] = g;
        s_o[e] = make_int4(r0 * W + c0, r1 * W + c1, r0 * W + c1, r1 * W + c0);
      }
  }
  __syncthreads();
  const int cv = CV > 0 ? CV : C / V;
  for (int it = threadIdx.x; it < NP * cv; it += blockDim.x) {
    const int pl = it / cv, vc = it - pl * cv;
    const int Y = Y0 + pl / PW, X = X0 + pl % PW;
    if (Y >= H || X >= W) continue;
    const float4 g = s_w[pl];
    const int4 o = s_o[pl];
    const Vec<T, V> t_lt = ldvi<T, V>(x, o.x * cv + vc), t_rb = ldvi<T, V>(x, o.y * cv + vc),
                    t_lb = ldvi<T, V>(x, o.z * cv + vc), t_rt = ldvi<T, V>(x, o.w * cv + vc);
    stvi<T, V>(out, (Y * W + X) * cv + vc,
               KS == 4 ? blend4_as_generic<T, V>(t_lt, t_rb, t_lb, t_rt, g) : blend4<T, V>(t_lt, t_rb, t_lb, t_rt, g));
  }
}

// one kernel per ks, so that a profile names the path that ran
template <typename T, int CV>
__global__ void __launch_bounds__(256) aligned_sample2_kernel(const T* __restrict__ x, int h, int w, int C,
                                                              const float* __restrict__ affine, T* __restrict__ out) {
  aligned_sample_tiled<2, T, CV>(x, h, w, C, affine, out);
}
template <typename T, int CV>
__global__ void __launch_bounds__(256) aligned_sample4_kernel(const T* __restrict__ x, int h, int w, int C,
                                                              const float* __restrict__ affine, T* __restrict__ out) {
  aligned_sample_tiled<4, T, CV>(x, h, w, C, affine, out);
}

// ---------------------------------------------------------------------------------------------
// bicubic helpers (aten upsample_bicubic2d, align_corners=False, explicit scale factor)
// ---------------------------------------------------------------------------------------------
// planar source, bounded access
__device__ __forceinline__ float bicubic_planar(const float* __restrict__ s, int H, int W, int Y,
                                                int X, float inv_scale) {
  float ry = inv_scale * ((float)Y + 0.5f) - 0.5f, rx = inv_scale * ((float)X + 0.5f) - 0.5f;
  float fy = floorf(ry), fx = floorf(rx);
  int iy = (int)fy, ix = (int)fx;
  float wy[4], wx[4];
  cubic_weights(ry - fy, wy);
  cubic_weights(rx - fx, wx);
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    int yy = clampi(iy - 1 + j, 0, H - 1);
    const float* r = s + (size_t)yy * W;
    float row = wx[0] * r[clampi(ix - 1, 0, W - 1)] + wx[1] * r[clampi(ix, 0, W - 1)] +
                wx[2] * r[clampi(ix + 1, 0, W - 1)] + wx[3] * r[clampi(ix + 2, 0, W - 1)];
    acc += wy[j] * row;
  }
  return acc;
}

__global__ void resize_planes_kernel(const float* __restrict__ src, int n, int H, int W, float inv_scale, int Ho,
                                     int Wo, int mode, int clamp01, float* __restrict__ out) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n * Ho * Wo) return;
  int c = (int)(i / ((long long)Ho * Wo));
  int p = (int)(i - (long long)c * Ho * Wo);
  int Y = p / Wo, X = p - Y * Wo;
  const float* s = src + (size_t)c * H * W;
  float v;
  if (mode == 0) {
    v = bicubic_planar(s, H, W, Y, X, inv_scale);
  } else {
    int sy = min((int)floorf((float)Y * inv_scale), H - 1), sx = min((int)floorf((float)X * inv_scale), W - 1);
    v = s[(size_t)sy * W + sx];
  }
  if (clamp01) v = fminf(fmaxf(v, 0.f), 1.f);
  out[i] = v;
}

template <typename T>
__global__ void maxpool2_kernel(const T* __restrict__ src, int H, int W, int C, T* __restrict__ out) {
  int Ho = H / 2, Wo = W / 2;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)Ho * Wo * C) return;
  int c = (int)(i % C);
  int p = (int)(i / C);
  int y = p / Wo, x = p - y * Wo;
  const T* s = src + ((size_t)(2 * y) * W + 2 * x) * C + c;
  float v = fmaxf(fmaxf(to_f(s[0]), to_f(s[C])), fmaxf(to_f(s[(size_t)W * C]), to_f(s[(size_t)W * C + C])));
  out[i] = from_f<T>(v);
}

template <typename T>
__global__ void bicubic_up2_image_kernel(const float* __restrict__ src, int H, int W,
                                         T* __restrict__ out, int out_c) {
  int Ho = 2 * H, Wo = 2 * W;
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Ho * Wo) return;
  int Y = p / Wo, X = p % Wo;
  T* o = out + (size_t)p * out_c;
  for (int c = 0; c < out_c; ++c)
    o[c] = from_f<T>(c < 3 ? bicubic_planar(src + (size_t)c * H * W, H, W, Y, X, 0.5f) : 0.f);
}

template <typename T>
__global__ void conf_pair_kernel(const float* __restrict__ a, const float* __restrict__ b, int h,
                                 int w, int up2, T* __restrict__ out, int out_c) {
  int Ho = up2 ? 2 * h : h, Wo = up2 ? 2 * w : w;
  a += (size_t)blockIdx.z * h * w;                   // image blockIdx.z of a batch (rv_conf_pair_batched)
  b += (size_t)blockIdx.z * h * w;
  out += (size_t)blockIdx.z * Ho * Wo * out_c;
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Ho * Wo) return;
  float va, vb;
  if (up2) {
    int Y = p / Wo, X = p % Wo;
    va = fminf(fmaxf(bicubic_planar(a, h, w, Y, X, 0.5f), 0.f), 1.f);
    vb = fminf(fmaxf(bicubic_planar(b, h, w, Y, X, 0.5f), 0.f), 1.f);
  } else {
    va = a[p];
    vb = b[p];
  }
  T* o = out + (size_t)p * out_c;
  o[0] = from_f<T>(va);
  o[1] = from_f<T>(vb);
  for (int c = 2; c < out_c; ++c) o[c] = from_f<T>(0.f);
}

__global__ void conf_max_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                float* __restrict__ out, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = fmaxf(a[i], b[i]);
}

// rv_reconstruct's value of output pixel p = (Y, X), channel c: x + clamp01(bicubic xS of the LR image) [+ clamp01]
template <typename T>
__device__ __forceinline__ float reconstruct_at(const T* __restrict__ x, int xc, const float* __restrict__ lr, int h, int w, int Y,
                                                int X, int p, int c, float inv, int clamp01) {
  float base = bicubic_planar(lr + (size_t)c * h * w, h, w, Y, X, inv);
  base = fminf(fmaxf(base, 0.f), 1.f);
  float v = to_f(x[(size_t)p * xc + c]) + base;
  if (clamp01) v = fminf(fmaxf(v, 0.f), 1.f);
  return v;
}

template <typename T>
__global__ void reconstruct_kernel(const T* __restrict__ x, int xc, const float* __restrict__ lr,
                                   int h, int w, int scale, int clamp01,
                                   float* __restrict__ out) {
  int Ho = scale * h, Wo = scale * w;
  x += (size_t)blockIdx.z * Ho * Wo * xc;            // image blockIdx.z of a batch (rv_reconstruct_batched)
  lr += (size_t)blockIdx.z * 3 * h * w;
  out += (size_t)blockIdx.z * 3 * Ho * Wo;
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Ho * Wo) return;
  int Y = p / Wo, X = p % Wo;
  float inv = 1.0f / (float)scale;
#pragma unroll
  for (int c = 0; c < 3; ++c) out[(size_t)c * Ho * Wo + p] = reconstruct_at(x, xc, lr, h, w, Y, X, p, c, inv, clamp01);
}

// ---------------------------------------------------------------------------------------------
// rv_frames_differ : guard of the sliding-window reuse cache (network.py).  Up to 16 (a, b, bytes) buffer pairs are
// compared in one launch; *flag |= 1 as soon as any pair differs.  blockIdx.y = pair.
// ---------------------------------------------------------------------------------------------
struct CmpPairs {
  const void* a[16];
  const void* b[16];
  unsigned long long nbytes[16];
};

template <typename V>
__global__ void frames_differ_kernel(const CmpPairs P, int* __restrict__ flag) {
  const V* a = reinterpret_cast<const V*>(P.a[blockIdx.y]);
  const V* b = reinterpret_cast<const V*>(P.b[blockIdx.y]);
  const size_t n = (size_t)(P.nbytes[blockIdx.y] / sizeof(V));
  bool diff = false;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const V x = a[i], y = b[i];
    if constexpr (sizeof(V) == 16) diff |= (x.x != y.x) | (x.y != y.y) | (x.z != y.z) | (x.w != y.w);
    else diff |= (x != y);
  }
  if (__any_sync(0xffffffffu, diff) && (threadIdx.x & 31) == 0) atomicOr(flag, 1);
}


// x4 fast path: one thread per LR pixel produces its 4 x 4 output pixels.  The 16 outputs share one 5 x 5 LR neighbourhood
// (the per-output version re-reads 16 taps per output pixel and channel); the four horizontal phases are evaluated once per
// neighbourhood row (separable), conv_last's output is read as one 16-byte vector per pixel and each thread writes 16-byte
// vectors of the planar result.  Weights, tap order and summation order are those of bicubic_planar (bit-identical).
__global__ void __launch_bounds__(128) reconstruct4_kernel(const float4* __restrict__ x, const float* __restrict__ lr, int h, int w,
                                                           int clamp01, float* __restrict__ out) {
  x += (size_t)blockIdx.z * 16 * h * w;              // image blockIdx.z of a batch (rv_reconstruct_batched)
  lr += (size_t)blockIdx.z * 3 * h * w;
  out += (size_t)blockIdx.z * 48 * h * w;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= h * w) return;
  const int ly = p / w, lx = p - ly * w;
  const int Ho = 4 * h, Wo = 4 * w;
  float wt[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const float r = 0.25f * ((float)a + 0.5f) - 0.5f;          // fractional part of the source coordinate of phase a
    cubic_weights(r - floorf(r), wt[a]);
  }
  int ry[5], rx[5];
#pragma unroll
  for (int i = 0; i < 5; ++i) { ry[i] = clampi(ly - 2 + i, 0, h - 1); rx[i] = clampi(lx - 2 + i, 0, w - 1); }
  float res[3][4][4];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float* s = lr + (size_t)c * h * w;
    float hrow[4][5];                                          // [phase b][neighbourhood row]
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const float* r = s + (size_t)ry[i] * w;
      const float v0 = __ldg(r + rx[0]), v1 = __ldg(r + rx[1]), v2 = __ldg(r + rx[2]), v3 = __ldg(r + rx[3]), v4 = __ldg(r + rx[4]);
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        // phases 0, 1 look left (taps lx-2 .. lx+1), phases 2, 3 look right (lx-1 .. lx+2)
        hrow[b][i] = (b < 2) ? (wt[b][0] * v0 + wt[b][1] * v1 + wt[b][2] * v2 + wt[b][3] * v3)
                             : (wt[b][0] * v1 + wt[b][1] * v2 + wt[b][2] * v3 + wt[b][3] * v4);
      }
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int r0 = (a < 2) ? 0 : 1;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) acc += wt[a][j] * hrow[b][r0 + j];
        res[c][a][b] = fminf(fmaxf(acc, 0.f), 1.f);
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const size_t row = (size_t)(4 * ly + a) * Wo + 4 * lx;
    float4 xv[4];
#pragma unroll
    for (int b = 0; b < 4; ++b) xv[b] = __ldg(x + row + b);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float o[4];
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const float xr = (c == 0) ? xv[b].x : (c == 1 ? xv[b].y : xv[b].z);
        float v = xr + res[c][a][b];
        if (clamp01) v = fminf(fmaxf(v, 0.f), 1.f);
        o[b] = v;
      }
      *reinterpret_cast<float4*>(out + (size_t)c * Ho * Wo + row) = make_float4(o[0], o[1], o[2], o[3]);
    }
  }
}

// one horizontal tap row of bicubic_planar as reconstruct_kernel evaluates it: fma(w3, v3, fma(w2, v2, fma(w0, v0, w1 * v1)))
__device__ __forceinline__ float row4(const float* wt, float v0, float v1, float v2, float v3) {
  return __fmaf_rn(wt[3], v3, __fmaf_rn(wt[2], v2, __fmaf_rn(wt[0], v0, __fmul_rn(wt[1], v1))));
}

// x2 fast path, the counterpart of reconstruct4_kernel: one thread per LR pixel produces its 2 x 2 output pixels from one shared
// 5 x 5 LR neighbourhood (phase 0 looks left / up: taps l-2 .. l+1, phase 1 right / down: l-1 .. l+2).  conv_last's output is read
// as 16-byte vectors, the planar result written as 8-byte pairs.  Weights, taps and summation are those of bicubic_planar, with
// the products fused the way the compiler contracts it (bit-identical to reconstruct_kernel at scale 2; the weights here are
// compile-time constants, which would otherwise let the compiler fuse the other product of a row).
__global__ void __launch_bounds__(128) reconstruct2_kernel(const float4* __restrict__ x, const float* __restrict__ lr, int h, int w,
                                                           int clamp01, float* __restrict__ out) {
  x += (size_t)blockIdx.z * 4 * h * w;               // image blockIdx.z of a batch (rv_reconstruct_batched)
  lr += (size_t)blockIdx.z * 3 * h * w;
  out += (size_t)blockIdx.z * 12 * h * w;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= h * w) return;
  const int ly = p / w, lx = p - ly * w;
  const int Ho = 2 * h, Wo = 2 * w;
  float wt[2][4];
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    const float r = 0.5f * ((float)a + 0.5f) - 0.5f;           // fractional part of the source coordinate of phase a
    cubic_weights(r - floorf(r), wt[a]);
  }
  int ry[5], rx[5];
#pragma unroll
  for (int i = 0; i < 5; ++i) { ry[i] = clampi(ly - 2 + i, 0, h - 1); rx[i] = clampi(lx - 2 + i, 0, w - 1); }
  float res[3][2][2];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float* s = lr + (size_t)c * h * w;
    float hrow[2][5];                                          // [phase b][neighbourhood row]
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const float* r = s + (size_t)ry[i] * w;
      const float v0 = __ldg(r + rx[0]), v1 = __ldg(r + rx[1]), v2 = __ldg(r + rx[2]), v3 = __ldg(r + rx[3]), v4 = __ldg(r + rx[4]);
      hrow[0][i] = row4(wt[0], v0, v1, v2, v3);
      hrow[1][i] = row4(wt[1], v1, v2, v3, v4);
    }
#pragma unroll
    for (int a = 0; a < 2; ++a) {
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) acc = __fmaf_rn(wt[a][j], hrow[b][a + j], acc);
        res[c][a][b] = fminf(fmaxf(acc, 0.f), 1.f);
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    const size_t row = (size_t)(2 * ly + a) * Wo + 2 * lx;
    const float4 x0 = __ldg(x + row), x1 = __ldg(x + row + 1);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v0 = ((c == 0) ? x0.x : (c == 1 ? x0.y : x0.z)) + res[c][a][0];
      float v1 = ((c == 0) ? x1.x : (c == 1 ? x1.y : x1.z)) + res[c][a][1];
      if (clamp01) { v0 = fminf(fmaxf(v0, 0.f), 1.f); v1 = fminf(fmaxf(v1, 0.f), 1.f); }
      *reinterpret_cast<float2*>(out + (size_t)c * Ho * Wo + row) = make_float2(v0, v1);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// 8-bit output of the reconstruction tail (rv_reconstruct_u8): one variant per fp32 kernel above, each computing the same
// fp32 value with the same expressions before rv::frame_u8 turns it into a byte.  A thread owns runs of 16 consecutive output
// pixels of a row and writes each as 16-byte stores where the row and the buffer allow it (vec), byte by byte elsewhere.
// FMT (RV_FRAME_*): RGB / BGR write a run's 48 HWC bytes, R, G, B or B, G, R.  I420 / NV12 write its 16 Y bytes, and from each
// even row the U, V bytes of its 2 x 2 blocks, taken from the blocks' top-left pixels (COLOR_RGB2YUV_I420, rv::rgb8_y/u/v).  The
// x4 / x2 threads own whole blocks (4 or 2 output rows from an even row and column), so each writes its blocks' chroma itself.
// ---------------------------------------------------------------------------------------------
template <int FMT>
__host__ __device__ constexpr bool is_yuv420() { return FMT == RV_FRAME_I420 || FMT == RV_FRAME_NV12; }

template <int FMT>
__host__ __device__ constexpr int run_words() { return is_yuv420<FMT>() ? 4 : 12; }    // the words of one 16-pixel run's bytes

// pixel j of a run from its R, G, B values: HWC bytes, or a Y byte and, for a block's top-left pixel (tl), the block's U and V
// as chroma sample j / 2 of the run (chroma: I420 U bytes 0-7 and V bytes 8-15, NV12 U, V pairs)
template <int FMT>
__device__ __forceinline__ void put_px(uint32_t* words, uint32_t* chroma, int j, bool tl, float r, float g, float b) {
  const uint32_t R = frame_u8(r), G = frame_u8(g), B = frame_u8(b);
  if constexpr (is_yuv420<FMT>()) {
    words[j >> 2] |= rgb8_y(R, G, B) << (8 * (j & 3));
    if (tl) {
      const int iu = FMT == RV_FRAME_NV12 ? j : j / 2, iv = FMT == RV_FRAME_NV12 ? j + 1 : 8 + j / 2;
      chroma[iu >> 2] |= rgb8_u(R, G, B) << (8 * (iu & 3));
      chroma[iv >> 2] |= rgb8_v(R, G, B) << (8 * (iv & 3));
    }
  } else {
    const uint32_t px = FMT == RV_FRAME_BGR ? (B | (G << 8) | (R << 16)) : (R | (G << 8) | (B << 16));
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int i = 3 * j + c;
      words[i >> 2] |= ((px >> (8 * c)) & 0xffu) << (8 * (i & 3));
    }
  }
}

// the first nbytes of a run of NB bytes (NB: 8 or a multiple of 16)
template <int NB>
__device__ __forceinline__ void store_run(uint8_t* o, const uint32_t* words, int nbytes, bool vec) {
  if (vec && nbytes == NB) {
    if constexpr (NB == 8) {
      *reinterpret_cast<uint2*>(o) = make_uint2(words[0], words[1]);
    } else {
#pragma unroll
      for (int k = 0; k < NB / 16; ++k)
        reinterpret_cast<uint4*>(o)[k] = make_uint4(words[4 * k], words[4 * k + 1], words[4 * k + 2], words[4 * k + 3]);
    }
  } else {
#pragma unroll
    for (int i = 0; i < NB; ++i)
      if (i < nbytes) o[i] = (uint8_t)(words[i >> 2] >> (8 * (i & 3)));
  }
}

// one output run of an (Ho, Wo) image: n pixels of row y from column x; a 4:2:0 run from an even row also writes its n / 2
// chroma samples
template <int FMT>
__device__ __forceinline__ void store_px_run(uint8_t* img, int Ho, int Wo, int y, int x, const uint32_t* words,
                                             const uint32_t* chroma, int n, bool vec) {
  if constexpr (is_yuv420<FMT>()) {
    store_run<16>(img + (size_t)y * Wo + x, words, n, vec);
    if (y % 2 == 0) {
      uint8_t* c = img + (size_t)Ho * Wo;
      if (FMT == RV_FRAME_NV12) {
        store_run<16>(c + (size_t)(y / 2) * Wo + x, chroma, n, vec);
      } else {
        store_run<8>(c + (size_t)(y / 2) * (Wo / 2) + x / 2, chroma, n / 2, vec);
        store_run<8>(c + (size_t)Ho * Wo / 4 + (size_t)(y / 2) * (Wo / 2) + x / 2, chroma + 2, n / 2, vec);
      }
    }
  } else {
    store_run<48>(img + 3 * ((size_t)y * Wo + x), words, 3 * n, vec);
  }
}

// x4: reconstruct4_kernel's arithmetic for 4 neighbouring LR pixels per thread -> 4 output rows of 16 pixels
template <int FMT>
__global__ void __launch_bounds__(128) reconstruct4_u8_kernel(const float4* __restrict__ x, const float* __restrict__ lr, int h, int w,
                                                              int clamp01, int vec, uint8_t* __restrict__ out) {
  x += (size_t)blockIdx.z * 16 * h * w;
  lr += (size_t)blockIdx.z * 3 * h * w;
  out += (size_t)blockIdx.z * (is_yuv420<FMT>() ? 24 : 48) * h * w;
  const int wq = (w + 3) / 4;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= h * wq) return;
  const int ly = q / wq, lx0 = 4 * (q - ly * wq);
  const int nk = min(4, w - lx0);
  const int Wo = 4 * w;
  float wt[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const float r = 0.25f * ((float)a + 0.5f) - 0.5f;
    cubic_weights(r - floorf(r), wt[a]);
  }
  uint32_t ob[4][run_words<FMT>()] = {};                       // [output row a][little-endian byte words of the 16-pixel run]
  uint32_t cb[2][4] = {};                                      // 4:2:0: [even row a / 2][chroma words of its 8 blocks]
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (k >= nk) break;
    const int lx = lx0 + k;
    int ry[5], rx[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) { ry[i] = clampi(ly - 2 + i, 0, h - 1); rx[i] = clampi(lx - 2 + i, 0, w - 1); }
    float res[3][4][4];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float* s = lr + (size_t)c * h * w;
      float hrow[4][5];
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const float* r = s + (size_t)ry[i] * w;
        const float v0 = __ldg(r + rx[0]), v1 = __ldg(r + rx[1]), v2 = __ldg(r + rx[2]), v3 = __ldg(r + rx[3]), v4 = __ldg(r + rx[4]);
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          hrow[b][i] = (b < 2) ? (wt[b][0] * v0 + wt[b][1] * v1 + wt[b][2] * v2 + wt[b][3] * v3)
                               : (wt[b][0] * v1 + wt[b][1] * v2 + wt[b][2] * v3 + wt[b][3] * v4);
        }
      }
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const int r0 = (a < 2) ? 0 : 1;
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          float acc = 0.f;
#pragma unroll
          for (int j = 0; j < 4; ++j) acc += wt[a][j] * hrow[b][r0 + j];
          res[c][a][b] = fminf(fmaxf(acc, 0.f), 1.f);
        }
      }
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const size_t row = (size_t)(4 * ly + a) * Wo + 4 * lx;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const float4 xv = __ldg(x + row + b);
        float v[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float xr = (c == 0) ? xv.x : (c == 1 ? xv.y : xv.z);
          v[c] = xr + res[c][a][b];
          if (clamp01) v[c] = fminf(fmaxf(v[c], 0.f), 1.f);
        }
        put_px<FMT>(ob[a], cb[a / 2], 4 * k + b, a % 2 == 0 && b % 2 == 0, v[0], v[1], v[2]);
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) store_px_run<FMT>(out, 4 * h, Wo, 4 * ly + a, 4 * lx0, ob[a], cb[a / 2], 4 * nk, vec);
}

// x2: reconstruct2_kernel's arithmetic for 8 neighbouring LR pixels per thread -> 2 output rows of 16 pixels
template <int FMT>
__global__ void __launch_bounds__(128) reconstruct2_u8_kernel(const float4* __restrict__ x, const float* __restrict__ lr, int h, int w,
                                                              int clamp01, int vec, uint8_t* __restrict__ out) {
  x += (size_t)blockIdx.z * 4 * h * w;
  lr += (size_t)blockIdx.z * 3 * h * w;
  out += (size_t)blockIdx.z * (is_yuv420<FMT>() ? 6 : 12) * h * w;
  const int wq = (w + 7) / 8;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= h * wq) return;
  const int ly = q / wq, lx0 = 8 * (q - ly * wq);
  const int nk = min(8, w - lx0);
  const int Wo = 2 * w;
  float wt[2][4];
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    const float r = 0.5f * ((float)a + 0.5f) - 0.5f;
    cubic_weights(r - floorf(r), wt[a]);
  }
  uint32_t ob[2][run_words<FMT>()] = {};
  uint32_t cb[4] = {};                                         // 4:2:0: the chroma words of row 0's 8 blocks
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (k >= nk) break;
    const int lx = lx0 + k;
    int ry[5], rx[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) { ry[i] = clampi(ly - 2 + i, 0, h - 1); rx[i] = clampi(lx - 2 + i, 0, w - 1); }
    float res[3][2][2];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float* s = lr + (size_t)c * h * w;
      float hrow[2][5];
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const float* r = s + (size_t)ry[i] * w;
        const float v0 = __ldg(r + rx[0]), v1 = __ldg(r + rx[1]), v2 = __ldg(r + rx[2]), v3 = __ldg(r + rx[3]), v4 = __ldg(r + rx[4]);
        hrow[0][i] = row4(wt[0], v0, v1, v2, v3);
        hrow[1][i] = row4(wt[1], v1, v2, v3, v4);
      }
#pragma unroll
      for (int a = 0; a < 2; ++a) {
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          float acc = 0.f;
#pragma unroll
          for (int j = 0; j < 4; ++j) acc = __fmaf_rn(wt[a][j], hrow[b][a + j], acc);
          res[c][a][b] = fminf(fmaxf(acc, 0.f), 1.f);
        }
      }
    }
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const size_t row = (size_t)(2 * ly + a) * Wo + 2 * lx;
      const float4 x0 = __ldg(x + row), x1 = __ldg(x + row + 1);
      float v0[3], v1[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        v0[c] = ((c == 0) ? x0.x : (c == 1 ? x0.y : x0.z)) + res[c][a][0];
        v1[c] = ((c == 0) ? x1.x : (c == 1 ? x1.y : x1.z)) + res[c][a][1];
        if (clamp01) { v0[c] = fminf(fmaxf(v0[c], 0.f), 1.f); v1[c] = fminf(fmaxf(v1[c], 0.f), 1.f); }
      }
      put_px<FMT>(ob[a], cb, 2 * k, a == 0, v0[0], v0[1], v0[2]);
      put_px<FMT>(ob[a], cb, 2 * k + 1, false, v1[0], v1[1], v1[2]);
    }
  }
#pragma unroll
  for (int a = 0; a < 2; ++a) store_px_run<FMT>(out, 2 * h, Wo, 2 * ly + a, 2 * lx0, ob[a], cb, 2 * nk, vec);
}

// any scale, x dtype and channel count: reconstruct_kernel's arithmetic for 16 consecutive output pixels (row-major) per thread
// (4:2:0: the thread of a block's top-left pixel writes the block's U and V bytes)
template <typename T, int FMT>
__global__ void __launch_bounds__(256) reconstruct_u8_kernel(const T* __restrict__ x, int xc, const float* __restrict__ lr, int h, int w,
                                                             int scale, int clamp01, int vec, uint8_t* __restrict__ out) {
  const int Ho = scale * h, Wo = scale * w;
  constexpr bool YUV = is_yuv420<FMT>();
  x += (size_t)blockIdx.z * Ho * Wo * xc;
  lr += (size_t)blockIdx.z * 3 * h * w;
  out += (size_t)blockIdx.z * (YUV ? 3 * (size_t)Ho * Wo / 2 : 3 * (size_t)Ho * Wo);
  const int p0 = (blockIdx.x * blockDim.x + threadIdx.x) * 16;
  if (p0 >= Ho * Wo) return;
  const int n = min(16, Ho * Wo - p0);
  const float inv = 1.0f / (float)scale;
  uint32_t ob[run_words<FMT>()] = {};
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    if (j >= n) break;
    const int p = p0 + j;
    const int Y = p / Wo, X = p % Wo;
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = reconstruct_at(x, xc, lr, h, w, Y, X, p, c, inv, clamp01);
    if constexpr (YUV) {
      const uint32_t R = frame_u8(v[0]), G = frame_u8(v[1]), B = frame_u8(v[2]);
      ob[j >> 2] |= rgb8_y(R, G, B) << (8 * (j & 3));
      if (Y % 2 == 0 && X % 2 == 0) {
        uint8_t* c = out + (size_t)Ho * Wo;
        const size_t iu = FMT == RV_FRAME_NV12 ? (size_t)(Y / 2) * Wo + X : (size_t)(Y / 2) * (Wo / 2) + X / 2;
        c[iu] = (uint8_t)rgb8_u(R, G, B);
        c[FMT == RV_FRAME_NV12 ? iu + 1 : iu + (size_t)Ho * Wo / 4] = (uint8_t)rgb8_v(R, G, B);
      }
    } else {
      put_px<FMT>(ob, nullptr, j, false, v[0], v[1], v[2]);
    }
  }
  if constexpr (YUV) store_run<16>(out + (size_t)p0, ob, n, vec);
  else store_run<48>(out + 3 * (size_t)p0, ob, 3 * n, vec);
}

}  // namespace rv

// =================================================================================================
// C ABI
// =================================================================================================
using namespace rv;

// REFVSR_NO_FAST_POINTWISE set: the generic gather, aligned-sample and reconstruct kernels only (the reference the fast paths are
// checked against).  Read once per process.
static bool fast_pointwise() {
  static const bool ok = getenv("REFVSR_NO_FAST_POINTWISE") == nullptr;
  return ok;
}

extern "C" int rv_frames_differ(const void* const* a, const void* const* b, const uint64_t* nbytes, int n, int32_t* flag,
                                void* stream) {
  RV_REQUIRE(a && b && nbytes && flag && n > 0 && n <= 16, "rv_frames_differ: 1..16 buffer pairs (got %d)", n);
  CmpPairs P;
  bool vec = true;
  for (int i = 0; i < n; ++i) {
    RV_REQUIRE(a[i] && b[i] && nbytes[i] % 4 == 0, "rv_frames_differ: null buffer or size not a multiple of 4 (pair %d)", i);
    P.a[i] = a[i]; P.b[i] = b[i]; P.nbytes[i] = nbytes[i];
    vec = vec && ((uintptr_t)a[i] % 16 == 0) && ((uintptr_t)b[i] % 16 == 0) && (nbytes[i] % 16 == 0);
  }
  dim3 grid(64, n);
  if (vec) frames_differ_kernel<uint4><<<grid, 256, 0, (cudaStream_t)stream>>>(P, flag);
  else frames_differ_kernel<uint32_t><<<grid, 256, 0, (cudaStream_t)stream>>>(P, flag);
  RV_LAUNCH_CHECK("frames_differ");
  return RV_OK;
}

extern "C" int rv_prep_image(const float* src, int H, int W, const float* mat12_host, int pool2,
                             void* out, int out_c, int out_dtype, void* stream) {
  RV_REQUIRE(src && out && H > 0 && W > 0 && out_c >= 3, "rv_prep_image: bad arguments");
  RV_REQUIRE(!pool2 || (H % 2 == 0 && W % 2 == 0), "rv_prep_image: pool2 needs even H,W (%d,%d)", H, W);
  Mat12 m;
  m.use = mat12_host != nullptr;
  for (int i = 0; i < 12; ++i) m.m[i] = mat12_host ? mat12_host[i] : 0.f;
  int n = (pool2 ? H / 2 : H) * (pool2 ? W / 2 : W);
  RV_DISPATCH_DTYPE(out_dtype, T, (prep_image_kernel<T><<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(
                                      src, H, W, m, pool2, (T*)out, out_c)));
  RV_LAUNCH_CHECK("prep_image");
  return RV_OK;
}

extern "C" int rv_spynet_resize_norm(const float* src, int H, int W, float* out, int Ho, int Wo,
                                     void* stream) {
  RV_REQUIRE(src && out && H > 0 && W > 0 && Ho > 0 && Wo > 0, "rv_spynet_resize_norm: bad arguments");
  spynet_resize_norm_kernel<<<cdiv(Ho * Wo, 256), 256, 0, (cudaStream_t)stream>>>(src, H, W, out, Ho, Wo);
  RV_LAUNCH_CHECK("spynet_resize_norm");
  return RV_OK;
}

extern "C" int rv_avgpool2(const float* src, int H, int W, int C, float* out, void* stream) {
  RV_REQUIRE(src && out && H >= 2 && W >= 2 && C > 0, "rv_avgpool2: bad arguments");
  int n = (H / 2) * (W / 2) * C;
  avgpool2_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(src, H, W, C, out);
  RV_LAUNCH_CHECK("avgpool2");
  return RV_OK;
}

extern "C" int rv_spynet_level_input(const float* ref, const float* supp, const float* flow_prev,
                                     int H, int W, void* out8, int out_dtype, float* flow_up,
                                     void* stream) {
  RV_REQUIRE(ref && supp && out8 && flow_up && H > 0 && W > 0, "rv_spynet_level_input: bad arguments");
  RV_REQUIRE(flow_prev == nullptr || (H % 2 == 0 && W % 2 == 0),
             "rv_spynet_level_input: level size must be even (%d,%d)", H, W);
  RV_DISPATCH_DTYPE(out_dtype, T,
                    (spynet_level_input_kernel<T><<<cdiv(H * W, 128), 128, 0, (cudaStream_t)stream>>>(
                        ref, supp, flow_prev, H, W, (T*)out8, flow_up)));
  RV_LAUNCH_CHECK("spynet_level_input");
  return RV_OK;
}

extern "C" int rv_flow_resize(const float* flow, int H, int W, float* out, int h, int w, void* stream) {
  RV_REQUIRE(flow && out && H > 0 && W > 0 && h > 0 && w > 0, "rv_flow_resize: bad arguments");
  flow_resize_kernel<<<cdiv(h * w, 256), 256, 0, (cudaStream_t)stream>>>(flow, H, W, out, h, w);
  RV_LAUNCH_CHECK("flow_resize");
  return RV_OK;
}

template <typename T>
static int warp_launch(const void* src, int Hi, int Wi, int C, const float* flow, int hf, int wf,
                       int up2, void* out, int nimg, cudaStream_t st) {
  constexpr int VMAX = 16 / sizeof(T);
  long long px = (long long)(up2 ? 4 : 1) * hf * wf;
  bool aligned = ((uintptr_t)src % 16 == 0) && ((uintptr_t)out % 16 == 0);
  if (C % VMAX == 0 && aligned && C / VMAX <= 256) {
    const int cv = C / VMAX, ppb = 256 / cv;         // pixels per block
    warp_vec_kernel<T, VMAX><<<dim3(cdiv(px, ppb), 1, nimg), 256, 0, st>>>((const T*)src, Hi, Wi, C, flow, hf, wf, up2, (T*)out, ppb);
  } else {
    long long n = px * C;
    warp_kernel<T, 1><<<dim3(cdiv(n, 256), 1, nimg), 256, 0, st>>>((const T*)src, Hi, Wi, C, flow, hf, wf, up2, (T*)out);
  }
  RV_LAUNCH_CHECK("warp");
  return RV_OK;
}

extern "C" int rv_warp_batched(const void* src, int Hi, int Wi, int C, int dtype, const float* flow, int hf,
                               int wf, int flow_up2, void* out, int n, void* stream) {
  RV_REQUIRE(src && flow && out && Hi > 1 && Wi > 1 && C > 0 && hf > 0 && wf > 0, "rv_warp: bad arguments");
  RV_REQUIRE(n >= 1 && n <= 65535, "rv_warp: n=%d images out of range", n);
  RV_REQUIRE((uintptr_t)flow % 8 == 0, "rv_warp: flow must be 8-byte aligned");
  RV_DISPATCH_DTYPE(dtype, T, return (warp_launch<T>(src, Hi, Wi, C, flow, hf, wf, flow_up2, out, n, (cudaStream_t)stream)));
  return RV_OK;
}

extern "C" int rv_warp(const void* src, int Hi, int Wi, int C, int dtype, const float* flow, int hf,
                       int wf, int flow_up2, void* out, void* stream) {
  return rv_warp_batched(src, Hi, Wi, C, dtype, flow, hf, wf, flow_up2, out, 1, stream);
}

extern "C" int rv_warp3_batched(const void* feat, const void* featUP, const float* conf, const float* flow, int h, int w, int C,
                                int dtype, void* out_feat, void* out_featUP, float* out_conf, int n, void* stream) {
  RV_REQUIRE(n >= 1 && n <= 65535, "rv_warp3: n=%d images out of range", n);
  RV_REQUIRE(feat && featUP && conf && flow && out_feat && out_featUP && out_conf && h > 0 && w > 0, "rv_warp3: bad arguments");
  RV_REQUIRE(dtype == RV_F16 || dtype == RV_BF16, "rv_warp3: f16 / bf16 features only (use rv_warp for fp32)");
  RV_REQUIRE(C > 0 && C % 8 == 0, "rv_warp3: C=%d must be a multiple of 8", C);
  RV_REQUIRE((long long)4 * h * w * (C / 8) < (1ll << 31), "rv_warp3: map too large for 32-bit vector indices");
  const int tiles = ((h + W3_TH - 1) / W3_TH) * ((w + W3_TW - 1) / W3_TW);
  auto launch = [&](auto tag, auto cvtag) {
    using T = decltype(tag);
    warp3_kernel<T, decltype(cvtag)::value><<<dim3(tiles, 1, n), 256, 0, (cudaStream_t)stream>>>(
        (const T*)feat, (const T*)featUP, conf, flow, h, w, C, (T*)out_feat, (T*)out_featUP, out_conf);
  };
  auto by_cv = [&](auto tag) {           // the reference's widths (48 / 24 channels, config_RefVSR_*.py) + powers of two
    if (C == 48) launch(tag, std::integral_constant<int, 6>{});
    else if (C == 24) launch(tag, std::integral_constant<int, 3>{});
    else if (C == 64) launch(tag, std::integral_constant<int, 8>{});
    else launch(tag, std::integral_constant<int, 0>{});
  };
  if (dtype == RV_F16) by_cv(__half{});
  else by_cv(__nv_bfloat16{});
  RV_LAUNCH_CHECK("warp3");
  return RV_OK;
}

extern "C" int rv_warp3(const void* feat, const void* featUP, const float* conf, const float* flow, int h, int w, int C,
                        int dtype, void* out_feat, void* out_featUP, float* out_conf, void* stream) {
  return rv_warp3_batched(feat, featUP, conf, flow, h, w, C, dtype, out_feat, out_featUP, out_conf, 1, stream);
}

extern "C" int rv_patch_pack(const void* feat, int H, int W, int C, int dtype, int mode, void* out,
                             int kpad, void* stream) {
  RV_REQUIRE(feat && out && H >= 2 && W >= 2, "rv_patch_pack: bad arguments");
  RV_REQUIRE(C * 9 <= 256, "rv_patch_pack: C*9 must be <= 256 (got C=%d)", C);
  RV_REQUIRE(mode >= 0 && mode <= 2, "rv_patch_pack: bad mode %d", mode);
  RV_REQUIRE(kpad >= (mode == 0 ? 1 : 3) * C * 9, "rv_patch_pack: kpad %d too small", kpad);
  long long threads = (long long)H * W * 32;
  RV_DISPATCH_DTYPE(dtype, T, (patch_pack_kernel<T><<<cdiv(threads, 256), 256, 0, (cudaStream_t)stream>>>(
                                  (const T*)feat, H, W, C, mode, (__half*)out, kpad)));
  RV_LAUNCH_CHECK("patch_pack");
  return RV_OK;
}

extern "C" int rv_gather_blocks(const void* value, int Hv, int Wv, int C, int dtype,
                                const int32_t* idx, int hq, int wq, int ks, void* out, void* stream) {
  RV_REQUIRE(value && idx && out && ks >= 1 && Hv % ks == 0 && Wv % ks == 0 && hq > 0 && wq > 0,
             "rv_gather_blocks: bad arguments");
  int rowbytes = C * dtype_size(dtype);
  long long px = (long long)ks * hq * ks * wq;
  cudaStream_t st = (cudaStream_t)stream;
  const uint8_t* v = (const uint8_t*)value;
  uint8_t* o = (uint8_t*)out;
  bool a16 = ((uintptr_t)value % 16 == 0) && ((uintptr_t)out % 16 == 0);
  bool a4 = ((uintptr_t)value % 4 == 0) && ((uintptr_t)out % 4 == 0);   // 4-byte words need 4-byte aligned rows
  if (fast_pointwise() && rowbytes % 16 == 0 && a16 && (ks == 1 || ks == 2 || ks == 4) && hq <= 65535) {
    const int nv = rowbytes / 16;
    const dim3 grid((unsigned)cdiv((long long)wq * nv, 256), (unsigned)hq);
    const uint4* v4 = (const uint4*)value;
    uint4* o4 = (uint4*)out;
    if (ks == 4 && nv == 6) gather_cells_kernel<4, 6><<<grid, 256, 0, st>>>(v4, Wv, nv, idx, wq, o4);
    else if (ks == 4 && nv == 3) gather_cells_kernel<4, 3><<<grid, 256, 0, st>>>(v4, Wv, nv, idx, wq, o4);
    else if (ks == 4) gather_cells_kernel<4, 0><<<grid, 256, 0, st>>>(v4, Wv, nv, idx, wq, o4);
    else if (ks == 2 && nv == 6) gather_cells_kernel<2, 6><<<grid, 256, 0, st>>>(v4, Wv, nv, idx, wq, o4);
    else if (ks == 2 && nv == 3) gather_cells_kernel<2, 3><<<grid, 256, 0, st>>>(v4, Wv, nv, idx, wq, o4);
    else if (ks == 2) gather_cells_kernel<2, 0><<<grid, 256, 0, st>>>(v4, Wv, nv, idx, wq, o4);
    else if (nv == 6) gather_cells_kernel<1, 6><<<grid, 256, 0, st>>>(v4, Wv, nv, idx, wq, o4);
    else if (nv == 3) gather_cells_kernel<1, 3><<<grid, 256, 0, st>>>(v4, Wv, nv, idx, wq, o4);
    else gather_cells_kernel<1, 0><<<grid, 256, 0, st>>>(v4, Wv, nv, idx, wq, o4);
  } else if (rowbytes % 16 == 0 && a16)
    gather_blocks_kernel<16><<<cdiv(px * (rowbytes / 16), 256), 256, 0, st>>>(v, Hv, Wv, rowbytes, idx, hq, wq, ks, o);
  else if (rowbytes % 4 == 0 && a4)
    gather_blocks_kernel<4><<<cdiv(px * (rowbytes / 4), 256), 256, 0, st>>>(v, Hv, Wv, rowbytes, idx, hq, wq, ks, o);
  else
    gather_blocks_kernel<2><<<cdiv(px * (rowbytes / 2), 256), 256, 0, st>>>(v, Hv, Wv, rowbytes, idx, hq, wq, ks, o);
  RV_LAUNCH_CHECK("gather_blocks");
  return RV_OK;
}

template <typename T>
static int aligned_sample_launch(const void* x, int h, int w, int ks, int C, const float* affine,
                                 void* out, cudaStream_t st) {
  constexpr int VMAX = 16 / sizeof(T);
  long long px = (long long)ks * h * ks * w;
  bool a16 = ((uintptr_t)x % 16 == 0) && ((uintptr_t)out % 16 == 0);
  if (fast_pointwise() && (ks == 2 || ks == 4) && C % VMAX == 0 && a16 && px * (C / VMAX) < (1ll << 31)) {   // (32-bit vector indices)
    const int cv = C / VMAX;
    auto launch = [&](auto kstag) {
      constexpr int KS = decltype(kstag)::value, TH = KS == 2 ? 4 : 8, TW = KS == 2 ? 16 : 8;
      const int tiles = ((h + TH - 1) / TH) * ((w + TW - 1) / TW);
      auto run = [&](auto cvtag) {
        constexpr int CV = decltype(cvtag)::value;
        const auto kernel = KS == 2 ? aligned_sample2_kernel<T, CV> : aligned_sample4_kernel<T, CV>;
        kernel<<<tiles, 256, 0, st>>>((const T*)x, h, w, C, affine, (T*)out);
      };
      if (cv == 6) run(std::integral_constant<int, 6>{});
      else if (cv == 3) run(std::integral_constant<int, 3>{});
      else if (cv == 12) run(std::integral_constant<int, 12>{});
      else run(std::integral_constant<int, 0>{});
    };
    if (ks == 2) launch(std::integral_constant<int, 2>{});
    else launch(std::integral_constant<int, 4>{});
  }
  else if (C % VMAX == 0 && a16)
    aligned_sample_kernel<T, VMAX><<<cdiv(px * (C / VMAX), 256), 256, 0, st>>>((const T*)x, h, w, ks, C, affine, (T*)out);
  else
    aligned_sample_kernel<T, 1><<<cdiv(px * C, 256), 256, 0, st>>>((const T*)x, h, w, ks, C, affine, (T*)out);
  RV_LAUNCH_CHECK("aligned_sample");
  return RV_OK;
}

extern "C" int rv_aligned_sample(const void* x, int h, int w, int ks, int C, int dtype,
                                 const float* affine, void* out, void* stream) {
  RV_REQUIRE(x && affine && out && h > 0 && w > 0 && ks >= 1 && C > 0, "rv_aligned_sample: bad arguments");
  RV_REQUIRE(ks * h >= 2 && ks * w >= 2, "rv_aligned_sample: input too small for reflection padding");
  RV_DISPATCH_DTYPE(dtype, T, return (aligned_sample_launch<T>(x, h, w, ks, C, affine, out, (cudaStream_t)stream)));
  return RV_OK;
}

extern "C" int rv_space_to_depth2(const void* src, int H, int W, int C, int dtype, void* out, void* stream) {
  RV_REQUIRE(src && out && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0, "rv_space_to_depth2: H, W must be even (%d,%d)", H, W);
  int rowbytes = C * dtype_size(dtype);
  RV_REQUIRE(rowbytes % 16 == 0 && ((uintptr_t)src % 16 == 0) && ((uintptr_t)out % 16 == 0),
             "rv_space_to_depth2: pixel rows must be 16-byte multiples and aligned");
  int cv = rowbytes / 16;
  long long n = (long long)(H / 2) * (W / 2) * 4 * cv;
  space_to_depth2_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>((const uint4*)src, H, W, cv, (uint4*)out);
  RV_LAUNCH_CHECK("space_to_depth2");
  return RV_OK;
}

extern "C" int rv_bicubic_up2_image(const float* src, int H, int W, void* out, int out_c,
                                    int out_dtype, void* stream) {
  RV_REQUIRE(src && out && H > 0 && W > 0 && out_c >= 3, "rv_bicubic_up2_image: bad arguments");
  RV_DISPATCH_DTYPE(out_dtype, T, (bicubic_up2_image_kernel<T><<<cdiv(4LL * H * W, 256), 256, 0, (cudaStream_t)stream>>>(
                                      src, H, W, (T*)out, out_c)));
  RV_LAUNCH_CHECK("bicubic_up2_image");
  return RV_OK;
}

extern "C" int rv_maxpool2(const void* src, int H, int W, int C, int dtype, void* out, void* stream) {
  RV_REQUIRE(src && out && H >= 2 && W >= 2 && C > 0, "rv_maxpool2: bad arguments");
  long long n = (long long)(H / 2) * (W / 2) * C;
  RV_DISPATCH_DTYPE(dtype, T, (maxpool2_kernel<T><<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>((const T*)src, H, W, C, (T*)out)));
  RV_LAUNCH_CHECK("maxpool2");
  return RV_OK;
}

extern "C" int rv_resize_planes(const float* src, int n, int H, int W, float inv_scale, int Ho, int Wo, int mode,
                                int clamp01, float* out, void* stream) {
  RV_REQUIRE(src && out && n > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && inv_scale > 0.f && (mode == 0 || mode == 1),
             "rv_resize_planes: bad arguments");
  long long tot = (long long)n * Ho * Wo;
  resize_planes_kernel<<<cdiv(tot, 256), 256, 0, (cudaStream_t)stream>>>(src, n, H, W, inv_scale, Ho, Wo, mode, clamp01, out);
  RV_LAUNCH_CHECK("resize_planes");
  return RV_OK;
}

extern "C" int rv_conf_pair_batched(const float* a, const float* b, int h, int w, int up2, void* out,
                                    int out_c, int out_dtype, int nimg, void* stream) {
  RV_REQUIRE(a && b && out && h > 0 && w > 0 && out_c >= 2, "rv_conf_pair: bad arguments");
  RV_REQUIRE(nimg >= 1 && nimg <= 65535, "rv_conf_pair: n=%d images out of range", nimg);
  long long n = (long long)(up2 ? 4 : 1) * h * w;
  RV_DISPATCH_DTYPE(out_dtype, T, (conf_pair_kernel<T><<<dim3(cdiv(n, 256), 1, nimg), 256, 0, (cudaStream_t)stream>>>(
                                      a, b, h, w, up2, (T*)out, out_c)));
  RV_LAUNCH_CHECK("conf_pair");
  return RV_OK;
}

extern "C" int rv_conf_pair(const float* a, const float* b, int h, int w, int up2, void* out,
                            int out_c, int out_dtype, void* stream) {
  return rv_conf_pair_batched(a, b, h, w, up2, out, out_c, out_dtype, 1, stream);
}

extern "C" int rv_conf_max(const float* a, const float* b, float* out, int n, void* stream) {
  RV_REQUIRE(a && b && out && n > 0, "rv_conf_max: bad arguments");
  conf_max_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(a, b, out, n);
  RV_LAUNCH_CHECK("conf_max");
  return RV_OK;
}

// The reconstruction path of rv_reconstruct{,_u8}_batched: the x4 / x2 kernels for an aligned 4-channel fp32 conv_last output,
// the generic kernels otherwise.  The 8-bit tail follows the same choice, so each byte comes from the value the fp32 kernel writes.
enum class RecPath { X4, X2, GENERIC };
static RecPath reconstruct_path(const void* x, int xc, int x_dtype, int scale) {
  if (fast_pointwise() && x_dtype == RV_F32 && xc == 4 && (uintptr_t)x % 16 == 0) return scale == 4 ? RecPath::X4 : RecPath::X2;
  return RecPath::GENERIC;
}

extern "C" int rv_reconstruct_batched(const void* x, int xc, int x_dtype, const float* lr, int h, int w,
                                      int scale, int clamp01, float* out, int nimg, void* stream) {
  RV_REQUIRE(x && lr && out && h > 0 && w > 0 && xc >= 3 && (scale == 2 || scale == 4),
             "rv_reconstruct: bad arguments");
  RV_REQUIRE(nimg >= 1 && nimg <= 65535, "rv_reconstruct: n=%d images out of range", nimg);
  long long n = (long long)scale * h * scale * w;
  const RecPath path = reconstruct_path(x, xc, x_dtype, scale);
  if (path == RecPath::X4 && (uintptr_t)out % 16 == 0) {
    reconstruct4_kernel<<<dim3(cdiv((long long)h * w, 128), 1, nimg), 128, 0, (cudaStream_t)stream>>>((const float4*)x, lr, h, w, clamp01, out);
  } else if (path == RecPath::X2 && (uintptr_t)out % 8 == 0) {
    reconstruct2_kernel<<<dim3(cdiv((long long)h * w, 128), 1, nimg), 128, 0, (cudaStream_t)stream>>>((const float4*)x, lr, h, w, clamp01, out);
  } else {
    RV_DISPATCH_DTYPE(x_dtype, T, (reconstruct_kernel<T><<<dim3(cdiv(n, 256), 1, nimg), 256, 0, (cudaStream_t)stream>>>(
                                      (const T*)x, xc, lr, h, w, scale, clamp01, out)));
  }
  RV_LAUNCH_CHECK("reconstruct");
  return RV_OK;
}

extern "C" int rv_reconstruct(const void* x, int xc, int x_dtype, const float* lr, int h, int w,
                              int scale, int clamp01, float* out, void* stream) {
  return rv_reconstruct_batched(x, xc, x_dtype, lr, h, w, scale, clamp01, out, 1, stream);
}

template <int FMT>
static int launch_reconstruct_u8(RecPath path, const void* x, int xc, int x_dtype, const float* lr, int h, int w, int scale,
                                  int clamp01, uint8_t* out, int nimg, cudaStream_t st) {
  const bool aligned = (uintptr_t)out % 16 == 0;
  if (path == RecPath::X4) {
    const int vec = aligned && (4 * w) % 16 == 0;
    const dim3 grid(cdiv((long long)h * ((w + 3) / 4), 128), 1, nimg);
    reconstruct4_u8_kernel<FMT><<<grid, 128, 0, st>>>((const float4*)x, lr, h, w, clamp01, vec, out);
  } else if (path == RecPath::X2) {
    const int vec = aligned && (2 * w) % 16 == 0;
    const dim3 grid(cdiv((long long)h * ((w + 7) / 8), 128), 1, nimg);
    reconstruct2_u8_kernel<FMT><<<grid, 128, 0, st>>>((const float4*)x, lr, h, w, clamp01, vec, out);
  } else {
    const long long n = (long long)scale * h * scale * w;
    const int vec = aligned && (is_yuv420<FMT>() ? 3 * n / 2 : 3 * n) % 16 == 0;
    const dim3 grid(cdiv(cdiv(n, 16), 256), 1, nimg);
    RV_DISPATCH_DTYPE(x_dtype, T, (reconstruct_u8_kernel<T, FMT><<<grid, 256, 0, st>>>((const T*)x, xc, lr, h, w, scale, clamp01, vec, out)));
  }
  return RV_OK;
}

extern "C" int rv_reconstruct_u8_batched(const void* x, int xc, int x_dtype, const float* lr, int h, int w, int scale, int clamp01,
                                         int fmt, uint8_t* out, int nimg, void* stream) {
  RV_REQUIRE(x && lr && out && h > 0 && w > 0 && xc >= 3 && (scale == 2 || scale == 4),
             "rv_reconstruct_u8: bad arguments");
  RV_REQUIRE(fmt >= RV_FRAME_RGB && fmt <= RV_FRAME_NV12, "rv_reconstruct_u8: unknown frame format %d", fmt);
  RV_REQUIRE(nimg >= 1 && nimg <= 65535, "rv_reconstruct_u8: n=%d images out of range", nimg);
  RV_REQUIRE((long long)scale * h * scale * w <= (1ll << 30), "rv_reconstruct_u8: %d x %d output too large", scale * h, scale * w);
  const RecPath path = reconstruct_path(x, xc, x_dtype, scale);
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  switch (fmt) {
    case RV_FRAME_RGB: rc = launch_reconstruct_u8<RV_FRAME_RGB>(path, x, xc, x_dtype, lr, h, w, scale, clamp01, out, nimg, st); break;
    case RV_FRAME_BGR: rc = launch_reconstruct_u8<RV_FRAME_BGR>(path, x, xc, x_dtype, lr, h, w, scale, clamp01, out, nimg, st); break;
    case RV_FRAME_I420: rc = launch_reconstruct_u8<RV_FRAME_I420>(path, x, xc, x_dtype, lr, h, w, scale, clamp01, out, nimg, st); break;
    default: rc = launch_reconstruct_u8<RV_FRAME_NV12>(path, x, xc, x_dtype, lr, h, w, scale, clamp01, out, nimg, st); break;
  }
  if (rc != RV_OK) return rc;
  RV_LAUNCH_CHECK("reconstruct_u8");
  return RV_OK;
}

extern "C" int rv_reconstruct_u8(const void* x, int xc, int x_dtype, const float* lr, int h, int w, int scale, int clamp01, int fmt,
                                 uint8_t* out, void* stream) {
  return rv_reconstruct_u8_batched(x, xc, x_dtype, lr, h, w, scale, clamp01, fmt, out, 1, stream);
}
