// rv_conf_map_images: the bytes evaluation/eval_quan_conf_map.py writes for one frame - up to four min/max-normalised,
// colour-mapped confidence maps, the input and the output - as one packed uint8 BGR HWC buffer, so the host only encodes.
//
// Launch 1 (minmax_kernel, normalised maps only): RED_BLK CTAs per map each reduce a strided share of the map to
// order-preserving uint32 keys of its min and max and store the pair in `work`.  Launch 2 (images_kernel): every CTA owns 4 * NT consecutive pixels of one
// image; a map CTA first folds its map's RED_BLK partials (so no CTA waits on another and nothing is initialised between
// calls), then normalises with IEEE float32 operations, takes matplotlib's colormap index and looks the bytes up in the LUT;
// a frame CTA scales by 255 and rounds like cv::Mat::convertTo(CV_8U) (rv::frame_bgr8, shared with rv_eval_images).
#include "common.cuh"
#include "frame_u8.cuh"

namespace {

constexpr int NT = 256, PPT = 4, RED_BLK = 64, MAXSEG = 6;

static_assert(4 * RED_BLK * 2 == RV_CONF_MAP_WORK, "work holds a (min, max) key per reducing CTA of every map");
static_assert(RED_BLK == 64, "images_kernel folds the partials with two per lane");

// float -> uint32 with the same order (-0 < +0); NaN gets the smallest key for the min and the largest for the max, so a
// map holding NaN has NaN as both, as torch's min() / max() return it
__device__ __forceinline__ uint32_t key_of(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float float_of(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__global__ void __launch_bounds__(NT) minmax_kernel(const float* m0, const float* m1, const float* m2, const float* m3,
                                                    int npix, uint32_t* __restrict__ work) {
  __shared__ uint32_t part[NT / 32][2];
  const float* m = blockIdx.y == 0 ? m0 : blockIdx.y == 1 ? m1 : blockIdx.y == 2 ? m2 : m3;
  uint32_t lo = 0xffffffffu, hi = 0u;
  for (int i = blockIdx.x * NT + threadIdx.x; i < npix; i += RED_BLK * NT) {
    const float x = m[i];
    const bool nan = x != x;
    lo = min(lo, nan ? 0u : key_of(x));
    hi = max(hi, nan ? 0xffffffffu : key_of(x));
  }
  lo = __reduce_min_sync(0xffffffffu, lo);
  hi = __reduce_max_sync(0xffffffffu, hi);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    part[warp][0] = lo;
    part[warp][1] = hi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < NT / 32; ++w) {
      lo = min(lo, part[w][0]);
      hi = max(hi, part[w][1]);
    }
    work[(blockIdx.y * RED_BLK + blockIdx.x) * 2] = lo;
    work[(blockIdx.y * RED_BLK + blockIdx.x) * 2 + 1] = hi;
  }
}

struct Segs {
  const float* src[MAXSEG];     // a map plane, or a frame's R plane (G and B follow at npix and 2 * npix)
  int npix[MAXSEG];
  long long off[MAXSEG];        // byte offset of the image in dst
  int first_blk[MAXSEG + 1];    // CTAs [first_blk[s], first_blk[s + 1]) own image s
  int nseg, nmaps, normalize;
};

__global__ void __launch_bounds__(NT) images_kernel(const Segs sg, const uint8_t* __restrict__ lut_rgb,
                                                    const uint32_t* __restrict__ work, uint8_t* __restrict__ dst) {
  __shared__ uint8_t lut[256 * 3];
  __shared__ float range[2];
  int s = 0;
  while (s + 1 < sg.nseg && blockIdx.x >= sg.first_blk[s + 1]) ++s;
  const int npix = sg.npix[s];
  const int p0 = (blockIdx.x - sg.first_blk[s]) * (NT * PPT) + threadIdx.x * PPT;
  const bool is_map = s < sg.nmaps;
  uint32_t b[PPT * 3 / 4] = {0u, 0u, 0u};      // the 12 output bytes of this thread's 4 pixels, little-endian

  if (is_map) {
    for (int i = threadIdx.x; i < 256 * 3; i += NT) lut[i] = lut_rgb[i];
    if (sg.normalize && threadIdx.x < 32) {
      const uint32_t* wk = work + s * RED_BLK * 2;
      const uint32_t lo = __reduce_min_sync(0xffffffffu, min(wk[2 * threadIdx.x], wk[2 * (threadIdx.x + 32)]));
      const uint32_t hi = __reduce_max_sync(0xffffffffu, max(wk[2 * threadIdx.x + 1], wk[2 * (threadIdx.x + 32) + 1]));
      if (threadIdx.x == 0) {
        const float mn = float_of(lo);
        range[0] = mn;
        range[1] = __fsub_rn(float_of(hi), mn);   // max(x - min) = fl(max - min): rounding is monotone
      }
    }
    __syncthreads();
    const float mn = sg.normalize ? range[0] : 0.f, den = sg.normalize ? range[1] : 1.f;
#pragma unroll
    for (int j = 0; j < PPT; ++j) {
      if (p0 + j >= npix) break;
      float y = sg.src[s][p0 + j];
      if (sg.normalize) y = __fdiv_rn(__fsub_rn(y, mn), den);
      const float t = __fmul_rn(y, 256.f);          // matplotlib: xa *= N on the float32 array
      uint32_t bgr = 0u;                            // NaN: the "bad" colour, (0, 0, 0)
      if (t == t) {
        const int idx = t >= 256.f ? 255 : (t < 0.f ? 0 : (int)t);   // 256 -> 255, over -> 255, under -> 0, else trunc
        bgr = (uint32_t)lut[3 * idx + 2] | ((uint32_t)lut[3 * idx + 1] << 8) | ((uint32_t)lut[3 * idx] << 16);
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) b[(3 * j + c) >> 2] |= ((bgr >> (8 * c)) & 0xffu) << (8 * ((3 * j + c) & 3));
    }
  } else {
    const float* plane = sg.src[s];
#pragma unroll
    for (int j = 0; j < PPT; ++j) {
      if (p0 + j >= npix) break;
      const uint32_t bgr = rv::frame_bgr8(plane[p0 + j], plane[(size_t)npix + p0 + j], plane[2 * (size_t)npix + p0 + j]);
#pragma unroll
      for (int c = 0; c < 3; ++c) b[(3 * j + c) >> 2] |= ((bgr >> (8 * c)) & 0xffu) << (8 * ((3 * j + c) & 3));
    }
  }

  if (p0 >= npix) return;
  uint8_t* o = dst + sg.off[s] + 3ll * p0;
  if (p0 + PPT <= npix && ((uintptr_t)o & 3) == 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) reinterpret_cast<uint32_t*>(o)[k] = b[k];
  } else {
    const int nb = 3 * min(PPT, npix - p0);
    for (int k = 0; k < nb; ++k) o[k] = (uint8_t)(b[k >> 2] >> (8 * (k & 3)));
  }
}

}  // namespace

extern "C" int rv_conf_map_images(const float* conf, const float* prop, const float* prop_b, const float* prop_f, int h,
                                  int w, int normalize, const float* inp, int ih, int iw, const float* out, int oh, int ow,
                                  const uint8_t* lut_rgb, uint32_t* work, uint8_t* dst, void* stream) {
  RV_REQUIRE(normalize == 0 || normalize == 1, "rv_conf_map_images: normalize must be 0 or 1 (got %d)", normalize);
  RV_REQUIRE(conf && inp && out && lut_rgb && work && dst, "rv_conf_map_images: null pointer");
  RV_REQUIRE(!normalize || (prop && prop_b && prop_f), "rv_conf_map_images: normalize needs all four maps");
  RV_REQUIRE(h >= 1 && w >= 1 && ih >= 1 && iw >= 1 && oh >= 1 && ow >= 1,
             "rv_conf_map_images: empty image (maps %d x %d, input %d x %d, output %d x %d)", h, w, ih, iw, oh, ow);
  const long long caps[3] = {(long long)h * w, (long long)ih * iw, (long long)oh * ow};
  for (long long c : caps) RV_REQUIRE(c <= (1ll << 28), "rv_conf_map_images: an image of %lld pixels is too large", c);

  Segs sg{};
  sg.nmaps = normalize ? 4 : 1;
  sg.normalize = normalize;
  sg.nseg = sg.nmaps + 2;
  const float* srcs[MAXSEG] = {conf, prop, prop_b, prop_f};
  long long off = 0;
  int blk = 0;
  for (int s = 0; s < sg.nseg; ++s) {
    const bool frame = s >= sg.nmaps;
    sg.src[s] = frame ? (s == sg.nmaps ? inp : out) : srcs[s];
    sg.npix[s] = (int)(frame ? (s == sg.nmaps ? caps[1] : caps[2]) : caps[0]);
    sg.off[s] = off;
    sg.first_blk[s] = blk;
    off += 3ll * sg.npix[s];
    blk += (int)rv::cdiv(sg.npix[s], NT * PPT);
  }
  sg.first_blk[sg.nseg] = blk;

  if (normalize) {
    minmax_kernel<<<dim3(RED_BLK, 4), NT, 0, (cudaStream_t)stream>>>(conf, prop, prop_b, prop_f, h * w, work);
    RV_LAUNCH_CHECK("conf_map_minmax");
  }
  images_kernel<<<blk, NT, 0, (cudaStream_t)stream>>>(sg, lut_rgb, work, dst);
  RV_LAUNCH_CHECK("conf_map_images");
  return RV_OK;
}
