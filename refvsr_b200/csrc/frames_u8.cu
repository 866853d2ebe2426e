// rv_frames_from_u8: decoded 8-bit video frames (HWC, RGB or BGR) -> the engine's fp32 planar (3, H, W) frames in [0, 1].
// Byte u becomes fl32(u / 255) (IEEE division, round to nearest): the value data_loader/utils.py::read_frame produces in
// float64 and casts to float32, and the one torch's u8.float() / 255 gives.
//
// A frame is H * W pixels of 3 bytes without row padding, so a thread owns PPT = 16 consecutive pixels (48 bytes) wherever they
// fall in the rows.  The runs start `head` pixels in, where the source is 16-byte aligned, so each run is three 16-byte loads
// whatever the frame's address; its planes are written as 16-byte stores when they are aligned too.  The head and the tail
// (under 16 pixels each) go to one extra thread per frame, byte by byte.
#include "common.cuh"

namespace {

constexpr int NT = 256, PPT = 16, MAXF = 16;

struct U8Frames {
  const uint8_t* src[MAXF];
  float* dst[MAXF];
  int head[MAXF];      // pixels before the first 16-byte aligned run
  int vst[MAXF];       // 16-byte stores for the runs
};

__device__ __forceinline__ float unorm8(uint32_t u) { return __fdiv_rn((float)u, 255.f); }

template <bool BGR>
__global__ void __launch_bounds__(NT) frames_from_u8_kernel(const __grid_constant__ U8Frames f, int npix) {
  const int s = blockIdx.y;
  const uint8_t* __restrict__ src = f.src[s];
  float* __restrict__ dst = f.dst[s];
  const int head = f.head[s];
  const int nrun = (npix - head) / PPT;
  const int i = blockIdx.x * NT + threadIdx.x;
  if (i > nrun) return;
  if (i == nrun) {                                    // the head and the tail, pixel by pixel
    auto one = [&](int p) {
#pragma unroll
      for (int c = 0; c < 3; ++c) dst[(size_t)(BGR ? 2 - c : c) * npix + p] = unorm8(src[3 * (size_t)p + c]);
    };
    for (int p = 0; p < head; ++p) one(p);
    for (int p = head + nrun * PPT; p < npix; ++p) one(p);
    return;
  }
  const int p0 = head + i * PPT;
  const uint4* q = reinterpret_cast<const uint4*>(src + 3 * (size_t)p0);
  uint32_t wd[12];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const uint4 v = __ldg(q + k);
    wd[4 * k] = v.x; wd[4 * k + 1] = v.y; wd[4 * k + 2] = v.z; wd[4 * k + 3] = v.w;
  }
  float v[3][PPT];
#pragma unroll
  for (int j = 0; j < PPT; ++j)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int b = 3 * j + c;
      v[BGR ? 2 - c : c][j] = unorm8((wd[b >> 2] >> (8 * (b & 3))) & 0xffu);
    }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float* o = dst + (size_t)c * npix + p0;
    if (f.vst[s]) {
#pragma unroll
      for (int k = 0; k < PPT / 4; ++k)
        reinterpret_cast<float4*>(o)[k] = make_float4(v[c][4 * k], v[c][4 * k + 1], v[c][4 * k + 2], v[c][4 * k + 3]);
    } else {
#pragma unroll
      for (int j = 0; j < PPT; ++j) o[j] = v[c][j];
    }
  }
}

}  // namespace

extern "C" int rv_frames_from_u8(const uint8_t* const* src, float* const* dst, int k, int h, int w, int bgr, void* stream) {
  RV_REQUIRE(src && dst, "rv_frames_from_u8: null pointer");
  RV_REQUIRE(k >= 1 && k <= MAXF, "rv_frames_from_u8: 1..%d frames (got %d)", MAXF, k);
  RV_REQUIRE(h >= 1 && w >= 1 && (long long)h * w <= (1ll << 28), "rv_frames_from_u8: frames of %d x %d (1..2^28 pixels)", h, w);
  const int npix = h * w;
  U8Frames f{};
  for (int s = 0; s < k; ++s) {
    RV_REQUIRE(src[s] && dst[s], "rv_frames_from_u8: frame %d has a null pointer", s);
    // the first pixel p with src + 3p 16-byte aligned: 3p = -addr (mod 16), and 11 is 3's inverse mod 16
    const int head = min(npix, (int)(((16 - (uintptr_t)src[s] % 16) * 11) % 16));
    f.src[s] = src[s];
    f.dst[s] = dst[s];
    f.head[s] = head;
    f.vst[s] = ((uintptr_t)(dst[s] + head) % 16) == 0 && npix % 4 == 0;
  }
  const dim3 grid(rv::cdiv(npix / PPT + 1, NT), k);
  if (bgr) frames_from_u8_kernel<true><<<grid, NT, 0, (cudaStream_t)stream>>>(f, npix);
  else frames_from_u8_kernel<false><<<grid, NT, 0, (cudaStream_t)stream>>>(f, npix);
  RV_LAUNCH_CHECK("frames_from_u8");
  return RV_OK;
}
