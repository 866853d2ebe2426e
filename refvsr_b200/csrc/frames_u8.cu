// rv_frames_from_u8: decoded 8-bit video frames (HWC, RGB or BGR) -> the engine's fp32 planar (3, H, W) frames in [0, 1].
// Byte u becomes fl32(u / 255) (IEEE division, round to nearest): the value data_loader/utils.py::read_frame produces in
// float64 and casts to float32, and the one torch's u8.float() / 255 gives.
//
// A frame is H * W pixels of 3 bytes without row padding, so a thread owns PPT = 16 consecutive pixels (48 bytes) wherever they
// fall in the rows.  The runs start `head` pixels in, where the source is 16-byte aligned, so each run is three 16-byte loads
// whatever the frame's address; its planes are written as 16-byte stores when they are aligned too.  The head and the tail
// (under 16 pixels each) go to one extra thread per frame, byte by byte.
//
// YUV 4:2:0 frames (I420 / NV12) are first turned into the RGB bytes cv2.cvtColor gives for them (rv::yuv_rgb8), then into
// fl32(u / 255) like the bytes of an RGB frame.  A thread owns a row pair and 16 columns: 2 x 16 Y bytes and the 8 U, V samples
// of its 8 blocks, each read once.  Where the frame is 16-byte aligned and w a multiple of 16, the Y rows are 16-byte loads and
// the chroma 8-byte (I420) or 16-byte (NV12) loads; elsewhere the same bytes are read one by one.
#include "common.cuh"
#include "frame_u8.cuh"

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

struct Yuv420Frames {
  const uint8_t* src[MAXF];
  float* dst[MAXF];
  int vld[MAXF];       // 16-byte Y and 8 / 16-byte chroma loads
  int vst[MAXF];       // 16-byte stores
};

// the 16 bytes a thread reads from one run of a plane: one load of NB / 4 words where vec, n byte loads otherwise
template <int NB>
__device__ __forceinline__ void load_run(const uint8_t* p, int n, bool vec, uint32_t* wd) {
  if (vec) {
    if constexpr (NB == 16) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
      wd[0] = v.x; wd[1] = v.y; wd[2] = v.z; wd[3] = v.w;
    } else {
      const uint2 v = __ldg(reinterpret_cast<const uint2*>(p));
      wd[0] = v.x; wd[1] = v.y;
    }
  } else {
#pragma unroll
    for (int k = 0; k < NB / 4; ++k) wd[k] = 0;
#pragma unroll
    for (int i = 0; i < NB; ++i)
      if (i < n) wd[i >> 2] |= (uint32_t)__ldg(p + i) << (8 * (i & 3));
  }
}

__device__ __forceinline__ uint32_t byte_of(const uint32_t* wd, int i) { return (wd[i >> 2] >> (8 * (i & 3))) & 0xffu; }

template <bool NV12>
__global__ void __launch_bounds__(NT) frames_from_yuv420_kernel(const __grid_constant__ Yuv420Frames f, int h, int w) {
  const int s = blockIdx.y;
  const uint8_t* __restrict__ src = f.src[s];
  float* __restrict__ dst = f.dst[s];
  const int nx = (w + 15) / 16;
  const int i = blockIdx.x * NT + threadIdx.x;
  if (i >= (h / 2) * nx) return;
  const int cy = i / nx, x0 = 16 * (i - cy * nx);
  const int n = min(16, w - x0);                      // even: w is
  const size_t npix = (size_t)h * w;
  const bool vld = f.vld[s];
  uint32_t cw[4];                                     // I420: U bytes 0-7, V bytes 8-15; NV12: U, V pairs
  if (NV12) {
    load_run<16>(src + npix + (size_t)cy * w + x0, n, vld, cw);
  } else {
    load_run<8>(src + npix + (size_t)cy * (w / 2) + x0 / 2, n / 2, vld, cw);
    load_run<8>(src + npix + npix / 4 + (size_t)cy * (w / 2) + x0 / 2, n / 2, vld, cw + 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int y = 2 * cy + r;
    uint32_t yw[4];
    load_run<16>(src + (size_t)y * w + x0, n, vld, yw);
    float v[3][16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const uint32_t u = byte_of(cw, NV12 ? 2 * (j / 2) : j / 2), vv = byte_of(cw, NV12 ? 2 * (j / 2) + 1 : 8 + j / 2);
      uint32_t R, G, B;
      rv::yuv_rgb8(byte_of(yw, j), u, vv, R, G, B);
      v[0][j] = unorm8(R); v[1][j] = unorm8(G); v[2][j] = unorm8(B);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float* o = dst + (size_t)c * npix + (size_t)y * w + x0;
      if (f.vst[s]) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
          reinterpret_cast<float4*>(o)[k] = make_float4(v[c][4 * k], v[c][4 * k + 1], v[c][4 * k + 2], v[c][4 * k + 3]);
      } else {
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (j < n) o[j] = v[c][j];
      }
    }
  }
}

}  // namespace

extern "C" int rv_frames_from_u8(const uint8_t* const* src, float* const* dst, int k, int h, int w, int fmt, void* stream) {
  RV_REQUIRE(src && dst, "rv_frames_from_u8: null pointer");
  RV_REQUIRE(k >= 1 && k <= MAXF, "rv_frames_from_u8: 1..%d frames (got %d)", MAXF, k);
  RV_REQUIRE(h >= 1 && w >= 1 && (long long)h * w <= (1ll << 28), "rv_frames_from_u8: frames of %d x %d (1..2^28 pixels)", h, w);
  RV_REQUIRE(fmt >= RV_FRAME_RGB && fmt <= RV_FRAME_NV12, "rv_frames_from_u8: unknown frame format %d", fmt);
  if (fmt == RV_FRAME_I420 || fmt == RV_FRAME_NV12) {
    RV_REQUIRE(h % 2 == 0 && w % 2 == 0, "rv_frames_from_u8: 4:2:0 frames of %d x %d (even sizes only)", h, w);
    Yuv420Frames f{};
    for (int s = 0; s < k; ++s) {
      RV_REQUIRE(src[s] && dst[s], "rv_frames_from_u8: frame %d has a null pointer", s);
      f.src[s] = src[s];
      f.dst[s] = dst[s];
      f.vld[s] = (uintptr_t)src[s] % 16 == 0 && w % 16 == 0;
      f.vst[s] = (uintptr_t)dst[s] % 16 == 0 && w % 16 == 0;
    }
    const dim3 grid(rv::cdiv((long long)(h / 2) * ((w + 15) / 16), NT), k);
    if (fmt == RV_FRAME_NV12) frames_from_yuv420_kernel<true><<<grid, NT, 0, (cudaStream_t)stream>>>(f, h, w);
    else frames_from_yuv420_kernel<false><<<grid, NT, 0, (cudaStream_t)stream>>>(f, h, w);
    RV_LAUNCH_CHECK("frames_from_yuv420");
    return RV_OK;
  }
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
  if (fmt == RV_FRAME_BGR) frames_from_u8_kernel<true><<<grid, NT, 0, (cudaStream_t)stream>>>(f, npix);
  else frames_from_u8_kernel<false><<<grid, NT, 0, (cudaStream_t)stream>>>(f, npix);
  RV_LAUNCH_CHECK("frames_from_u8");
  return RV_OK;
}
