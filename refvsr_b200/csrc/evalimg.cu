// rv_eval_images: the bytes evaluation/eval_qual_quan.py writes for one frame - the input, the output and the ground truth
// as uint8 BGR HWC images - from their fp32 NCHW RGB frames in one launch, so the host copies 8-bit images and only encodes.
//
// Every thread owns PPT = 16 consecutive pixels of one image.  Where the image's planes and its place in dst are 16-byte
// aligned it reads each plane's 16 values as four 16-byte loads and writes the 48 BGR bytes as three 16-byte stores; an
// image's last partial group, and every group of an unaligned image, converts pixel by pixel.  The conversion is
// rv::frame_bgr8, the one rv_conf_map_images uses for its frames.
#include "common.cuh"
#include "frame_u8.cuh"

namespace {

constexpr int NT = 256, PPT = 16, MAXIMG = 3;

struct Images {
  const float* src[MAXIMG];     // R plane; G and B follow at npix and 2 * npix
  int npix[MAXIMG];
  long long off[MAXIMG];        // byte offset of the image in dst
  int vec[MAXIMG];              // 16-byte loads and stores
  unsigned first_blk[MAXIMG];   // image s owns the CTAs from first_blk[s] on; ~0u for the slots past the last image
};

// a[s] with selects, so the kernel parameter is not copied to local memory for a run-time index
template <typename T>
__device__ __forceinline__ T pick(const T (&a)[MAXIMG], int s) {
  return s == 0 ? a[0] : (s == 1 ? a[1] : a[2]);
}

__global__ void __launch_bounds__(NT) eval_images_kernel(const Images im, uint8_t* __restrict__ dst) {
  const int s = (int)(blockIdx.x >= im.first_blk[1]) + (int)(blockIdx.x >= im.first_blk[2]);
  const int npix = pick(im.npix, s);
  const int p0 = (blockIdx.x - pick(im.first_blk, s)) * (NT * PPT) + threadIdx.x * PPT;
  if (p0 >= npix) return;
  const float* __restrict__ r = pick(im.src, s);
  uint8_t* o = dst + pick(im.off, s) + 3ll * p0;

  if (pick(im.vec, s) && p0 + PPT <= npix) {
    float v[3][PPT];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float4* q = reinterpret_cast<const float4*>(r + (size_t)c * npix + p0);
#pragma unroll
      for (int k = 0; k < PPT / 4; ++k) {
        const float4 f = q[k];
        v[c][4 * k] = f.x;
        v[c][4 * k + 1] = f.y;
        v[c][4 * k + 2] = f.z;
        v[c][4 * k + 3] = f.w;
      }
    }
    uint32_t b[3 * PPT / 4] = {};                   // the 48 output bytes, little-endian
#pragma unroll
    for (int j = 0; j < PPT; ++j) {
      const uint32_t bgr = rv::frame_bgr8(v[0][j], v[1][j], v[2][j]);
#pragma unroll
      for (int c = 0; c < 3; ++c) b[(3 * j + c) >> 2] |= ((bgr >> (8 * c)) & 0xffu) << (8 * ((3 * j + c) & 3));
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) reinterpret_cast<uint4*>(o)[k] = make_uint4(b[4 * k], b[4 * k + 1], b[4 * k + 2], b[4 * k + 3]);
  } else {
    const int n = min(PPT, npix - p0);
    for (int j = 0; j < n; ++j) {
      const size_t p = (size_t)p0 + j;
      const uint32_t bgr = rv::frame_bgr8(r[p], r[npix + p], r[2 * (size_t)npix + p]);
      o[3 * j] = (uint8_t)bgr;
      o[3 * j + 1] = (uint8_t)(bgr >> 8);
      o[3 * j + 2] = (uint8_t)(bgr >> 16);
    }
  }
}

}  // namespace

extern "C" int rv_eval_images(const float* const* frames, const int* hw_host, int nframes, uint8_t* dst, void* stream) {
  RV_REQUIRE(frames && hw_host && dst, "rv_eval_images: null pointer");
  RV_REQUIRE(nframes >= 1 && nframes <= MAXIMG, "rv_eval_images: 1..%d frames (got %d)", MAXIMG, nframes);
  Images im{};
  for (int s = 0; s < MAXIMG; ++s) im.first_blk[s] = ~0u;
  long long off = 0;
  long long blk = 0;
  for (int s = 0; s < nframes; ++s) {
    const int H = hw_host[2 * s], W = hw_host[2 * s + 1];
    RV_REQUIRE(frames[s], "rv_eval_images: frame %d is a null pointer", s);
    RV_REQUIRE(H >= 1 && W >= 1 && (long long)H * W <= (1ll << 28), "rv_eval_images: frame %d is %d x %d (1..2^28 pixels)", s, H,
               W);
    im.src[s] = frames[s];
    im.npix[s] = H * W;
    im.off[s] = off;
    im.vec[s] = ((uintptr_t)frames[s] & 15) == 0 && (im.npix[s] & 3) == 0 && (((uintptr_t)dst + off) & 15) == 0;
    im.first_blk[s] = (unsigned)blk;
    off += 3ll * im.npix[s];
    blk += rv::cdiv(im.npix[s], NT * PPT);
  }
  eval_images_kernel<<<(unsigned)blk, NT, 0, (cudaStream_t)stream>>>(im, dst);
  RV_LAUNCH_CHECK("eval_images");
  return RV_OK;
}
