// The 8-bit BGR bytes the evaluation loops store for an fp32 RGB frame.  The reference writes a frame x as
// cv2.imwrite(path, cv2.cvtColor(x * 255, cv2.COLOR_RGB2BGR)): numpy scales in float32, cvtColor only reorders the channels,
// and imwrite converts the float image with cv::Mat::convertTo(CV_8U).  rv_conf_map_images, rv_eval_images and the 8-bit frame
// paths (rv_frames_from_u8, rv_reconstruct_u8) use these.
#pragma once
#include "common.cuh"

namespace rv {

// cv::Mat::convertTo(CV_8U) of fl32(x * 255): cvRound (round half to even), then saturation; x86's conversion turns NaN and
// values outside int32 into INT_MIN, which saturates to 0
__device__ __forceinline__ uint32_t frame_u8(float x) {
  const float v = __fmul_rn(x, 255.f);
  if (!(v > -2147483648.f && v < 2147483648.f)) return 0u;
  return (uint32_t)clampi(__float2int_rn(v), 0, 255);
}

// one pixel's B, G and R bytes, in that order from the low byte up, from its R, G and B values
__device__ __forceinline__ uint32_t frame_bgr8(float r, float g, float b) {
  return frame_u8(b) | (frame_u8(g) << 8) | (frame_u8(r) << 16);
}

// ---- YUV 4:2:0 (RV_FRAME_I420 / RV_FRAME_NV12): OpenCV's cvtColor conversions, BT.601 limited range in 20-bit fixed point.
// These are the integer formulas of COLOR_YUV2RGB_I420 / _NV12 (nearest chroma: one U, V sample per 2 x 2 block) and of
// COLOR_RGB2YUV_I420 (U and V from each block's top-left pixel), bit for bit; tests/yuv_ops.py restates them.
__device__ __forceinline__ uint32_t sat8(int v) { return (uint32_t)clampi(v, 0, 255); }

// the R, G, B bytes of a pixel from its Y byte and its block's U, V bytes
__device__ __forceinline__ void yuv_rgb8(uint32_t y, uint32_t u, uint32_t v, uint32_t& r, uint32_t& g, uint32_t& b) {
  const int yy = max((int)y - 16, 0) * 1220542, uu = (int)u - 128, vv = (int)v - 128;
  r = sat8((yy + 1673527 * vv + (1 << 19)) >> 20);
  g = sat8((yy - 852492 * vv - 409993 * uu + (1 << 19)) >> 20);
  b = sat8((yy + 2116026 * uu + (1 << 19)) >> 20);
}

// the Y byte of a pixel, and the U, V bytes of the block whose top-left pixel it is, from its R, G, B bytes
__device__ __forceinline__ uint32_t rgb8_y(uint32_t r, uint32_t g, uint32_t b) {
  return sat8((269484 * (int)r + 528482 * (int)g + 102760 * (int)b + (16 << 20) + (1 << 19)) >> 20);
}
__device__ __forceinline__ uint32_t rgb8_u(uint32_t r, uint32_t g, uint32_t b) {
  return sat8((-155188 * (int)r - 305135 * (int)g + 460324 * (int)b + (128 << 20) + (1 << 19)) >> 20);
}
__device__ __forceinline__ uint32_t rgb8_v(uint32_t r, uint32_t g, uint32_t b) {
  return sat8((460324 * (int)r - 385875 * (int)g - 74448 * (int)b + (128 << 20) + (1 << 19)) >> 20);
}

}  // namespace rv
