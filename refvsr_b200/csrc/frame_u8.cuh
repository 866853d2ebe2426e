// The 8-bit BGR bytes the evaluation loops store for an fp32 RGB frame.  The reference writes a frame x as
// cv2.imwrite(path, cv2.cvtColor(x * 255, cv2.COLOR_RGB2BGR)): numpy scales in float32, cvtColor only reorders the channels,
// and imwrite converts the float image with cv::Mat::convertTo(CV_8U).  rv_conf_map_images and rv_eval_images both use these.
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

}  // namespace rv
