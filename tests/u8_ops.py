"""The 8-bit frame operators on the CPU, for the tests: `frame_u8` (csrc/frame_u8.cuh restated in torch) and `U8OracleOps`, the
oracle's test double (oracle/oracle_ops.py) with the two operators the 8-bit entries add (rv_frames_from_u8, rv_reconstruct_u8)."""
import torch

from oracle.oracle_ops import OracleOps


def frame_u8(x):
    """cv::Mat::convertTo(CV_8U) of fl32(x * 255), as csrc/frame_u8.cuh computes it: round half to even, saturated to [0, 255];
    NaN and values outside int32 become 0"""
    v = x.float() * 255.0
    ok = (v > -2147483648.0) & (v < 2147483648.0)
    return torch.where(ok, torch.round(v).clamp(0, 255), torch.zeros_like(v)).to(torch.uint8)


def hwc_u8(planar, bgr):
    """fp32 RGB (..., 3, H, W) -> the (..., H, W, 3) uint8 bytes rv_reconstruct_u8 writes for it"""
    b = frame_u8(planar)
    if bgr:
        b = b.flip(-3)
    return b.movedim(-3, -1).contiguous()


def planar_f32(u8, bgr):
    """uint8 (..., H, W, 3) frames -> the fp32 (..., 3, H, W) frames forward() takes for them: u8.float() / 255 with IEEE division,
    computed on the CPU (torch's CUDA division by a scalar multiplies by the rounded reciprocal, which is 1 ulp off for 126 of the
    256 bytes), on u8's device"""
    x = u8.cpu().movedim(-1, -3)
    if bgr:
        x = x.flip(-3)
    return (x.float() / 255).contiguous().to(u8.device)


class U8OracleOps(OracleOps):
    def frames_from_u8(self, srcs, dsts, bgr):
        for s, d in zip(srcs, dsts):
            d.copy_(planar_f32(s, bgr))

    def reconstruct_u8(self, x, lr, scale, clamp01, out, bgr):
        tmp = torch.empty(3, out.shape[0], out.shape[1], dtype=torch.float32)
        self.reconstruct(x, lr, scale, clamp01, tmp)
        out.copy_(hwc_u8(tmp, bgr))
