"""The YUV 4:2:0 frame conversions on the CPU, for the tests: OpenCV's cvtColor (BT.601 limited range, 20-bit fixed point) restated
in numpy, as csrc/frame_u8.cuh computes it, and `YuvOracleOps`, the 8-bit test double (tests/u8_ops.py) with the I420 and NV12
formats of rv_frames_from_u8 and rv_reconstruct_u8."""
import numpy as np
import torch

from u8_ops import U8OracleOps, hwc_u8, planar_f32

FRAME_I420, FRAME_NV12 = 2, 3


def _sat8(x):
    return np.clip(x, 0, 255).astype(np.uint8)


def yuv420_to_rgb(frame, nv12=False):
    """cv2.cvtColor(frame, COLOR_YUV2RGB_I420 / _NV12) for uint8 (..., 3h/2, w) frames -> (..., h, w, 3) uint8; nearest chroma"""
    f = np.asarray(frame.cpu() if isinstance(frame, torch.Tensor) else frame)
    h, w = 2 * f.shape[-2] // 3, f.shape[-1]
    y = f[..., :h, :].astype(np.int32)
    c = f[..., h:, :]
    if nv12:
        u, v = c[..., 0::2], c[..., 1::2]                                   # (..., h/2, w/2) each
    else:
        flat = c.reshape(c.shape[:-2] + (-1,))
        u = flat[..., :h * w // 4].reshape(c.shape[:-2] + (h // 2, w // 2))
        v = flat[..., h * w // 4:].reshape(c.shape[:-2] + (h // 2, w // 2))
    u = np.repeat(np.repeat(u.astype(np.int32) - 128, 2, -2), 2, -1)
    v = np.repeat(np.repeat(v.astype(np.int32) - 128, 2, -2), 2, -1)
    yy = np.maximum(y - 16, 0) * 1220542
    r = _sat8((yy + 1673527 * v + (1 << 19)) >> 20)
    g = _sat8((yy - 852492 * v - 409993 * u + (1 << 19)) >> 20)
    b = _sat8((yy + 2116026 * u + (1 << 19)) >> 20)
    out = np.stack([r, g, b], -1)
    return torch.from_numpy(out) if isinstance(frame, torch.Tensor) else out


def rgb_y(r, g, b):
    return _sat8((269484 * r + 528482 * g + 102760 * b + (16 << 20) + (1 << 19)) >> 20)


def rgb_u(r, g, b):
    return _sat8((-155188 * r - 305135 * g + 460324 * b + (128 << 20) + (1 << 19)) >> 20)


def rgb_v(r, g, b):
    return _sat8((460324 * r - 385875 * g - 74448 * b + (128 << 20) + (1 << 19)) >> 20)


def rgb_to_yuv420(rgb, nv12=False):
    """cv2.cvtColor(rgb, COLOR_RGB2YUV_I420) for uint8 (..., h, w, 3) frames -> (..., 3h/2, w) uint8, U and V from each 2 x 2
    block's top-left pixel; nv12: the same samples interleaved (cv2 has no RGB -> NV12 conversion)"""
    a = np.asarray(rgb.cpu() if isinstance(rgb, torch.Tensor) else rgb).astype(np.int32)
    h, w = a.shape[-3], a.shape[-2]
    y = rgb_y(a[..., 0], a[..., 1], a[..., 2])
    tl = a[..., 0::2, 0::2, :]
    u, v = rgb_u(tl[..., 0], tl[..., 1], tl[..., 2]), rgb_v(tl[..., 0], tl[..., 1], tl[..., 2])
    if nv12:
        c = np.stack([u, v], -1).reshape(u.shape[:-2] + (h // 2, w))
    else:
        c = np.concatenate([u.reshape(u.shape[:-2] + (-1,)), v.reshape(v.shape[:-2] + (-1,))], -1).reshape(u.shape[:-2] + (h // 2, w))
    out = np.ascontiguousarray(np.concatenate([y, c], -2))
    return torch.from_numpy(out) if isinstance(rgb, torch.Tensor) else out


class YuvOracleOps(U8OracleOps):
    def frames_from_u8(self, srcs, dsts, fmt):
        if fmt not in (FRAME_I420, FRAME_NV12):
            return super().frames_from_u8(srcs, dsts, fmt)
        for s, d in zip(srcs, dsts):
            d.copy_(planar_f32(yuv420_to_rgb(s, fmt == FRAME_NV12), False))

    def reconstruct_u8(self, x, lr, scale, clamp01, out, fmt):
        if fmt not in (FRAME_I420, FRAME_NV12):
            return super().reconstruct_u8(x, lr, scale, clamp01, out, fmt)
        tmp = torch.empty(3, 2 * out.shape[0] // 3, out.shape[1], dtype=torch.float32)
        self.reconstruct(x, lr, scale, clamp01, tmp)
        out.copy_(rgb_to_yuv420(hwc_u8(tmp, False), fmt == FRAME_NV12))
