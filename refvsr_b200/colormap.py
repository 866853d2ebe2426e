"""The colour table of the confidence-map evaluation mode (evaluation/eval_quan_conf_map.py:19-20: matplotlib's `inferno`) as
the 8-bit values the reference's images hold.

The reference colours a map with `colormap(x)[:, :, :3]` (float64 RGB), turns it into a float32 tensor, multiplies by 255 and
hands it to cv2.imwrite, which rounds half to even.  So entry i of the table is round(fl32(fl32(lut[i]) * 255)).  The float
table comes from matplotlib when it imports; otherwise from OpenCV's COLORMAP_INFERNO, which carries the same 6-decimal data
and is already 8-bit (its float32 entries times 255, rounded the same way)."""
import numpy as np
import torch

_device_luts = {}


def rgb8_of(rgb):
    """(256, 3) float RGB in [0, 1] -> uint8: round half to even of fl32(fl32(v) * 255), as cv2.imwrite stores fl32(v) * 255"""
    v = np.asarray(rgb, dtype=np.float64).astype(np.float32) * np.float32(255)
    return np.clip(np.rint(v), 0, 255).astype(np.uint8)


def matplotlib_inferno_rgb8():
    """the table from matplotlib's get_cmap('inferno'), as the reference takes it; ImportError without matplotlib"""
    import matplotlib.pyplot as plt
    cmap = plt.get_cmap('inferno')
    return rgb8_of(np.asarray(cmap(np.arange(256)))[:, :3])           # integer inputs index the table directly


def opencv_inferno_rgb8():
    """the table from OpenCV's COLORMAP_INFERNO (BGR, applied to 0..255), as RGB"""
    import cv2
    bgr = cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(256, 1), cv2.COLORMAP_INFERNO)
    return np.ascontiguousarray(bgr[:, 0, ::-1])


def inferno_rgb8():
    """(256, 3) uint8 RGB inferno table: matplotlib's when it imports, else OpenCV's"""
    try:
        return matplotlib_inferno_rgb8()
    except ImportError:
        return opencv_inferno_rgb8()


def inferno_lut(device):
    """inferno_rgb8() as a uint8 (256, 3) tensor on `device`, uploaded once per device"""
    device = torch.device(device)
    if device not in _device_luts:
        _device_luts[device] = torch.from_numpy(inferno_rgb8()).to(device)
    return _device_luts[device]
