"""TEST INFRASTRUCTURE - the fp64 yardstick of `CudaOps.region_metrics` (rv_region_metrics), never imported by the product.

`region_metrics(a, b, boxes)` takes the same arguments and returns the same (sq, s) pair, computed in numpy: the float32
squared error summed in fp64, and skimage's SSIM map (uniform 7x7 window in fp64, sample covariance, C1 = 1e-4, C2 = 9e-4)
over the full frame with scipy `reflect` borders (numpy's `symmetric` padding), summed over each box.  The GPU tests compare
the kernel with it, and `install()` makes it the FOV drop-in's metric on the CPU test double (oracle.oracle_ops.OracleOps)
inside a `run.py` subprocess."""
import numpy as np


def _box7(p, H, W):
    """7 x 7 window means of a (C, H + 6, W + 6) padded array"""
    r = sum(p[:, :, k:k + W] for k in range(7))
    return sum(r[:, k:k + H, :] for k in range(7)) / 49.0


def ssim_map(a, b):
    """(3, H, W) float64 SSIM map of two (3, H, W) arrays"""
    H, W = a.shape[1:]
    pa = np.pad(np.asarray(a, np.float64), ((0, 0), (3, 3), (3, 3)), mode='symmetric')
    pb = np.pad(np.asarray(b, np.float64), ((0, 0), (3, 3), (3, 3)), mode='symmetric')
    ux, uy = _box7(pa, H, W), _box7(pb, H, W)
    uxx, uyy, uxy = _box7(pa * pa, H, W), _box7(pb * pb, H, W), _box7(pa * pb, H, W)
    cov_norm = 49.0 / 48.0
    vx, vy, vxy = cov_norm * (uxx - ux * ux), cov_norm * (uyy - uy * uy), cov_norm * (uxy - ux * uy)
    C1, C2 = 1e-4, 9e-4
    return ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux ** 2 + uy ** 2 + C1) * (vx + vy + C2))


def region_metrics(a, b, boxes):
    """a, b: (1, 3, H, W) float32 tensors (any device); boxes: (y0, y1, x0, x1) half-open -> float64 arrays (sq, s)"""
    a32 = a.detach().float().cpu().numpy()[0]
    b32 = b.detach().float().cpu().numpy()[0]
    sq = ((a32 - b32) ** 2).astype(np.float64)
    S = ssim_map(a32, b32)
    sums = [(sq[:, y0:y1, x0:x1].sum(), S[:, y0:y1, x0:x1].sum()) for y0, y1, x0, x1 in boxes]
    return np.array([q for q, _ in sums], np.float64), np.array([s for _, s in sums], np.float64)


def install():
    """give the CPU test double of the operator set this metric (the product has no CPU path)"""
    from oracle.oracle_ops import OracleOps
    OracleOps.region_metrics = lambda self, a, b, boxes: region_metrics(a, b, boxes)
