"""TEST INFRASTRUCTURE - the yardstick of `CudaOps.conf_map_images` (rv_conf_map_images), never imported by the product.

`reference_images(maps, inp, out, normalize)` repeats the reference's per-frame steps (evaluation/eval_quan_conf_map.py:64-165)
on the host: torch float32 min/max normalisation, the `inferno` colormap called on the float32 map, `torch.Tensor` of its RGB,
`* 255`, RGB -> BGR, and the 8-bit conversion cv2.imwrite makes, taken from cv2 itself through a lossless PNG round trip.  The
colormap is matplotlib's when it imports, else the stand-in under tests/conf_map_env (loaded by path, so this process's
`matplotlib` stays unset).  `install()` makes the restatement the drop-in's image kernel on the CPU test double
(oracle.oracle_ops.OracleOps) inside a `run.py` subprocess."""
import importlib.util
import os

import cv2
import numpy as np
import torch

ENV = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'conf_map_env')


def have_matplotlib():
    try:
        import matplotlib.pyplot  # noqa: F401
        return True
    except ImportError:
        return False


def colormap():
    """plt.get_cmap('inferno'): matplotlib's, or the stand-in's"""
    if have_matplotlib():
        import matplotlib.pyplot as plt
        return plt.get_cmap('inferno')
    spec = importlib.util.spec_from_file_location('_conf_map_env_matplotlib', os.path.join(ENV, 'matplotlib', '__init__.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.get_cmap('inferno')


def imwrite_u8(img):
    """the uint8 image cv2.imwrite stores for a float32 image (its convertTo(CV_8U)), read back from a PNG encoding"""
    ok, buf = cv2.imencode('.png', img)
    assert ok
    return cv2.imdecode(buf, cv2.IMREAD_UNCHANGED).reshape(img.shape)


def reference_images(maps, inp, out, normalize, cmap=None):
    """[uint8 BGR (h, w, 3)] in rv_conf_map_images' order: each map, the input, the output.  maps: (1, 1, h, w) tensors,
    inp / out: (1, 3, H, W) tensors, any device"""
    cmap = cmap or colormap()
    imgs = []
    for m in maps:
        m = m.detach().float().cpu()
        if normalize:                                                 # :68-80
            m = m - m.min()
            m = m / m.max()
        rgb = cmap(m.numpy()[0].transpose(1, 2, 0)[:, :, 0])[:, :, :3]   # :82-84
        arr = torch.Tensor(rgb)[None, :].permute(0, 3, 1, 2).numpy()[0].transpose(1, 2, 0)
        imgs.append(imwrite_u8(cv2.cvtColor(arr * 255, cv2.COLOR_RGB2BGR)))
    for f in (inp, out):                                              # :121-122, 142, 146
        arr = f.detach().float().cpu().numpy()[0].transpose(1, 2, 0)
        imgs.append(imwrite_u8(cv2.cvtColor(arr * 255, cv2.COLOR_RGB2BGR)))
    return imgs


def packed(imgs):
    return np.concatenate([np.ascontiguousarray(i).reshape(-1) for i in imgs])


def install():
    """give the CPU test double of the operator set this image step (the product has no CPU path)"""
    from oracle.oracle_ops import OracleOps
    OracleOps.conf_map_images = lambda self, maps, inp, out, lut, normalize: torch.from_numpy(
        packed(reference_images(maps, inp, out, normalize)))
