"""TEST INFRASTRUCTURE - a stand-in for the part of matplotlib the reference's confidence-map evaluation uses
(evaluation/eval_quan_conf_map.py:19-20, 83: `plt.get_cmap('inferno')` called on a float32 array).  tests/test_conf_map_eval.py
puts this directory on a subprocess's PYTHONPATH only when the real matplotlib does not import, and never ships it.

The table is OpenCV's COLORMAP_INFERNO (8-bit) divided by 255; `__call__` restates matplotlib's `Colormap.__call__` for float
arrays: xa = X * N in X's dtype, N -> N - 1, then under (< 0) -> the first colour, over (>= N) -> the last, NaN -> the "bad"
colour (0, 0, 0, 0), the rest truncated to an index."""
import numpy as np


class ListedColormap:
    def __init__(self, rgb, name):
        self.name, self.N = name, len(rgb)
        self._i_under, self._i_over, self._i_bad = self.N, self.N + 1, self.N + 2
        lut = np.ones((self.N + 3, 4), np.float64)
        lut[:self.N, :3] = rgb
        lut[self._i_under] = lut[0]
        lut[self._i_over] = lut[self.N - 1]
        lut[self._i_bad] = 0.
        self._lut = lut

    def __call__(self, X):
        xa = np.array(X, copy=True)
        if xa.dtype.kind == 'f':
            xa *= self.N
            xa[xa == self.N] = self.N - 1
        mask_under, mask_over = xa < 0, xa >= self.N
        mask_bad = np.isnan(xa) if xa.dtype.kind == 'f' else np.zeros(xa.shape, bool)
        with np.errstate(invalid='ignore'):
            xa = xa.astype(int)
        xa[mask_under] = self._i_under
        xa[mask_over] = self._i_over
        xa[mask_bad] = self._i_bad
        return self._lut.take(xa, axis=0, mode='clip')


def _inferno():
    import cv2
    bgr = cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(256, 1), cv2.COLORMAP_INFERNO)[:, 0]
    return ListedColormap(bgr[:, ::-1].astype(np.float64) / 255.0, 'inferno')


def get_cmap(name):
    if name != 'inferno':
        raise ValueError(f'the test stand-in of matplotlib only has inferno, not {name!r}')
    return _inferno()
