"""Golden outputs of the UNMODIFIED reference (codeslake/RefVSR) for tests/test_oracle_golden.py::test_oracle_matches_reference_outputs.

Run where a reference checkout exists (its path as the only argument):  python tests/golden/make_reference_small.py <reference dir>
RefVSR_small_MFID, 2 residual blocks, seeded weights (seed 77), a 3-frame 28x36 clip, T = 5; of each window's 1 x 3 x 112 x 144
result a fixed seeded sample of SAMPLE elements is stored (SAMPLE_SEED, flat indices recomputed by the test)."""
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
SAMPLE, SAMPLE_SEED = 8192, 5


def sample_idx(size):
    return np.sort(np.random.default_rng(SAMPLE_SEED).choice(size, size=SAMPLE, replace=False))


def main(ref_dir):
    sys.path[:0] = [os.path.join(ROOT, 'oracle', 'shims'), ref_dir, ROOT]
    import torch
    import torchvision
    _v = torchvision.models.vgg19
    torchvision.models.vgg19 = lambda pretrained=False, **kw: _v(weights=None)
    from models.SRNet import SRNet
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip, sliding_windows
    cfg = importlib.import_module('configs.config_RefVSR_small_MFID').get_config('p', 'm', 'config_RefVSR_small_MFID')
    cfg.cuda, cfg.device, cfg.dist = False, 'cpu', False
    cfg.num_blocks = 2
    ref = SRNet(cfg).eval()
    seeded_test_weights(ref, seed=77)
    lrs, refs = make_clip(3, 28, 36, 1, seed=77)
    outs = []
    with torch.no_grad():
        for k, wl, wr, first in sliding_windows(lrs, refs, 5):
            a = ref(wl, wr, first, False, False)['result'].numpy().astype(np.float32)
            outs.append(a.reshape(-1)[sample_idx(a.size)])
    np.savez(os.path.join(ROOT, 'tests', 'golden', 'reference_small_mfid_t5_28x36.npz'),
             result_sample=np.stack(outs), shape=np.array(a.shape))


if __name__ == '__main__':
    main(sys.argv[1])
