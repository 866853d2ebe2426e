"""Golden vectors of the x2 models (scale=2, matching_ksize=4: configs/config_RefVSR_*.py:30-34), produced by running the
UNMODIFIED reference on CPU - the same recipe as make_golden.py, whose build_case / load_reference this reuses.

    python tests/golden/make_golden_x2.py              # fixture cases + mid-size digest + state-dict keys
    python tests/golden/make_golden_x2.py <case> ...   # only these cases

Writes tests/golden/<case>.npz for the fixture cases, tests/golden/x2_mfid_136x240_digest.npz (8x8 block means, a 128x128
centre crop and sums per window, make_fullsize.py's digest format: the full results would be ~3 MB) and
tests/golden/state_dict_keys_x2.json.  These cases are deliberately not in make_golden.CASES / tests/util.py::CASES, which
the x4 tests parametrise over; tests/test_x2_cpu.py and tests/test_gpu_x2.py read X2_CASES from here.
"""
import importlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

X2 = dict(scale=2, matching_ksize=4)

X2_CASES = {
    # name: same fields as make_golden.CASES
    'x2_small_l1_t3_32x48': dict(config='config_RefVSR_small_L1', over=dict(X2, num_blocks=2, reset_branch=2), T=3, h=32, w=48,
                                 ref_scale=1, frames=4, seed=41),
    'x2_mfid_t5_40x56_ref2x': dict(config='config_RefVSR_MFID', over=dict(X2, num_blocks=2), T=5, h=40, w=56,
                                   ref_scale=2, frames=3, seed=42),
    'x2_small_mfid_t7_24x32': dict(config='config_RefVSR_small_MFID', over=dict(X2, num_blocks=1), T=7, h=24, w=32,
                                   ref_scale=1, frames=5, seed=43),
}

# mid-size parity case: full depth (30 blocks), first and steady window
X2_MID = dict(name='x2_mfid_136x240', config='config_RefVSR_MFID', over=dict(X2), T=7, h=136, w=240, ref_scale=1, frames=2,
              windows=2, seed=44)

X2_CONFIGS = ('config_RefVSR_small_L1', 'config_RefVSR_small_MFID', 'config_RefVSR_L1', 'config_RefVSR_MFID')


def make_mid(RefSRNet):
    from make_fullsize import digest
    from make_golden import ROOT
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip, sliding_windows
    spec = X2_MID
    cfg = importlib.import_module('configs.' + spec['config']).get_config('p', 'm', spec['config'])
    cfg.cuda, cfg.device, cfg.dist = False, 'cpu', False
    for k, v in spec['over'].items():
        setattr(cfg, k, v)
    torch.manual_seed(0)
    ref = RefSRNet(cfg).eval()
    seeded_test_weights(ref, seed=spec['seed'])
    lrs, refs = make_clip(spec['frames'], spec['h'], spec['w'], spec['ref_scale'], seed=spec['seed'])
    small = {}
    with torch.no_grad():
        for k, wl, wr, first in sliding_windows(lrs, refs, spec['T']):
            if k >= spec['windows']:
                break
            res = ref(wl, wr, first, False, False)['result'][0].numpy().astype(np.float32)
            bm, crop = digest(res)
            small[f'blockmean_{k}'] = bm
            small[f'crop_{k}'] = crop
            small[f'sum_{k}'] = np.array([res.astype(np.float64).sum(), (res.astype(np.float64) ** 2).sum()])
            print(spec['name'], 'window', k, 'mean', float(res.mean()), flush=True)
    small['meta'] = np.array([spec['T'], spec['h'], spec['w'], spec['ref_scale'], spec['frames'], spec['seed'], spec['windows']])
    path = os.path.join(ROOT, 'tests', 'golden', spec['name'] + '_digest.npz')
    np.savez_compressed(path, **small)
    print(spec['name'], 'written', os.path.getsize(path) // 1024, 'KiB')


def make_keys(RefSRNet):
    from make_golden import ROOT
    out = {}
    for name in X2_CONFIGS:
        cfg = importlib.import_module('configs.' + name).get_config('p', 'm', name)
        cfg.cuda, cfg.device, cfg.dist = False, 'cpu', False
        for k, v in X2.items():
            setattr(cfg, k, v)
        out[name] = {k: list(v.shape) for k, v in RefSRNet(cfg).state_dict().items()}
    json.dump(out, open(os.path.join(ROOT, 'tests', 'golden', 'state_dict_keys_x2.json'), 'w'))
    print({k: len(v) for k, v in out.items()})


if __name__ == '__main__':
    from make_golden import build_case, load_reference
    torch.set_num_threads(int(os.environ.get('GOLDEN_THREADS', '6')))
    RefSRNet = load_reference()
    want = sys.argv[1:]
    for name, spec in X2_CASES.items():
        if not want or name in want:
            build_case(name, spec, RefSRNet)
    if not want or X2_MID['name'] in want:
        make_mid(RefSRNet)
    if not want or 'keys' in want:
        make_keys(RefSRNet)
