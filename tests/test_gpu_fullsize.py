"""-m gpu: parity AT THE BENCHMARKED CONFIGURATIONS (VERDICT r1 item 2) - 270x480 LR -> 1080p, full depth (30 / 24 blocks):
first, steady, forced-reset and post-reset windows against full-size golden vectors computed in the build container by

  * the UNMODIFIED reference on CPU for BASELINE configs[2] (config_RefVSR_MFID, Ref 270x480), and
  * the oracle port for configs[1] (config_RefVSR_small_MFID, Ref 540x960: the reference's 67 GB similarity matrix does not
    fit the container; the oracle is pinned to the reference at fixture sizes, tests/test_oracle_golden.py),

tests/golden/make_fullsize.py -> tests/golden_large/*.npz (git-ignored, ~110 MB each, travels with the working tree) and the
committed digests tests/golden/*_digest.npz (8x8 block means + centre crops) used when the large file is absent.

Bars (north_star: 1e-3 relative fp32, PSNR delta < 0.01 dB):
  fp32 path   PSNR vs reference >= 80 dB, 99.9 % of the pixels within 1e-3 (the hard argmax may flip near-ties: a handful of
              pixels can differ by more, which is why max-abs is reported, not bounded at 1e-3)
  16-bit path PSNR vs reference >= 60 dB (VERDICT r1: "raise the 42 dB bar"); index-map flip rate reported.
With REFVSR_PARITY_LOG=<file> every run appends its numbers there as JSON lines."""
import json
import os

import numpy as np
import pytest
import torch

from util import GOLDEN_DIR, psnr

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LARGE = os.path.join(ROOT, 'tests', 'golden_large')

FULL = {
    'mfid_270x480': dict(config='config_RefVSR_MFID', ref_scale=1, order='reference'),
    'small_mfid_270x480_ref2x': dict(config='config_RefVSR_small_MFID', ref_scale=2, order='oracle'),
}


def _report(rec):
    path = os.environ.get('REFVSR_PARITY_LOG')
    if path:
        with open(path, 'a') as f:
            f.write(json.dumps(rec) + '\n')


def _load(name):
    big = os.path.join(LARGE, name + '.npz')
    small = os.path.join(GOLDEN_DIR, name + '_digest.npz')
    if os.path.isfile(big):
        return np.load(big), True
    if os.path.isfile(small):
        return np.load(small), False
    pytest.skip(f'no golden vectors for {name} (run tests/golden/make_fullsize.py in the build container)')


def _flow_slots(N, t, order):
    """ring flows of the first window in the golden file's order -> list of (golden index, tensor (h,w,2))"""
    mid = t // 2
    h, w = N._state[0]['shape'][1:3]
    out = []
    if order == 'reference':          # hooked FlowNet calls: fw j = 0..t-2, then bw for j = t-1..1 (index j-1)  RefVSR.py:182-189
        for j in range(0, mid + 1):
            out.append((j, N._ring('fw', j, t, (h, w, 2))))
        for j in range(mid, t - 1):
            out.append((t - 1 + (t - 2 - j), N._ring('bw', j, t, (h, w, 2))))
    else:                             # oracle trace: consumed flows only, fw sorted then bw sorted
        fw = list(range(0, mid + 1))
        bw = list(range(mid, t - 1))
        for n, j in enumerate(fw):
            out.append((n, N._ring('fw', j, t, (h, w, 2))))
        for n, j in enumerate(bw):
            out.append((len(fw) + n, N._ring('bw', j, t, (h, w, 2))))
    return out


@pytest.mark.parametrize('name,prec', [('mfid_270x480', 'fp32'), ('mfid_270x480', 'bf16'), ('mfid_270x480', 'fp16'),
                                       ('small_mfid_270x480_ref2x', 'fp16'), ('small_mfid_270x480_ref2x', 'fp32')])
def test_fullsize_parity(name, prec):
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip, sliding_windows
    spec = FULL[name]
    gold, full = _load(name)
    T, h, w, ref_scale, frames, seed, nwin = (int(v) for v in gold['meta'])
    cfg = get_config(spec['config'], device='cuda', reset_branch=2, b200_precision=prec)
    net = SRNet(cfg).eval()
    seeded_test_weights(net, seed=seed)
    net = net.cuda()
    lrs, refs = make_clip(frames, h, w, ref_scale, seed=seed)
    rec = dict(case=name, precision=prec, match_mode=net.Network.match_mode, golden='full' if full else 'digest', windows=[])
    kinds = ['first', 'steady', 'forced-reset', 'steady-after-reset']
    for k, wl, wr, first in sliding_windows(lrs, refs, T):
        if k >= nwin:
            break
        out = net(wl.cuda(), wr.cuda(), first, False, False)['result'][0].float().cpu()
        if k == 0 and full and 'idx_0' in gold.files:
            N = net.Network
            flips, dconf = [], []
            for i in range(T):
                slot = N._frame_slot(i % T, h, w)
                flips.append(float((slot['idx'].cpu().numpy() != gold['idx_0'][i]).mean()))
                dconf.append(float(np.abs(slot['conf'].cpu().numpy() - gold['conf_0'][i, 0]).max()))
            dflow = [float((fl.cpu() - torch.from_numpy(gold['flows_0'][gi]).permute(1, 2, 0)).abs().max())
                     for gi, fl in _flow_slots(N, T, spec['order'])]
            rec.update(index_flip_rate=float(np.mean(flips)), conf_max_abs=max(dconf), flow_max_abs_px=max(dflow))
        if full:
            g = torch.from_numpy(gold[f'result_{k}'])
            d = (out - g).abs()
            wrec = dict(window=k, kind=kinds[k], psnr_db=psnr(out, g), max_abs=float(d.max()), p999_abs=float(d.flatten().kthvalue(int(0.999 * d.numel())).values),
                        rel_l2=float((out - g).norm() / g.norm()), mean_out=float(out.mean()), mean_ref=float(g.mean()))
        else:
            bm = torch.nn.functional.avg_pool2d(out.unsqueeze(0), 8)[0]
            gb = torch.from_numpy(gold[f'blockmean_{k}'])
            H4, W4 = out.shape[1:]
            crop = out[:, H4 // 2 - 64:H4 // 2 + 64, W4 // 2 - 64:W4 // 2 + 64]
            gc = torch.from_numpy(gold[f'crop_{k}'])
            d = (crop - gc).abs()
            wrec = dict(window=k, kind=kinds[k], psnr_db=psnr(crop, gc), max_abs=float(d.max()), p999_abs=float(d.flatten().kthvalue(int(0.999 * d.numel())).values),
                        blockmean_max_abs=float((bm - gb).abs().max()), rel_l2=float((crop - gc).norm() / gc.norm()))
        print(f'{name}/{prec} window {k} ({kinds[k]}): ' + ', '.join(f'{a}={b:.3e}' if isinstance(b, float) else f'{a}={b}' for a, b in wrec.items() if a not in ('window', 'kind')))
        rec['windows'].append(wrec)
    _report(rec)
    if 'index_flip_rate' in rec:
        print(f'{name}/{prec}: index flip rate {rec["index_flip_rate"]:.4%}, conf max abs {rec["conf_max_abs"]:.2e}, flow max abs {rec["flow_max_abs_px"]:.2e} px')
    for wrec in rec['windows']:
        if prec == 'fp32':
            assert wrec['psnr_db'] >= 80.0 and wrec['p999_abs'] <= 1e-3, wrec
        else:
            assert wrec['psnr_db'] >= 60.0, wrec
    if prec == 'fp32' and 'flow_max_abs_px' in rec:
        assert rec['flow_max_abs_px'] <= 2e-2 and rec['index_flip_rate'] <= 2e-3
