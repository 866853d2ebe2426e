"""-m gpu: the x2 models (scale=2, matching_ksize=4) through SRNet.forward on the GPU against golden vectors of the unmodified
reference (tests/golden/make_golden_x2.py), the exactness of reuse / CUDA graphs / branch overlap / push_frame at x2, and the x2
pointwise fast paths (4x4 block gather, ks-4 aligned sampling, x2 reconstruction) against the generic kernels.

Bars are those of the x4 tests (tests/test_gpu_model.py, tests/test_gpu_fullsize.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from util import GOLDEN_DIR, psnr
from x2_util import X2_CASES, X2_MID, build_x2_case

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def run_clip(net, lrs, refs, T):
    from refvsr_b200.synth import sliding_windows
    return [net(wl.cuda(), wr.cuda(), first, False, False)['result'][0].float().cpu()
            for k, wl, wr, first in sliding_windows(lrs, refs, T)]


@pytest.mark.parametrize('name', list(X2_CASES))
def test_x2_fp32_path_matches_reference_golden(name):
    spec, cfg, net, lrs, refs, golden = build_x2_case(name, 'cuda', b200_precision='fp32')
    for k, o in enumerate(run_clip(net, lrs, refs, spec['T'])):
        g = torch.from_numpy(golden[f'result_{k}'])
        assert o.shape == g.shape == (3, 2 * spec['h'], 2 * spec['w'])
        p, err = psnr(o, g), (o - g).abs().max().item()
        print(f'{name} window {k}: psnr {p:.1f} dB, max abs {err:.2e}')
        assert p >= 80.0 and err <= 5e-3, f'{name} window {k}: PSNR {p:.1f} dB, max abs {err:.2e}'


@pytest.mark.parametrize('name', list(X2_CASES))
def test_x2_first_window_products_match_reference_golden(name):
    """flows, confidence maps (bicubic x2 of the 1/2-resolution relevance map) and index maps ((h/2)(w/2) entries) of the first
    window against the reference's hooked outputs"""
    from refvsr_b200.synth import sliding_windows
    spec, cfg, net, lrs, refs, golden = build_x2_case(name, 'cuda', b200_precision='fp32')
    T, h, w = spec['T'], spec['h'], spec['w']
    k, wl, wr, first = next(iter(sliding_windows(lrs, refs, T)))
    net(wl.cuda(), wr.cuda(), True, False, False)
    N = net.Network
    mid = T // 2
    for j in range(0, mid + 1):
        if mid == T - 1 and j == mid:
            continue
        f = N._ring('fw', j, T, (h, w, 2)).cpu()
        assert (f - torch.from_numpy(golden['flows_0'][j]).permute(1, 2, 0)).abs().max() <= 2e-3
    for j in range(mid, T - 1):
        f = N._ring('bw', j, T, (h, w, 2)).cpu()
        assert (f - torch.from_numpy(golden['flows_0'][T - 1 + (T - 2 - j)]).permute(1, 2, 0)).abs().max() <= 2e-3
    flips = []
    for i in range(T):
        slot = N._frame_slot(i % T, h, w)
        idx, conf = slot['idx'].cpu().numpy(), slot['conf'].cpu().numpy()
        assert idx.shape == ((h // 2) * (w // 2),) and conf.shape == (h, w)
        flips.append(float((idx != golden['idx_0'][i]).mean()))
        d = np.abs(conf - golden['conf_0'][i, 0]).max()
        assert d <= 2e-3, f'frame {i}: conf {d:.2e}'
    print(f'{name}: index flip rate vs reference {np.mean(flips):.4%}')
    assert np.mean(flips) <= 2e-3


@pytest.mark.parametrize('name', list(X2_CASES))
@pytest.mark.parametrize('prec,bar', [('fp16', 55.0), ('bf16', 42.0)])
def test_x2_16bit_tensor_core_path(name, prec, bar):
    spec, cfg, net, lrs, refs, golden = build_x2_case(name, 'cuda', b200_precision=prec)
    for k, o in enumerate(run_clip(net, lrs, refs, spec['T'])):
        g = torch.from_numpy(golden[f'result_{k}'])
        p = psnr(o, g)
        print(f'{name}/{prec} window {k}: psnr {p:.1f} dB, max abs {(o - g).abs().max().item():.2e}')
        assert p >= bar, f'{name}/{prec} window {k}: PSNR vs reference {p:.1f} dB < {bar}'


def test_x2_reuse_is_exact():
    res = {}
    for reuse in (True, False):
        spec, cfg, net, lrs, refs, golden = build_x2_case('x2_small_mfid_t7_24x32', 'cuda', b200_precision='bf16', b200_reuse=reuse)
        res[reuse] = run_clip(net, lrs, refs, spec['T'])
    for a, b in zip(res[True], res[False]):
        assert torch.equal(a, b)


def _x2_net(name, seed, **over):
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    net = SRNet(get_config(name, device='cuda', scale=2, matching_ksize=4, **over)).eval()
    seeded_test_weights(net, seed=seed)
    return net.cuda()


def test_x2_cuda_graphs_and_branch_overlap_are_exact():
    """whole-window CUDA graphs and the forward step on a second stream vs eager sequential launches: bit identical across steady
    windows, ring wrap-around and forced resets"""
    from refvsr_b200.synth import make_clip, sliding_windows
    lrs, refs = make_clip(20, 40, 56, 1, seed=9)
    res = {}
    for overlap, graphs in ((False, False), (False, True), (True, True), (True, False)):
        net = _x2_net('RefVSR_MFID', 9, num_blocks=3, b200_precision='bf16', b200_cuda_graphs=graphs, b200_overlap_branches=overlap,
                      b200_overlap_cap=70)
        res[(overlap, graphs)] = [net(wl.cuda(), wr.cuda(), first, False, False)['result'].cpu()
                                  for k, wl, wr, first in sliding_windows(lrs, refs, 7)]
        if graphs:
            assert len(net.Network._graphs) >= 8, 'graphs must actually have been captured'
    for key in ((False, True), (True, True), (True, False)):
        for k, (a, b) in enumerate(zip(res[key], res[(False, False)])):
            assert a.shape == (1, 3, 80, 112) and torch.equal(a, b), f'window {k}: {key} differs from eager sequential'


def test_x2_push_frame_equals_forward():
    from refvsr_b200.synth import make_clip, sliding_windows
    lrs, refs = make_clip(18, 40, 56, 1, seed=11)
    wins = list(sliding_windows(lrs, refs, 7))
    outs = {}
    for mode in ('forward', 'push'):
        net = _x2_net('RefVSR_MFID', 11, num_blocks=2, b200_precision='bf16')
        res = []
        for k, wl, wr, first in wins:
            if mode == 'forward' or k == 0:
                res.append(net(wl.cuda(), wr.cuda(), first, False, False)['result'][0].cpu())
            else:
                res.append(net.push_frame(wl[0, -1].cuda(), wr[0, -1].cuda()).cpu())
        outs[mode] = res
    for k, (a, b) in enumerate(zip(outs['push'], outs['forward'])):
        assert torch.equal(a, b), f'window {k}: push_frame differs from forward()'


@pytest.mark.parametrize('prec', ['fp32', 'bf16'])
def test_x2_mid_size_parity(prec):
    """MFID x2 at full depth (30 blocks), LR 136x240 -> 272x480, first and steady window, against the digest of the reference's
    results (8x8 block means + 128x128 centre crop)"""
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip, sliding_windows
    from refvsr_b200 import SRNet, get_config
    gold = np.load(os.path.join(GOLDEN_DIR, X2_MID['name'] + '_digest.npz'))
    T, h, w, ref_scale, frames, seed, nwin = (int(v) for v in gold['meta'])
    net = SRNet(get_config(X2_MID['config'], device='cuda', b200_precision=prec, **X2_MID['over'])).eval()
    seeded_test_weights(net, seed=seed)
    net = net.cuda()
    lrs, refs = make_clip(frames, h, w, ref_scale, seed=seed)
    for k, wl, wr, first in sliding_windows(lrs, refs, T):
        if k >= nwin:
            break
        out = net(wl.cuda(), wr.cuda(), first, False, False)['result'][0].float().cpu()
        assert out.shape == (3, 2 * h, 2 * w)
        bm = torch.nn.functional.avg_pool2d(out.unsqueeze(0), 8)[0]
        H, W = out.shape[1:]
        crop = out[:, H // 2 - 64:H // 2 + 64, W // 2 - 64:W // 2 + 64]
        gc = torch.from_numpy(gold[f'crop_{k}'])
        d = (crop - gc).abs()
        p, p999 = psnr(crop, gc), float(d.flatten().kthvalue(int(0.999 * d.numel())).values)
        bmd = float((bm - torch.from_numpy(gold[f'blockmean_{k}'])).abs().max())
        print(f'{X2_MID["name"]}/{prec} window {k}: crop psnr {p:.1f} dB, p99.9 abs {p999:.2e}, max abs {float(d.max()):.2e}, '
              f'block-mean max abs {bmd:.2e}')
        if prec == 'fp32':
            assert p >= 80.0 and p999 <= 1e-3 and bmd <= 1e-3
        else:
            assert p >= 42.0


def test_x2_pointwise_fast_paths_are_bit_identical(tmp_path):
    """gather_cells_kernel with 4x4 blocks, aligned_sample4_kernel and reconstruct2_kernel against the generic kernels
    (REFVSR_NO_FAST_POINTWISE=1, read once per process -> two subprocesses) on seeded inputs at x2 and 8K shapes, in every dtype;
    the fast kernels must actually have run; the fp32 outputs must agree with OracleOps"""
    from oracle.oracle_ops import OracleOps
    sys.path.insert(0, HERE)
    from x2_kernel_dump import SHAPES, inputs
    res = {}
    for fast in (True, False):
        env = dict(os.environ)
        env.pop('REFVSR_NO_FAST_POINTWISE', None)
        if not fast:
            env['REFVSR_NO_FAST_POINTWISE'] = '1'
        path = str(tmp_path / f'{int(fast)}.npz')
        subprocess.run([sys.executable, os.path.join(HERE, 'x2_kernel_dump.py'), path], check=True, env=env, cwd=tmp_path)
        res[fast] = np.load(path)
    kf, kg = list(res[True]['kernels']), list(res[False]['kernels'])
    for want in ('aligned_sample4_kernel', 'reconstruct2_kernel', 'gather_cells_kernel<4'):
        assert any(want in n for n in kf), (want, kf)
        assert not any(want in n for n in kg), (want, kg)
    keys = [k for k in res[True].files if k != 'kernels']
    assert sorted(keys) == sorted(k for k in res[False].files if k != 'kernels') and len(keys) >= 26
    for key in keys:
        assert np.array_equal(res[True][key], res[False][key]), f'{key}: fast path differs from the generic kernel'
    # fp32 outputs against the CPU operator definitions
    ops = OracleOps()
    sname, cells, value_hw = SHAPES[0]
    for C in (48, 24):
        value, idx, aff, x = inputs(cells, value_hw, C, torch.float32, seed=C)
        g = torch.empty(4 * cells[0], 4 * cells[1], C)
        ops.gather_blocks(value, idx, cells[0], cells[1], 4, g)
        assert np.array_equal(res[True][f'gather/{sname}/fp32/{C}'], g.numpy())
        a = torch.empty_like(x)
        ops.aligned_sample(x, aff, 4, a)
        # sin / cos and the blend order differ from torch on the CPU (tests/test_gpu_kernels.py uses the same bar)
        assert np.abs(res[True][f'aligned/{sname}/fp32/{C}'] - a.numpy()).max() <= 2e-4
    for h, w in ((136, 240), (37, 53)):
        gen = torch.Generator().manual_seed(h)
        last = 0.3 * (torch.rand(2 * h, 2 * w, 4, generator=gen) - 0.5)
        lr = torch.rand(3, h, w, generator=gen)
        for clamp in (True, False):
            o = torch.empty(3, 2 * h, 2 * w)
            ops.reconstruct(last, lr, 2, clamp, o)
            assert np.abs(res[True][f'reconstruct/{h}x{w}/{int(clamp)}'] - o.numpy()).max() <= 1e-5
