"""The x2 models (scale=2, matching_ksize=4) on CPU: parameter schema, the oracle and the engine's schedule (through the OracleOps
test double) against golden vectors of the unmodified reference (tests/golden/make_golden_x2.py), the refused combinations and
input sizes, and the frame-sharded clip.  No CUDA needed."""
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from util import GOLDEN_DIR, psnr
from x2_util import X2, X2_CASES, X2_CONFIGS, OracleRefVSRx2, build_x2_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_x2_state_dict_schema_matches_reference():
    """keys and shapes of the four x2 configs, dumped from the reference (no upsample2; aa1.align.* and map128 present)"""
    from refvsr_b200 import SRNet, get_config
    with open(os.path.join(GOLDEN_DIR, 'state_dict_keys_x2.json')) as f:
        ref_keys = json.load(f)
    assert sorted(ref_keys) == sorted(X2_CONFIGS)
    for name in X2_CONFIGS:
        sd = SRNet(get_config(name, device='cpu', **X2)).state_dict()
        assert {k: list(v.shape) for k, v in sd.items()} == ref_keys[name], name
        assert not any('upsample2' in k for k in sd)
        assert any(k.startswith('Network.aa1.align.') for k in sd) and any('map128' in k for k in sd)


@pytest.mark.parametrize('name', list(X2_CASES))
def test_x2_oracle_matches_reference_golden(name):
    from refvsr_b200.synth import sliding_windows
    spec, cfg, net, lrs, refs, golden = build_x2_case(name, 'cpu')
    orc = OracleRefVSRx2(cfg, net.state_dict())
    T, h, w = spec['T'], spec['h'], spec['w']
    for k, wl, wr, first in sliding_windows(lrs, refs, T):
        orc.trace = {} if k == 0 else None
        out = orc.forward(wl, wr, first)
        assert out.shape == (1, 3, 2 * h, 2 * w)
        err = np.abs(out[0].numpy() - golden[f'result_{k}']).max()
        assert err < 5e-6, f'{name} window {k}: oracle differs from the reference by {err:.2e}'
        if k == 0:
            fl = golden['flows_0']            # reference call order: forward j=0..T-2, then backward j=T-1..1
            for j, f in orc.trace['fw'].items():
                assert np.abs(f[0].numpy() - fl[j]).max() < 1e-4
            for j, f in orc.trace['bw'].items():
                assert np.abs(f[0].numpy() - fl[(T - 1) + (T - 2 - j)]).max() < 1e-4
            assert golden['idx_0'].shape == (T, (h // 2) * (w // 2))
            for i, c in orc.trace['conf'].items():
                assert np.abs(c[0].numpy() - golden['conf_0'][i]).max() < 1e-5
                assert (orc.trace['idx'][i][0].numpy() != golden['idx_0'][i]).mean() == 0.0


@pytest.mark.parametrize('name', list(X2_CASES))
def test_x2_schedule_matches_reference_golden(name, oracle_ops):
    from refvsr_b200.synth import sliding_windows
    spec, cfg, net, lrs, refs, golden = build_x2_case(name, 'cpu', ops=oracle_ops, b200_precision='fp32')
    T, h, w = spec['T'], spec['h'], spec['w']
    for k, wl, wr, first in sliding_windows(lrs, refs, T):
        o = net(wl, wr, first, False, False)['result']
        assert o.shape == (1, 3, 2 * h, 2 * w) and o.dtype == torch.float32
        g = torch.from_numpy(golden[f'result_{k}'])
        # an exact score tie may flip one argmax (fp16-split product vs fp32 bmm): PSNR bar + loose max
        assert psnr(o[0], g) > 95.0 and (o[0] - g).abs().max() < 2e-3, f'{name} window {k}'
        if k == 0:
            N = net.Network
            mism = np.mean([(N._frame_slot(i % T, h, w)['idx'].numpy() != golden['idx_0'][i]).mean() for i in range(T)])
            assert mism <= 1e-3


def test_x2_push_frame_equals_forward(oracle_ops):
    from refvsr_b200.synth import sliding_windows
    name = 'x2_small_l1_t3_32x48'
    spec, cfg, net, lrs, refs, golden = build_x2_case(name, 'cpu', ops=oracle_ops, b200_precision='fp32')
    wins = list(sliding_windows(lrs, refs, spec['T']))
    want = [net(wl, wr, first)['result'][0].clone() for k, wl, wr, first in wins]
    spec, cfg, net2, lrs, refs, golden = build_x2_case(name, 'cpu', ops=oracle_ops, b200_precision='fp32')
    got = [net2(wins[0][1], wins[0][2], True)['result'][0].clone()]
    got += [net2.push_frame(wl[0, -1], wr[0, -1]).clone() for k, wl, wr, first in wins[1:]]
    for k, (a, b) in enumerate(zip(got, want)):
        assert a.shape == (3, 2 * spec['h'], 2 * spec['w']) and torch.equal(a, b), f'window {k}'


def test_x2_refused_combinations_and_sizes(oracle_ops):
    from refvsr_b200 import SRNet, get_config
    # the reference itself cannot compute these (F.fold size mismatch / gather out of range, attention.py:143-144)
    with pytest.raises(NotImplementedError, match='matching_ksize=4'):
        SRNet(get_config('config_RefVSR_MFID', device='cpu', scale=2, matching_ksize=2))
    with pytest.raises(NotImplementedError, match='flag_HD_in'):
        SRNet(get_config('config_RefVSR_MFID_8K', device='cpu', scale=2, matching_ksize=8))
    with pytest.raises(NotImplementedError, match='flag_HD_in'):
        SRNet(get_config('config_RefVSR_MFID', device='cpu', scale=2, matching_ksize=4, flag_HD_in=True))
    with pytest.raises(NotImplementedError):
        SRNet(get_config('config_RefVSR_MFID', device='cpu', scale=3))
    spec, cfg, net, lrs, refs, golden = build_x2_case('x2_small_l1_t3_32x48', 'cpu', ops=oracle_ops, b200_precision='fp32')
    for lr_hw, ref_hw in (((31, 48), (32, 48)), ((32, 47), (32, 48)), ((32, 48), (30, 48)), ((32, 48), (32, 46))):
        x, r = torch.rand(1, 3, 3, *lr_hw), torch.rand(1, 3, 3, *ref_hw)
        with pytest.raises(ValueError, match='scale=2'):
            net(x, r, True)


def _frame_worker(rank, world, port, q, name, reset_branch, nframes):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    torch.set_num_threads(2)
    from oracle.oracle_ops import OracleOps
    from refvsr_b200.dist import exchange_halo, gather_frames, plan_frames, run_clip_frame_sharded
    from refvsr_b200.synth import make_clip
    from x2_util import build_x2_case
    spec, cfg, net, _, _, _ = build_x2_case(name, 'cpu', ops=OracleOps(), b200_precision='fp32', reset_branch=reset_branch)
    lrs, refs = make_clip(nframes, spec['h'], spec['w'], 1, seed=32)
    T = spec['T']
    plan = plan_frames(nframes, world)
    f0, f1 = plan[rank]
    fl, first = exchange_halo(lrs[f0:f1].clone(), plan, rank, T // 2)
    fr, _ = exchange_halo(refs[f0:f1].clone(), plan, rank, T // 2)
    res = run_clip_frame_sharded(net, fl, fr, first, plan, rank)
    allf = gather_frames(res, plan, rank, (3, 2 * spec['h'], 2 * spec['w']), 'cpu')
    if rank == 0:
        q.put([f.numpy() for f in allf])
    dist.barrier()
    dist.destroy_process_group()


def test_x2_frame_sharded_clip_equals_single_stream():
    from oracle.oracle_ops import OracleOps
    from refvsr_b200.synth import make_clip, sliding_windows
    name, world, reset_branch, nframes = 'x2_small_mfid_t7_24x32', 2, 4, 7
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 35500 + os.getpid() % 2000
    procs = [ctx.Process(target=_frame_worker, args=(r, world, port, q, name, reset_branch, nframes)) for r in range(world)]
    for p in procs:
        p.start()
    sharded = q.get(timeout=900)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    spec, cfg, net, _, _, _ = build_x2_case(name, 'cpu', ops=OracleOps(), b200_precision='fp32', reset_branch=reset_branch)
    lrs, refs = make_clip(nframes, spec['h'], spec['w'], 1, seed=32)
    nthr = torch.get_num_threads()
    torch.set_num_threads(2)          # same as the workers: oneDNN's summation order depends on the thread count
    try:
        single = [net(wl, wr, first)['result'][0].numpy() for k, wl, wr, first in sliding_windows(lrs, refs, spec['T'])]
    finally:
        torch.set_num_threads(nthr)
    assert len(sharded) == len(single) == nframes
    for k, (a, b) in enumerate(zip(sharded, single)):
        assert a.shape == (3, 2 * spec['h'], 2 * spec['w'])
        assert np.array_equal(a, b), f'frame {k}: frame-sharded output must be bit identical to the single stream'
