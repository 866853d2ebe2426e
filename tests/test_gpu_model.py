"""-m gpu: the whole hot path through SRNet.forward on the GPU against the golden vectors produced by the
unmodified reference (tests/golden/make_golden.py) and against the oracle at a larger size.

Bars (north_star): fp32 path <= 1e-3 relative; 16-bit paths are judged by PSNR against the reference output
(the hard argmax makes per-pixel bounds meaningless where an index flips; the flip rate is reported and
bounded separately)."""
import numpy as np
import pytest
import torch

from util import CASES, build_case, psnr

pytestmark = pytest.mark.gpu


def run_clip(net, lrs, refs, T, device='cuda'):
    from refvsr_b200.synth import sliding_windows
    outs = []
    for k, wl, wr, first in sliding_windows(lrs, refs, T):
        outs.append(net(wl.to(device), wr.to(device), first, False, False)['result'][0].float().cpu())
    return outs


@pytest.mark.parametrize('name', list(CASES))
def test_fp32_path_matches_reference_golden(name):
    spec, cfg, net, lrs, refs, golden = build_case(name, 'cuda', b200_precision='fp32')
    outs = run_clip(net, lrs, refs, spec['T'])
    for k, o in enumerate(outs):
        g = torch.from_numpy(golden[f'result_{k}'])
        p = psnr(o, g)
        err = (o - g).abs().max().item()
        print(f'{name} window {k}: psnr {p:.1f} dB, max abs {err:.2e}')
        assert p >= 80.0, f'{name} window {k}: PSNR vs reference {p:.1f} dB'
        assert err <= 5e-3


@pytest.mark.parametrize('name', list(CASES))
def test_first_window_products_match_reference_golden(name):
    """flows / confidence / index maps of the FIRST window against the reference's own hooked outputs (make_golden.py:
    flows_0 = fw j = 0..T-2 then bw for j = T-1..1; conf_0 / idx_0 per window frame) - fp32 path, so an index may only
    differ on an exact score tie."""
    from refvsr_b200.synth import sliding_windows
    spec, cfg, net, lrs, refs, golden = build_case(name, 'cuda', b200_precision='fp32')
    T, h, w = spec['T'], spec['h'], spec['w']
    k, wl, wr, first = next(iter(sliding_windows(lrs, refs, T)))
    net(wl.cuda(), wr.cuda(), True, False, False)
    N = net.Network
    mid = T // 2
    gradio = False
    if not gradio:
        for j in range(0, mid + 1):                      # consumed forward flows (RefVSR.py:182-184)
            if mid == T - 1 and j == mid:
                continue
            f = N._ring('fw', j, T, (h, w, 2)).cpu()
            g = torch.from_numpy(golden['flows_0'][j]).permute(1, 2, 0)
            assert (f - g).abs().max() <= 2e-3, f'forward flow {j}: {(f - g).abs().max():.2e} px'
        for j in range(mid, T - 1):                      # backward flows: hook order j = T-1..1 -> index j-1 (RefVSR.py:187-189)
            f = N._ring('bw', j, T, (h, w, 2)).cpu()
            g = torch.from_numpy(golden['flows_0'][T - 1 + (T - 2 - j)]).permute(1, 2, 0)
            assert (f - g).abs().max() <= 2e-3, f'backward flow {j}: {(f - g).abs().max():.2e} px'
    flips = []
    for i in range(T):
        slot = N._frame_slot(i % T, h, w)
        gi, gc = golden['idx_0'][i], golden['conf_0'][i, 0]
        idx = slot['idx'].cpu().numpy()
        conf = slot['conf'].cpu().numpy()
        same = idx == gi.reshape(-1)
        flips.append(1.0 - same.mean())
        assert np.abs(conf - gc).max() <= 2e-3, f'frame {i}: conf {np.abs(conf - gc).max():.2e}'
    print(f'{name}: index flip rate vs reference {np.mean(flips):.4%}')
    assert np.mean(flips) <= 2e-3


@pytest.mark.parametrize('name', list(CASES))
@pytest.mark.parametrize('prec,bar', [('fp16', 55.0), ('bf16', 42.0)])
def test_16bit_tensor_core_path(name, prec, bar):
    spec, cfg, net, lrs, refs, golden = build_case(name, 'cuda', b200_precision=prec)
    outs = run_clip(net, lrs, refs, spec['T'])
    for k, o in enumerate(outs):
        g = torch.from_numpy(golden[f'result_{k}'])
        p = psnr(o, g)
        print(f'{name}/{prec} window {k}: psnr {p:.1f} dB, max abs {(o - g).abs().max().item():.2e}')
        assert p >= bar, f'{name}/{prec} window {k}: PSNR vs reference {p:.1f} dB < {bar}'


def test_tensor_core_and_simt_paths_agree():
    name = 'mfid_t5_40x56_ref2x'
    res = {}
    for tc in (True, False):
        spec, cfg, net, lrs, refs, golden = build_case(name, 'cuda', b200_precision='fp16', b200_tensor_cores=tc)
        res[tc] = run_clip(net, lrs, refs, spec['T'])
    for a, b in zip(res[True], res[False]):
        assert psnr(a, b) >= 55.0


def test_fused_resblock_path_matches_unfused():
    """config.b200_fuse_resblocks=True routes every ResidualBlockNoBN / ResBlock through rv_resblock"""
    name = 'mfid_t5_40x56_ref2x'
    res = {}
    for fuse in (True, False):
        spec, cfg, net, lrs, refs, golden = build_case(name, 'cuda', b200_precision='fp16', b200_fuse_resblocks=fuse)
        res[fuse] = run_clip(net, lrs, refs, spec['T'])
    for k, (a, b) in enumerate(zip(res[True], res[False])):
        g = torch.from_numpy(golden[f'result_{k}'])
        print(f'fused window {k}: psnr vs unfused {psnr(a, b):.1f} dB, vs reference {psnr(a, g):.1f} dB')
        assert psnr(a, b) >= 60.0 and psnr(a, g) >= 55.0


def test_reuse_is_exact():
    """sliding-window reuse (flows / matches / ref features) must not change a single bit."""
    name = 'small_t7_24x32'
    res = {}
    for reuse in (True, False):
        spec, cfg, net, lrs, refs, golden = build_case(name, 'cuda', b200_precision='fp16', b200_reuse=reuse)
        res[reuse] = run_clip(net, lrs, refs, spec['T'])
    for a, b in zip(res[True], res[False]):
        assert torch.equal(a, b)


def test_cuda_graphs_are_exact():
    """whole-window CUDA graphs (one launch per window after first occurrence) vs eager launches: bit identical,
    across steady windows, ring wrap-around and forced resets (reset_branch)."""
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip, sliding_windows
    lrs, refs = make_clip(24, 24, 32, 1, seed=7)
    res = {}
    for graphs in (True, False):
        cfg = get_config('RefVSR_small_MFID', device='cuda', num_blocks=2, b200_precision='fp16', b200_cuda_graphs=graphs)
        net = SRNet(cfg).eval()
        seeded_test_weights(net, seed=7)
        net = net.cuda()
        res[graphs] = [net(wl.cuda(), wr.cuda(), first, False, False)['result'].cpu()
                       for k, wl, wr, first in sliding_windows(lrs, refs, 7)]
        if graphs:
            assert len(net.Network._graphs) >= 8, 'graphs must actually have been captured'
    for k, (a, b) in enumerate(zip(res[True], res[False])):
        assert torch.equal(a, b), f'window {k}: graph replay differs from eager'


def test_branch_overlap_is_exact():
    """forward step of a steady window on a second stream + capped conv grids (network.py, rv_set_conv_cta_cap) vs the sequential
    schedule: bit identical, with CUDA graphs and eagerly, across steady windows, ring wrap-around and forced resets."""
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip, sliding_windows
    lrs, refs = make_clip(24, 40, 56, 1, seed=9)
    res = {}
    for overlap, graphs in ((False, True), (True, True), (True, False)):
        cfg = get_config('RefVSR_MFID', device='cuda', num_blocks=3, b200_precision='bf16', b200_cuda_graphs=graphs,
                         b200_overlap_branches=overlap, b200_overlap_cap=70)
        net = SRNet(cfg).eval()
        seeded_test_weights(net, seed=9)
        net = net.cuda()
        assert net.Network.overlap_branches == overlap
        res[(overlap, graphs)] = [net(wl.cuda(), wr.cuda(), first, False, False)['result'].cpu()
                                  for k, wl, wr, first in sliding_windows(lrs, refs, 7)]
        assert net.Network.ops.set_conv_cta_cap(0) == 0, 'the grid cap must be back to 0 after every window'
    for key in ((True, True), (True, False)):
        for k, (a, b) in enumerate(zip(res[key], res[(False, True)])):
            assert torch.equal(a, b), f'window {k}: overlapped schedule {key} differs from the sequential one'


def test_push_frame_equals_forward_on_gpu():
    """streaming entry (one entering frame per call, no reuse-guard launch) vs forward() on the sliding windows: bit identical with
    CUDA graphs, stream overlap, ring wrap-around and forced resets."""
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip, sliding_windows
    lrs, refs = make_clip(22, 40, 56, 1, seed=11)
    wins = list(sliding_windows(lrs, refs, 7))
    outs = {}
    for mode in ('forward', 'push'):
        cfg = get_config('RefVSR_MFID', device='cuda', num_blocks=2, b200_precision='bf16')
        net = SRNet(cfg).eval()
        seeded_test_weights(net, seed=11)
        net = net.cuda()
        res = []
        for k, wl, wr, first in wins:
            if mode == 'forward' or k == 0:
                res.append(net(wl.cuda(), wr.cuda(), first, False, False)['result'][0].cpu())
            else:
                res.append(net.push_frame(wl[0, -1].cuda(), wr[0, -1].cuda()).cpu())
        outs[mode] = res
        if mode == 'push':
            assert net.Network.reuse_fallbacks == 0
    for k, (a, b) in enumerate(zip(outs['push'], outs['forward'])):
        assert torch.equal(a, b), f'window {k}: push_frame differs from forward()'


def test_medium_size_against_oracle():
    """96x128 LR, RefVSR_small_MFID with all 24 blocks, 3 windows: CUDA fp32 path vs the CPU oracle."""
    from oracle.refvsr_oracle import OracleRefVSR
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip, sliding_windows
    cfg = get_config('RefVSR_small_MFID', device='cuda', b200_precision='fp32')
    net = SRNet(cfg).eval()
    seeded_test_weights(net, seed=21)
    orc = OracleRefVSR(cfg, net.state_dict())
    net = net.cuda()
    lrs, refs = make_clip(3, 96, 128, 1, seed=21)
    for k, wl, wr, first in sliding_windows(lrs, refs, 7):
        o = net(wl.cuda(), wr.cuda(), first, False, False)['result'].float().cpu()
        e = orc.forward(wl, wr, first)
        p = psnr(o, e)
        print(f'96x128 window {k}: psnr {p:.1f} dB max abs {(o - e).abs().max().item():.2e}')
        assert p >= 75.0


def test_full_size_properties():
    """BASELINE size (270x480 -> 1080x1920), MFID, bf16: shape, range, determinism, state handling."""
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip, sliding_windows
    cfg = get_config('RefVSR_MFID', device='cuda')
    net = SRNet(cfg).eval()
    seeded_test_weights(net, seed=5)
    net = net.cuda()
    lrs, refs = make_clip(3, 270, 480, 1, seed=5)
    outs = []
    for rep in range(2):
        cur = []
        for k, wl, wr, first in sliding_windows(lrs, refs, 7):
            o = net(wl.cuda(), wr.cuda(), first, False, False)['result']
            assert o.shape == (1, 3, 1080, 1920) and o.dtype == torch.float32
            assert float(o.min()) >= 0.0 and float(o.max()) <= 1.0 and torch.isfinite(o).all()
            cur.append(o.cpu())
        outs.append(cur)
    for a, b in zip(*outs):
        assert torch.equal(a, b), 'two passes over the same clip must be bit identical (is_first_frame resets state)'
    with pytest.raises(RuntimeError):
        fresh = SRNet(cfg).eval().cuda()
        wl, wr = lrs[:7].unsqueeze(0).cuda() if lrs.shape[0] >= 7 else lrs[[0] * 7].unsqueeze(0).cuda(), refs[[0] * 7].unsqueeze(0).cuda()
        fresh(wl, wr, False, False, False)      # no propagated state yet: the reference fails here too


def test_reuse_guard_under_cuda_graphs_non_sliding_caller():
    """With CUDA graphs and reuse on, a caller that does NOT slide by one frame (is_first_frame=False) must still get exactly what a
    cache-free, graph-free engine computes for the same calls: the overlap check turns such a call into a full recompute."""
    from refvsr_b200.synth import make_clip, sliding_windows
    name = 'small_t7_24x32'
    spec, cfg, net, _, _, _ = build_case(name, 'cuda', b200_precision='bf16')
    spec, cfg, ref, _, _, _ = build_case(name, 'cuda', b200_precision='bf16', b200_reuse=False, b200_cuda_graphs=False)
    lrs, refs = make_clip(16, spec['h'], spec['w'], 1, seed=3)
    wins = list(sliding_windows(lrs, refs, spec['T']))
    order = list(range(0, 9)) + [11, 12, 13, 5, 6, 7, 8, 9]       # slides (graphs get captured), a jump forward, slides, a jump back
    for n, k in enumerate(order):
        _, wl, wr, _ = wins[k]
        a = net(wl.cuda(), wr.cuda(), n == 0, False, False)['result']
        b = ref(wl.cuda(), wr.cuda(), n == 0, False, False)['result']
        assert torch.equal(a, b), f'call {n} (window {k}): {(a - b).abs().max().item():.3e}'
    assert net.Network.reuse_fallbacks == 2 and len(net.Network._graphs) > 0
