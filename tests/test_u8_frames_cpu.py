"""The 8-bit streaming entries (Network.forward_u8 / push_frame_u8 / push_frames_u8) on the CPU: the engine's schedule through
the oracle's test double with the 8-bit operators (tests/u8_ops.py).  Their bytes must be frame_u8 of what the fp32 entries
return for u8 / 255, in both channel orders, with the fp32 and 8-bit calls sharing one stream."""
import numpy as np
import pytest
import torch

from u8_ops import U8OracleOps, frame_u8, hwc_u8, planar_f32
from util import build_case
from x2_util import build_x2_case

CASES = [('small_t3_32x48', build_case),            # x4, reset_branch = 2 (forced resets)
         ('x2_small_l1_t3_32x48', build_x2_case),   # x2, reset_branch = 2
         ('small8k_t3_32x48', build_case)]          # flag_HD_in, reset_branch = 2


def u8_clip(name, builder):
    """the fixture's engine (oracle ops, fp32) and its clip as uint8 HWC RGB frames"""
    spec, cfg, net, lrs, refs, _ = builder(name, 'cpu', ops=U8OracleOps(), b200_precision='fp32')
    return spec, net, hwc_u8(lrs, False), hwc_u8(refs, False)


def windows(lrs, refs, t):
    """(k, lr window, ref window, first) of data_loader/datasets.py's clamped sliding windows, n = 1"""
    n = lrs.shape[0]
    for k in range(n):
        idx = [min(max(k - t // 2 + j, 0), n - 1) for j in range(t)]
        yield k, lrs[idx].unsqueeze(0), refs[idx].unsqueeze(0), k == 0


def bgr(x):
    return x.flip(-1).contiguous()


def test_byte_conversion_is_read_frames():
    """fl32(u / 255) in float32 equals data_loader/utils.py::read_frame's float64 np.array(frame) / 255. cast to float32"""
    u = torch.arange(256, dtype=torch.uint8)
    f64 = (u.numpy().astype(np.float64) / 255.).astype(np.float32)
    assert np.array_equal(planar_f32(u.view(256, 1, 1).expand(256, 1, 3).contiguous(), False)[0, :, 0].numpy(), f64)
    assert torch.equal(frame_u8(torch.from_numpy(f64)), u)             # and every byte survives the round trip


@pytest.mark.parametrize('name,builder', CASES, ids=[c[0] for c in CASES])
def test_forward_u8_is_frame_u8_of_forward(name, builder):
    spec, net, lrs, refs = u8_clip(name, builder)
    _, net_rgb, _, _ = u8_clip(name, builder)
    _, net_bgr, _, _ = u8_clip(name, builder)
    t, s = spec['T'], net.Network.scale
    nwin = 0
    for k, wl, wr, first in windows(lrs, refs, t):
        want = net(planar_f32(wl, False), planar_f32(wr, False), first)['result']
        got = net_rgb.Network.forward_u8(wl, wr, first)
        assert got.dtype == torch.uint8 and tuple(got.shape) == (1, s * spec['h'], s * spec['w'], 3)
        assert torch.equal(got, hwc_u8(want, False)), f'{name} window {k}: RGB bytes'
        got_bgr = net_bgr.Network.forward_u8(bgr(wl), bgr(wr), first, bgr=True)
        assert torch.equal(got_bgr, hwc_u8(want, True)), f'{name} window {k}: BGR bytes'
        nwin += 1
    assert nwin >= 4
    assert net_rgb.Network.frame_itr_num == net.Network.frame_itr_num
    assert net_rgb.Network.reuse_fallbacks == 0          # the 8-bit reuse guard sees the windows slide


@pytest.mark.parametrize('name,builder', CASES, ids=[c[0] for c in CASES])
def test_push_frame_u8_equals_sliding_forward_u8(name, builder):
    """one entering frame per call against whole sliding windows: steady windows, ring wrap-around and forced resets"""
    spec, net, lrs, refs = u8_clip(name, builder)
    _, net2, _, _ = u8_clip(name, builder)
    wins = list(windows(lrs, refs, spec['T']))
    want = [net.Network.forward_u8(bgr(wl), bgr(wr), first, bgr=True)[0] for k, wl, wr, first in wins]
    got = [net2.forward_u8(bgr(wins[0][1]), bgr(wins[0][2]), True, bgr=True)[0]]
    got += [net2.push_frame_u8(bgr(wl[0, -1]), bgr(wr[0, -1]), bgr=True) for k, wl, wr, first in wins[1:]]
    assert len(got) >= 4 and net.Network.max_frame_itr_num == 2
    for k, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), f'{name} window {k}: push_frame_u8 differs from forward_u8'
    assert net2.Network.frame_itr_num == net.Network.frame_itr_num


def test_u8_and_fp32_calls_interleave():
    """alternating 8-bit and fp32 calls on one clip (forward and push) give what either kind gives alone"""
    spec, net_f, lrs, refs = u8_clip('small_t3_32x48', build_case)
    _, net_u, _, _ = u8_clip('small_t3_32x48', build_case)
    _, net_mix, _, _ = u8_clip('small_t3_32x48', build_case)
    wins = list(windows(lrs, refs, spec['T']))
    alone = []
    for k, wl, wr, first in wins:
        f = net_f(planar_f32(wl, False), planar_f32(wr, False), first)['result']
        u = net_u.Network.forward_u8(wl, wr, first)
        assert torch.equal(u, hwc_u8(f, False))
        alone.append(u[0])
        if k % 2:
            m = net_mix.Network.forward_u8(wl, wr, first)
            assert torch.equal(m, u), f'window {k}: 8-bit call after fp32 calls'
        else:
            m = net_mix(planar_f32(wl, False), planar_f32(wr, False), first)['result']
            assert torch.equal(m, f), f'window {k}: fp32 call after 8-bit calls'
    assert net_mix.Network.reuse_fallbacks == 0
    # the streaming entries too: push_frame and push_frame_u8 alternate on one stream
    _, net_push, _, _ = u8_clip('small_t3_32x48', build_case)
    net_push(planar_f32(wins[0][1], False), planar_f32(wins[0][2], False), True)
    for k, wl, wr, first in wins[1:]:
        if k % 2:
            got = net_push.Network.push_frame_u8(wl[0, -1], wr[0, -1])
        else:
            got = hwc_u8(net_push.Network.push_frame(planar_f32(wl[0, -1], False), planar_f32(wr[0, -1], False)), False)
        assert torch.equal(got, alone[k]), f'window {k}: interleaved push calls'


def test_push_frames_u8_matches_push_frame_u8():
    """push_frames_u8 with n = 1 is push_frame_u8 (the operator set on the CPU runs n > 1 windows one by one)"""
    spec, net, lrs, refs = u8_clip('small_t3_32x48', build_case)
    _, net2, _, _ = u8_clip('small_t3_32x48', build_case)
    wins = list(windows(lrs, refs, spec['T']))
    net.Network.forward_u8(wins[0][1], wins[0][2], True)
    net2.Network.forward_u8(wins[0][1], wins[0][2], True)
    for k, wl, wr, first in wins[1:]:
        a = net.Network.push_frame_u8(wl[0, -1], wr[0, -1])
        b = net2.Network.push_frames_u8(wl[:, -1].contiguous(), wr[:, -1].contiguous())
        assert tuple(b.shape) == (1,) + tuple(a.shape) and torch.equal(a, b[0]), f'window {k}'


def test_u8_entries_refuse_bad_input():
    spec, net, lrs, refs = u8_clip('small_t3_32x48', build_case)
    N = net.Network
    k, wl, wr, first = next(windows(lrs, refs, spec['T']))
    bad = {
        'dtype': (planar_f32(wl, False), wr),
        'layout': (wl.permute(0, 1, 4, 2, 3).contiguous(), wr),                      # (n, t, 3, h, w) bytes
        'dims': (wl[0], wr),
        'contiguous': (wl.transpose(2, 3), wr),
        'device': (torch.empty(wl.shape, dtype=torch.uint8, device='meta'), wr),
        'n_t': (wl, wr[:, :2].contiguous()),
        'size rule': (wl, wr[:, :, :-1].contiguous()),                               # odd Ref height
        'ref dtype': (wl, wr.float()),
        'not a tensor': (wl.numpy(), wr),
    }
    for why, (a, b) in bad.items():
        with pytest.raises(ValueError):
            N.forward_u8(a, b, True)
        assert N._u8 is None, why
    with pytest.raises(RuntimeError, match='previous forward'):                      # not a bad input: no stream yet
        N.push_frame_u8(wl[0, -1], wr[0, -1])
    N.forward_u8(wl, wr, True)
    lr, ref = wl[0, -1], wr[0, -1]
    for why, (a, b) in {'dtype': (lr.float(), ref), 'layout': (lr.permute(2, 0, 1).contiguous(), ref),
                        'contiguous': (lr.transpose(0, 1), ref), 'device': (torch.empty(lr.shape, dtype=torch.uint8, device='meta'), ref),
                        'stream size': (lr[:-4].contiguous(), ref), 'ref stream size': (lr, ref[:, :-2].contiguous()),
                        'ref dtype': (lr, ref.double())}.items():
        with pytest.raises(ValueError):
            N.push_frame_u8(a, b)
        assert N._u8 is None, why
    with pytest.raises(ValueError):
        N.push_frames_u8(lr, ref)                                                    # (h, w, 3): no batch dimension
    with pytest.raises(ValueError):
        N.push_frames_u8(torch.stack([lr, lr]), torch.stack([ref, ref]))             # 2 frames for a stream of 1
    with pytest.raises(ValueError):
        N.push_frames_u8(lr.unsqueeze(0).float(), ref.unsqueeze(0))
    # the stream is intact after the refusals
    k2, wl2, wr2, _ = list(windows(lrs, refs, spec['T']))[1]
    _, ref_net, _, _ = u8_clip('small_t3_32x48', build_case)
    ref_net.Network.forward_u8(wl, wr, True)
    assert torch.equal(N.push_frame_u8(wl2[0, -1], wr2[0, -1]), ref_net.Network.forward_u8(wl2, wr2, False)[0])
