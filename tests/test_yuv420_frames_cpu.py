"""YUV 4:2:0 frames on the CPU.  The restatement of OpenCV's conversions (tests/yuv_ops.py) against cv2 itself, over every RGB
triple and every (Y, U, V) triple; and the engine's 4:2:0 entries (Network.forward_yuv420 / push_frame_yuv420 /
push_frames_yuv420) through the test double, whose frames must be exactly cvtColor(forward_u8(cvtColor(frames))), with fp32,
8-bit and 4:2:0 calls sharing one stream."""
import numpy as np
import pytest
import torch

from u8_ops import hwc_u8, planar_f32
from util import build_case
from x2_util import build_x2_case
from yuv_ops import YuvOracleOps, rgb_to_yuv420, yuv420_to_rgb

CASES = [('small_t3_32x48', build_case),            # x4, reset_branch = 2 (forced resets)
         ('x2_small_l1_t3_32x48', build_x2_case),   # x2, reset_branch = 2
         ('small8k_t3_32x48', build_case)]          # flag_HD_in, reset_branch = 2


def _cube_chunk(k):
    """the RGB triples k * 2^20 .. (k + 1) * 2^20 - 1 as (1024, 1024, 3) uint8"""
    i = np.arange(k << 20, (k + 1) << 20, dtype=np.uint32)
    return np.stack([i >> 16, (i >> 8) & 255, i & 255], -1).astype(np.uint8).reshape(1024, 1024, 3)


def test_rgb_to_i420_is_cv2_over_the_rgb_cube():
    """Y of every pixel and U, V of each block's top-left pixel, for all 2^24 RGB triples in each position of a 2 x 2 block"""
    cv2 = pytest.importorskip('cv2')
    for k in range(16):
        a = _cube_chunk(k)
        img = np.empty((2048, 2048, 3), np.uint8)
        img[0::2, 0::2], img[0::2, 1::2] = a, np.roll(a, 1, 0)               # the other three pixels of a block differ from the
        img[1::2, 0::2], img[1::2, 1::2] = np.roll(a, 1, 1), a[::-1, ::-1]   # top-left one, so an averaged chroma would show
        want = cv2.cvtColor(img, cv2.COLOR_RGB2YUV_I420)
        got = rgb_to_yuv420(img)
        assert np.array_equal(got, want), f'chunk {k}: {int((got != want).sum())} bytes differ'
        nv = rgb_to_yuv420(img, nv12=True)
        assert np.array_equal(nv[:2048], want[:2048])
        assert np.array_equal(nv[2048:, 0::2].ravel(), want[2048:2560].ravel())       # U, V interleaved
        assert np.array_equal(nv[2048:, 1::2].ravel(), want[2560:].ravel())


@pytest.mark.parametrize('nv12', [False, True], ids=['i420', 'nv12'])
def test_yuv420_to_rgb_is_cv2_over_all_triples(nv12):
    """all 2^24 (Y, U, V) triples: 4 frames of 2048 x 2048, each (U, V) pair shared by the 4 pixels of 64 blocks holding every Y"""
    cv2 = pytest.importorskip('cv2')
    code = cv2.COLOR_YUV2RGB_NV12 if nv12 else cv2.COLOR_YUV2RGB_I420
    blk = np.arange(1024 * 1024, dtype=np.uint32).reshape(1024, 1024)
    for k in range(4):
        pair = (k << 14) + (blk >> 6)                                        # 2^14 (U, V) pairs per frame
        yq = (blk & 63) * 4                                                  # the block's first Y; its 4 pixels hold yq .. yq + 3
        y = np.empty((2048, 2048), np.uint8)
        y[0::2, 0::2], y[0::2, 1::2], y[1::2, 0::2], y[1::2, 1::2] = yq, yq + 1, yq + 2, yq + 3
        u, v = (pair >> 8).astype(np.uint8), (pair & 255).astype(np.uint8)
        if nv12:
            c = np.stack([u, v], -1).reshape(1024, 2048)
        else:
            c = np.concatenate([u.ravel(), v.ravel()]).reshape(1024, 2048)
        frame = np.ascontiguousarray(np.concatenate([y, c], 0))
        want = cv2.cvtColor(frame, code)
        got = yuv420_to_rgb(frame, nv12)
        assert np.array_equal(got, want), f'frame {k}: {int((got != want).sum())} bytes differ'


def yuv_clip(name, builder, nv12):
    """the fixture's engine (oracle ops with the 4:2:0 formats, fp32) and its clip as 4:2:0 frames"""
    spec, cfg, net, lrs, refs, _ = builder(name, 'cpu', ops=YuvOracleOps(), b200_precision='fp32')
    return spec, net, rgb_to_yuv420(hwc_u8(lrs, False), nv12), rgb_to_yuv420(hwc_u8(refs, False), nv12)


def windows(lrs, refs, t):
    n = lrs.shape[0]
    for k in range(n):
        idx = [min(max(k - t // 2 + j, 0), n - 1) for j in range(t)]
        yield k, lrs[idx].unsqueeze(0), refs[idx].unsqueeze(0), k == 0


def rgb(x, nv12):
    return yuv420_to_rgb(x, nv12).contiguous()


@pytest.mark.parametrize('nv12', [False, True], ids=['i420', 'nv12'])
@pytest.mark.parametrize('name,builder', CASES, ids=[c[0] for c in CASES])
def test_yuv420_entries_are_cvtcolor_of_forward_u8(name, builder, nv12):
    """forward_yuv420 on sliding windows, push_frame_yuv420 and push_frames_yuv420 on the entering frames: each output is
    cvtColor(forward_u8(cvtColor(window)), RGB2YUV_I420), through steady windows, ring wrap-around and forced resets"""
    spec, net_u8, lrs, refs = yuv_clip(name, builder, nv12)
    _, net_f, _, _ = yuv_clip(name, builder, nv12)
    _, net_p, _, _ = yuv_clip(name, builder, nv12)
    _, net_ps, _, _ = yuv_clip(name, builder, nv12)
    t, s, h, w = spec['T'], net_u8.Network.scale, spec['h'], spec['w']
    nwin = 0
    for k, wl, wr, first in windows(lrs, refs, t):
        want = rgb_to_yuv420(net_u8.Network.forward_u8(rgb(wl, nv12), rgb(wr, nv12), first), nv12)
        got = net_f.Network.forward_yuv420(wl, wr, first, nv12=nv12)
        assert got.dtype == torch.uint8 and tuple(got.shape) == (1, 3 * s * h // 2, s * w)
        assert torch.equal(got, want), f'{name} window {k}: forward_yuv420'
        if first:
            p = net_p.forward_yuv420(wl, wr, True, nv12=nv12)[0]
            ps = net_ps.forward_yuv420(wl, wr, True, nv12=nv12)
        else:
            p = net_p.push_frame_yuv420(wl[0, -1], wr[0, -1], nv12=nv12)
            ps = net_ps.push_frames_yuv420(wl[:, -1].contiguous(), wr[:, -1].contiguous(), nv12=nv12)
        assert torch.equal(p, want[0]), f'{name} window {k}: push_frame_yuv420'
        assert tuple(ps.shape) == tuple(want.shape) and torch.equal(ps, want), f'{name} window {k}: push_frames_yuv420'
        nwin += 1
    assert nwin >= 4 and net_u8.Network.max_frame_itr_num == 2
    assert net_f.Network.frame_itr_num == net_p.Network.frame_itr_num == net_u8.Network.frame_itr_num
    assert net_f.Network.reuse_fallbacks == 0          # the 4:2:0 reuse guard sees the windows slide


def test_yuv420_u8_and_fp32_calls_interleave():
    """4:2:0, 8-bit and fp32 calls in turn on one clip (forward and push) give what each kind gives alone"""
    spec, net_u, lrs, refs = yuv_clip('small_t3_32x48', build_case, False)
    _, net_mix, _, _ = yuv_clip('small_t3_32x48', build_case, False)
    _, net_push, _, _ = yuv_clip('small_t3_32x48', build_case, False)
    wins = list(windows(lrs, refs, spec['T']))
    for k, wl, wr, first in wins:
        rl, rr = rgb(wl, False), rgb(wr, False)
        alone = net_u.Network.forward_u8(rl, rr, first)
        kind = k % 3
        if kind == 0:
            got = net_mix.Network.forward_yuv420(wl, wr, first)
            assert torch.equal(got, rgb_to_yuv420(alone)), f'window {k}: 4:2:0 call'
        elif kind == 1:
            assert torch.equal(net_mix.Network.forward_u8(rl, rr, first), alone), f'window {k}: 8-bit call'
        else:
            got = net_mix(planar_f32(rl, False), planar_f32(rr, False), first)['result']
            assert torch.equal(hwc_u8(got, False), alone), f'window {k}: fp32 call'
        if first:
            net_push.Network.forward_u8(rl, rr, True)
        elif kind == 0:
            assert torch.equal(net_push.Network.push_frame_yuv420(wl[0, -1], wr[0, -1]), rgb_to_yuv420(alone[0]))
        elif kind == 1:
            assert torch.equal(net_push.Network.push_frame_u8(rl[0, -1], rr[0, -1]), alone[0])
        else:
            got = net_push.Network.push_frame(planar_f32(rl[0, -1], False), planar_f32(rr[0, -1], False))
            assert torch.equal(hwc_u8(got, False), alone[0])
    assert net_mix.Network.reuse_fallbacks == 0


def test_yuv420_entries_refuse_bad_input():
    spec, net, lrs, refs = yuv_clip('small_t3_32x48', build_case, False)
    N = net.Network
    k, wl, wr, first = next(windows(lrs, refs, spec['T']))
    bad = {
        'dtype': (wl.float(), wr),
        'device': (torch.empty(wl.shape, dtype=torch.uint8, device='meta'), wr),
        'contiguous': (wl.transpose(2, 3).contiguous().transpose(2, 3), wr),
        'rows not a multiple of 3': (wl[:, :, :-1].contiguous(), wr),
        'odd w': (wl[..., :-1].contiguous(), wr),
        'HWC frames': (hwc_u8(torch.zeros(1, 3, 3, 32, 48), False), wr),
        'n_t': (wl, wr[:, :2].contiguous()),
        'not a tensor': (wl.numpy(), wr),
    }
    for why, (a, b) in bad.items():
        with pytest.raises(ValueError):
            N.forward_yuv420(a, b, True)
        assert N._u8 is None, why
    _, hd, _, _ = yuv_clip('small8k_t3_32x48', build_case, False)                   # a size forward() refuses: flag_HD_in
    with pytest.raises(ValueError, match='flag_HD_in'):                              # takes LR sizes in multiples of 4 only
        hd.Network.forward_yuv420(rgb_to_yuv420(torch.zeros(1, 3, 30, 48, 3, dtype=torch.uint8)), wr, True)
    assert hd.Network._u8 is None
    with pytest.raises(RuntimeError, match='previous forward'):                      # not a bad input: no stream yet
        N.push_frame_yuv420(wl[0, -1], wr[0, -1])
    N.forward_yuv420(wl, wr, True)
    lr, ref = wl[0, -1], wr[0, -1]
    smaller = rgb_to_yuv420(torch.zeros(28, 48, 3, dtype=torch.uint8))
    for why, (a, b) in {'dtype': (lr.float(), ref), 'dims': (lr[None], ref),
                        'contiguous': (lr.t().contiguous().t(), ref), 'rows': (lr[:-1].contiguous(), ref),
                        'odd w': (lr[:, :-1].contiguous(), ref),
                        'device': (torch.empty(lr.shape, dtype=torch.uint8, device='meta'), ref),
                        'stream size': (smaller, ref), 'ref dtype': (lr, ref.double())}.items():
        with pytest.raises(ValueError):
            N.push_frame_yuv420(a, b)
        assert N._u8 is None, why
    with pytest.raises(ValueError):
        N.push_frames_yuv420(lr, ref)                                                # (3h/2, w): no batch dimension
    with pytest.raises(ValueError):
        N.push_frames_yuv420(torch.stack([lr, lr]), torch.stack([ref, ref]))         # 2 frames for a stream of 1
    with pytest.raises(ValueError):
        N.push_frames_yuv420(smaller[None], ref[None])
    # the stream is intact after the refusals
    k2, wl2, wr2, _ = list(windows(lrs, refs, spec['T']))[1]
    _, ref_net, _, _ = yuv_clip('small_t3_32x48', build_case, False)
    ref_net.Network.forward_yuv420(wl, wr, True)
    assert torch.equal(N.push_frame_yuv420(wl2[0, -1], wr2[0, -1]), ref_net.Network.forward_yuv420(wl2, wr2, False)[0])
