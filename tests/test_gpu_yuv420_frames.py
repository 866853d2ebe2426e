"""-m gpu: YUV 4:2:0 frames on the H100.  rv_frames_from_u8's I420 / NV12 formats against the restatement of cv2's conversion
(tests/yuv_ops.py) over all (Y, U, V) triples and at every frame alignment; every I420 / NV12 instantiation of
rv_reconstruct_u8{,_batched} against the restatement of the RGB bytes the same call writes; and the engine's forward_yuv420 /
push_frame_yuv420 / push_frames_yuv420 against forward_u8, with fp32, 8-bit and 4:2:0 calls interleaved.  Synthetic clips and
seeded weights only."""
import numpy as np
import pytest
import torch

from u8_ops import hwc_u8, planar_f32
from yuv_ops import FRAME_I420, FRAME_NV12, rgb_to_yuv420, yuv420_to_rgb

pytestmark = pytest.mark.gpu

FMTS = [(FRAME_I420, False), (FRAME_NV12, True)]
FMT_IDS = ['i420', 'nv12']


def _engine(name, seed=7, **over):
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    net = SRNet(get_config(name, device='cuda', b200_precision='bf16', **over)).eval()
    seeded_test_weights(net, seed=seed)
    return net.cuda()


def _windows(lrs, refs, t):
    n = lrs.shape[0]
    for k in range(n):
        idx = [min(max(k - t // 2 + j, 0), n - 1) for j in range(t)]
        yield k, lrs[idx].unsqueeze(0), refs[idx].unsqueeze(0), k == 0


@pytest.mark.parametrize('fmt,nv12', FMTS, ids=FMT_IDS)
def test_frames_from_yuv420_over_all_triples(cuda_ops, fmt, nv12):
    """all 2^24 (Y, U, V) triples in one 4096 x 4096 frame: each (U, V) pair shared by 64 blocks of 4 Y values"""
    blk = np.arange(2048 * 2048, dtype=np.uint32).reshape(2048, 2048)
    pair, yq = blk >> 6, (blk & 63) * 4
    y = np.empty((4096, 4096), np.uint8)
    y[0::2, 0::2], y[0::2, 1::2], y[1::2, 0::2], y[1::2, 1::2] = yq, yq + 1, yq + 2, yq + 3
    u, v = (pair >> 8).astype(np.uint8), (pair & 255).astype(np.uint8)
    c = np.stack([u, v], -1).reshape(2048, 4096) if nv12 else np.concatenate([u.ravel(), v.ravel()]).reshape(2048, 4096)
    frame = torch.from_numpy(np.ascontiguousarray(np.concatenate([y, c], 0)))
    d = torch.empty(3, 4096, 4096, device='cuda')
    cuda_ops.frames_from_u8([frame.cuda()], [d], fmt)
    want = planar_f32(yuv420_to_rgb(frame, nv12), False)
    assert torch.equal(d.cpu(), want)


@pytest.mark.parametrize('h,w', [(2, 2), (6, 10), (32, 48), (34, 46), (270, 480), (136, 242)])
@pytest.mark.parametrize('fmt,nv12', FMTS, ids=FMT_IDS)
def test_frames_from_yuv420_any_alignment(cuda_ops, h, w, fmt, nv12):
    """16 frames in one launch, each source starting at another address mod 16, destinations aligned and not"""
    g = torch.Generator().manual_seed(h * 1000 + w + fmt)
    k, nb = 16, 3 * h * w // 2
    stride = 16 * ((nb + 15) // 16) + 16
    pool = torch.randint(0, 256, (k * stride + 16,), dtype=torch.uint8, generator=g).cuda()
    srcs = [pool[s * stride + s:][:nb].view(3 * h // 2, w) for s in range(k)]
    dpool = torch.full((k * (3 * h * w + 5),), float('nan'), device='cuda')
    dsts = [dpool[s * (3 * h * w + 5) + (s % 5):][:3 * h * w].view(3, h, w) for s in range(k)]
    cuda_ops.frames_from_u8(srcs, dsts, fmt)
    for s, d in zip(srcs, dsts):
        assert torch.equal(d.cpu(), planar_f32(yuv420_to_rgb(s.cpu(), nv12), False)), (h, w, s.data_ptr() % 16, d.data_ptr() % 16)
    assert {s.data_ptr() % 16 for s in srcs} == set(range(16))


def _tail_inputs(n, h, w, s, xc, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(n, s * h, s * w, xc, generator=g) * 1.4 - 0.7)
    x.view(-1, xc)[:64, 0] = torch.tensor([0.5 / 255, 1.5 / 255, 2.5 / 255, -0.0, 1e30, -1e30, float('nan'), 1.0] * 8)
    lr = torch.rand(n, 3, h, w, generator=g)
    return x.to(dtype).cuda(), lr.cuda()


TAIL = [  # (scale, xc, dtype, h, w): fp32 with xc = 4 takes the x4 / x2 fast paths, every other case the generic kernel
    (4, 4, torch.float32, 270, 480), (4, 4, torch.float32, 1080, 1920), (4, 4, torch.float32, 17, 23), (4, 4, torch.float32, 9, 4),
    (2, 4, torch.float32, 540, 960), (2, 4, torch.float32, 17, 21), (2, 4, torch.float32, 6, 8),
    (4, 4, torch.bfloat16, 270, 480), (4, 4, torch.float16, 20, 24), (2, 4, torch.bfloat16, 19, 26),
    (4, 6, torch.float32, 13, 21), (2, 3, torch.float16, 11, 15),
]


@pytest.mark.parametrize('scale,xc,dtype,h,w', TAIL, ids=[f'x{c[0]}-c{c[1]}-{str(c[2])[6:]}-{c[3]}x{c[4]}' for c in TAIL])
def test_reconstruct_yuv420_is_cvtcolor_of_reconstruct_u8(cuda_ops, scale, xc, dtype, h, w):
    """I420 / NV12 output = the restated cv2 RGB2YUV_I420 of the RGB bytes the same call writes, single and batched (n = 2)"""
    H, W = scale * h, scale * w
    big = H * W > 8_000_000
    for n in ((1,) if big else (1, 2)):
        x, lr = _tail_inputs(n, h, w, scale, xc, dtype, seed=h * w + n)
        xa, la = (x, lr) if n > 1 else (x[0], lr[0])
        rgb = torch.empty(n, H, W, 3, dtype=torch.uint8, device='cuda')
        for clamp in ((True,) if big else (True, False)):
            cuda_ops.reconstruct_u8(xa, la, scale, clamp, rgb if n > 1 else rgb[0], False)
            rgb_cpu = rgb.cpu()
            for fmt, nv12 in FMTS:
                out = torch.full((n, 3 * H // 2, W), 7, dtype=torch.uint8, device='cuda')
                cuda_ops.reconstruct_u8(xa, la, scale, clamp, out if n > 1 else out[0], fmt)
                want = rgb_to_yuv420(rgb_cpu, nv12)
                got = out.cpu()
                assert torch.equal(got, want), f'n={n} clamp={clamp} {FMT_IDS[fmt - 2]}: {int((got != want).sum())} bytes differ'
    if big:
        return
    # an unaligned output buffer takes the byte stores, to the same bytes
    x, lr = _tail_inputs(1, h, w, scale, xc, dtype, seed=3)
    rgb = torch.empty(H, W, 3, dtype=torch.uint8, device='cuda')
    cuda_ops.reconstruct_u8(x[0], lr[0], scale, True, rgb, False)
    for fmt, nv12 in FMTS:
        buf = torch.zeros(3 * H * W // 2 + 1, dtype=torch.uint8, device='cuda')
        out = buf[1:].view(3 * H // 2, W)
        cuda_ops.reconstruct_u8(x[0], lr[0], scale, True, out, fmt)
        assert torch.equal(out.cpu(), rgb_to_yuv420(rgb.cpu(), nv12))


def test_yuv420_refuses_bad_arguments(cuda_ops):
    import ctypes as C
    lib = cuda_ops.lib
    x = torch.zeros(16, 16, 4, device='cuda')
    lr = torch.zeros(3, 4, 4, device='cuda')
    o = torch.zeros(24, 16, dtype=torch.uint8, device='cuda')
    assert lib.rv_reconstruct_u8(x.data_ptr(), 4, 0, lr.data_ptr(), 4, 4, 4, 1, 4, o.data_ptr(), None) == -1      # format 4
    assert lib.rv_reconstruct_u8(x.data_ptr(), 4, 0, lr.data_ptr(), 4, 4, 4, 1, -1, o.data_ptr(), None) == -1
    p = (C.c_void_p * 1)(o.data_ptr())
    q = (C.c_void_p * 1)(x.data_ptr())
    assert lib.rv_frames_from_u8(p, q, 1, 4, 4, 4, None) == -1
    assert lib.rv_frames_from_u8(p, q, 1, 3, 4, FRAME_I420, None) == -1                                            # odd h
    assert lib.rv_frames_from_u8(p, q, 1, 4, 5, FRAME_NV12, None) == -1                                            # odd w
    torch.cuda.synchronize()


def _yuv_clip(frames, h, w, seed, nv12):
    from refvsr_b200.synth import make_clip
    lrs, refs = make_clip(frames, h, w, 1, seed=seed)
    return rgb_to_yuv420(hwc_u8(lrs, False), nv12).cuda(), rgb_to_yuv420(hwc_u8(refs, False), nv12).cuda()


def _rgb(x, nv12):
    return yuv420_to_rgb(x.cpu(), nv12).contiguous().cuda()


def _check_clip(name, h, w, frames, t, seed, **over):
    """n = 1: forward_yuv420 / push_frame_yuv420 (I420 and NV12) against forward_u8 on the converted frames; and one engine that
    takes 4:2:0, 8-bit and fp32 calls in turn"""
    for nv12 in (False, True):
        lrs, refs = _yuv_clip(frames, h, w, seed, nv12)
        nu, ny, npush, nmix = (_engine(name, seed=seed, **over) for _ in range(4))
        assert ny.Network.use_graphs and ny.Network.overlap_branches
        for k, wl, wr, first in _windows(lrs, refs, t):
            rl, rr = _rgb(wl, nv12), _rgb(wr, nv12)
            rgb = nu.forward_u8(rl, rr, first)
            want = rgb_to_yuv420(rgb.cpu(), nv12)
            assert torch.equal(ny.forward_yuv420(wl, wr, first, nv12=nv12).cpu(), want), f'{name} window {k}: forward_yuv420'
            got = npush.forward_yuv420(wl, wr, True, nv12=nv12)[0] if first else npush.push_frame_yuv420(wl[0, -1], wr[0, -1], nv12=nv12)
            assert torch.equal(got.cpu(), want[0]), f'{name} window {k}: push_frame_yuv420'
            kind = k % 3
            if kind == 0:
                assert torch.equal(nmix.forward_yuv420(wl, wr, first, nv12=nv12).cpu(), want), f'{name} window {k}: mixed 4:2:0'
            elif kind == 1:
                assert torch.equal(nmix.forward_u8(rl, rr, first), rgb), f'{name} window {k}: mixed 8-bit'
            else:
                res = nmix(planar_f32(rl, False), planar_f32(rr, False), first)['result']
                assert torch.equal(hwc_u8(res, False), rgb), f'{name} window {k}: mixed fp32'
        fmt = FRAME_NV12 if nv12 else FRAME_I420
        for net in (ny, npush, nmix):
            assert net.Network.reuse_fallbacks == 0
        assert any(key[-1] == fmt for key in ny.Network._graphs)                                # graphs captured for 4:2:0
        assert any(key[-1] == fmt for key in npush.Network._graphs)
        assert nu.Network.frame_itr_num == ny.Network.frame_itr_num == npush.Network.frame_itr_num


def test_forward_yuv420_mfid_270x480():
    """RefVSR_MFID at the bench shape with graphs and branch overlap; reset_branch = 4 puts a forced reset inside the clip"""
    _check_clip('RefVSR_MFID', 270, 480, 7, 7, 31, reset_branch=4)


def test_forward_yuv420_x2():
    _check_clip('RefVSR_MFID', 136, 240, 6, 7, 32, num_blocks=4, scale=2, matching_ksize=4, reset_branch=3)


def test_forward_yuv420_flag_hd_in():
    _check_clip('RefVSR_small_MFID_8K', 48, 64, 6, 3, 33, num_blocks=2, reset_branch=2)


@pytest.mark.parametrize('name,h,w,over', [
    ('RefVSR_MFID', 40, 56, dict(num_blocks=3, reset_branch=5)),
    ('RefVSR_MFID', 40, 56, dict(num_blocks=3, reset_branch=5, scale=2, matching_ksize=4)),
    ('RefVSR_small_MFID_8K', 48, 64, dict(num_blocks=2, reset_branch=3)),
], ids=['x4', 'x2', 'flag_hd_in'])
def test_forward_yuv420_batch_equals_single_streams(name, h, w, over):
    """n = 2 through one batched schedule (forward_yuv420, push_frames_yuv420 and 8-bit calls in turn) equals two n = 1 streams"""
    t, frames, nv12 = 7 if name == 'RefVSR_MFID' else 3, 9, True
    clips = [_yuv_clip(frames, h, w, 40 + i, nv12) for i in range(2)]
    wins = [list(_windows(*c, t)) for c in clips]
    batched = _engine(name, seed=40, **over)
    singles = [_engine(name, seed=40, **over) for _ in range(2)]
    for k in range(frames):
        first = wins[0][k][3]
        wl = torch.cat([wins[i][k][1] for i in range(2)])
        wr = torch.cat([wins[i][k][2] for i in range(2)])
        if first or k % 3 == 1:
            out = batched.forward_yuv420(wl, wr, first, nv12=nv12)
        elif k % 3 == 2:
            out = batched.push_frames_yuv420(wl[:, -1].contiguous(), wr[:, -1].contiguous(), nv12=nv12)
        else:
            out = rgb_to_yuv420(batched.push_frames_u8(_rgb(wl[:, -1], nv12), _rgb(wr[:, -1], nv12)).cpu(), nv12).cuda()
        for i in range(2):
            exp = singles[i].forward_yuv420(wins[i][k][1], wins[i][k][2], first, nv12=nv12)[0]
            assert torch.equal(out[i], exp), f'{name} window {k}, element {i}'
    assert batched.Network.batch_fallbacks == 0 and batched.Network.reuse_fallbacks == 0
    assert any(key[0] == 'batch' and key[-1] == FRAME_NV12 for key in batched.Network._graphs)


def test_yuv420_non_sliding_caller_recomputes():
    """a caller whose next window does not slide by one gets a full recompute (the reuse guard compares the converted values),
    equal to what forward_u8 gives for the same calls"""
    h, w, t = 40, 56, 7
    lrs, refs = _yuv_clip(9, h, w, 50, False)
    net, ref = (_engine('RefVSR_MFID', seed=50, num_blocks=3) for _ in range(2))
    wins = list(_windows(lrs, refs, t))
    for k in (0, 1, 4):                                                    # window 4 skips two windows
        got = net.forward_yuv420(wins[k][1], wins[k][2], k == 0)
        want = rgb_to_yuv420(ref.forward_u8(_rgb(wins[k][1], False), _rgb(wins[k][2], False), k == 0).cpu())
        assert torch.equal(got.cpu(), want), f'window {k}'
        assert net.Network.reuse_fallbacks == ref.Network.reuse_fallbacks == (1 if k == 4 else 0)
