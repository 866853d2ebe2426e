"""-m gpu: the 8-bit frame path on the H100.  rv_frames_from_u8 against torch's u8.float() / 255; rv_reconstruct_u8{,_batched}
against frame_u8 of rv_reconstruct's fp32 output on every path (x4, x2, generic) and x dtype; and the engine's forward_u8 /
push_frame_u8 / push_frames_u8 against rv_eval_images of the fp32 path's result (the bytes the evaluation loop writes).
Synthetic clips and seeded weights only."""
import pytest
import torch

from u8_ops import hwc_u8, planar_f32

pytestmark = pytest.mark.gpu


def _engine(name, seed=7, **over):
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    net = SRNet(get_config(name, device='cuda', b200_precision='bf16', **over)).eval()
    seeded_test_weights(net, seed=seed)
    return net.cuda()


def _u8_clip(frames, h, w, seed):
    from refvsr_b200.synth import make_clip
    lrs, refs = make_clip(frames, h, w, 1, seed=seed)
    return hwc_u8(lrs, False).cuda(), hwc_u8(refs, False).cuda()


def _windows(lrs, refs, t):
    n = lrs.shape[0]
    for k in range(n):
        idx = [min(max(k - t // 2 + j, 0), n - 1) for j in range(t)]
        yield k, lrs[idx].unsqueeze(0), refs[idx].unsqueeze(0), k == 0


def _bgr_bytes(cuda_ops, result):
    """the evaluation loop's bytes for forward()'s (n, 3, H, W) result: rv_eval_images, B, G, R"""
    H, W = result.shape[-2:]
    return torch.stack([cuda_ops.eval_images([r.unsqueeze(0).contiguous()]).view(H, W, 3).clone() for r in result])


@pytest.mark.parametrize('h,w', [(1, 1), (7, 37), (33, 45), (64, 96), (270, 481)])
@pytest.mark.parametrize('bgr', [False, True])
def test_frames_from_u8_is_division_by_255(cuda_ops, h, w, bgr):
    """every byte value, odd widths, every source alignment mod 16 and unaligned destinations"""
    g = torch.Generator().manual_seed(h * 1000 + w)
    k = 16
    stride = 16 * ((3 * h * w + 15) // 16) + 16
    pool = torch.randint(0, 256, (k * stride + 16,), dtype=torch.uint8, generator=g)
    pool[:min(256, 3 * h * w)] = torch.arange(min(256, 3 * h * w), dtype=torch.uint8)
    pool = pool.cuda()
    srcs = [pool[s * stride + s:][:3 * h * w].view(h, w, 3) for s in range(k)]          # source s starts at s mod 16
    dpool = torch.full((k * (3 * h * w + 5),), float('nan'), device='cuda')
    dsts = [dpool[s * (3 * h * w + 5) + (s % 5):][:3 * h * w].view(3, h, w) for s in range(k)]
    cuda_ops.frames_from_u8(srcs, dsts, bgr)
    for s, d in zip(srcs, dsts):
        assert torch.equal(d, planar_f32(s, bgr)), (h, w, s.data_ptr() % 16, d.data_ptr() % 16)
    assert {s.data_ptr() % 16 for s in srcs} == set(range(16))
    u = torch.arange(256, dtype=torch.uint8, device='cuda').view(256, 1, 1).expand(256, 1, 3).contiguous()
    d = torch.empty(3, 256, 1, device='cuda')
    cuda_ops.frames_from_u8([u], [d], bgr)
    assert torch.equal(d[0, :, 0].cpu(), torch.arange(256, dtype=torch.float32) / 255)


def _tail_inputs(n, h, w, s, xc, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(n, s * h, s * w, xc, generator=g) * 1.4 - 0.7)
    x.view(-1, xc)[:64, 0] = torch.tensor([0.5 / 255, 1.5 / 255, 2.5 / 255, -0.0, 1e30, -1e30, float('nan'), 1.0] * 8)
    lr = torch.rand(n, 3, h, w, generator=g)
    return x.to(dtype).cuda(), lr.cuda()


TAIL = [  # (scale, xc, dtype, h, w): fp32 with xc = 4 takes the x4 / x2 fast paths, every other case the generic kernel
    (4, 4, torch.float32, 270, 480), (4, 4, torch.float32, 17, 23), (4, 4, torch.float32, 9, 4),
    (2, 4, torch.float32, 136, 240), (2, 4, torch.float32, 17, 21), (2, 4, torch.float32, 6, 8),
    (4, 4, torch.bfloat16, 33, 41), (4, 4, torch.float16, 20, 24), (2, 4, torch.bfloat16, 19, 26),
    (4, 6, torch.float32, 13, 21), (2, 3, torch.float16, 11, 15),
]


@pytest.mark.parametrize('scale,xc,dtype,h,w', TAIL, ids=[f'x{c[0]}-c{c[1]}-{str(c[2])[6:]}-{c[3]}x{c[4]}' for c in TAIL])
def test_reconstruct_u8_is_frame_u8_of_reconstruct(cuda_ops, scale, xc, dtype, h, w):
    for n in (1, 3):
        x, lr = _tail_inputs(n, h, w, scale, xc, dtype, seed=h * w + n)
        ref = torch.empty(n, 3, scale * h, scale * w, device='cuda')
        for clamp in (True, False):
            cuda_ops.reconstruct(x if n > 1 else x[0], lr if n > 1 else lr[0], scale, clamp, ref if n > 1 else ref[0])
            for bgr in (False, True):
                out = torch.full((n, scale * h, scale * w, 3), 7, dtype=torch.uint8, device='cuda')
                cuda_ops.reconstruct_u8(x if n > 1 else x[0], lr if n > 1 else lr[0], scale, clamp, out if n > 1 else out[0], bgr)
                want = hwc_u8(ref, bgr)
                assert torch.equal(out, want), f'n={n} clamp={clamp} bgr={bgr}: {int((out != want).sum())} bytes differ'
    # an unaligned output buffer takes the byte stores, to the same bytes
    x, lr = _tail_inputs(1, h, w, scale, xc, dtype, seed=3)
    ref = torch.empty(3, scale * h, scale * w, device='cuda')
    cuda_ops.reconstruct(x[0], lr[0], scale, True, ref)
    buf = torch.zeros(3 * scale * h * scale * w + 1, dtype=torch.uint8, device='cuda')
    out = buf[1:].view(scale * h, scale * w, 3)
    cuda_ops.reconstruct_u8(x[0], lr[0], scale, True, out, True)
    assert torch.equal(out, hwc_u8(ref, True))


def test_reconstruct_u8_refuses_bad_arguments(cuda_ops):
    lib = cuda_ops.lib
    assert lib.rv_reconstruct_u8(None, 4, 0, None, 4, 4, 4, 1, 0, None, None) == -1
    x = torch.zeros(16, 16, 4, device='cuda')
    lr = torch.zeros(3, 4, 4, device='cuda')
    o = torch.zeros(16, 16, 3, dtype=torch.uint8, device='cuda')
    assert lib.rv_reconstruct_u8(x.data_ptr(), 4, 0, lr.data_ptr(), 4, 4, 3, 1, 0, o.data_ptr(), None) == -1     # scale 3
    assert lib.rv_reconstruct_u8_batched(x.data_ptr(), 4, 0, lr.data_ptr(), 4, 4, 4, 1, 0, o.data_ptr(), 0, None) == -1
    assert lib.rv_frames_from_u8(None, None, 1, 4, 4, 0, None) == -1
    import ctypes as C
    p = (C.c_void_p * 1)(o.data_ptr())
    q = (C.c_void_p * 1)(x.data_ptr())
    assert lib.rv_frames_from_u8(p, q, 17, 4, 4, 0, None) == -1
    assert lib.rv_frames_from_u8(p, q, 1, 0, 4, 0, None) == -1
    assert lib.rv_frames_from_u8((C.c_void_p * 1)(None), q, 1, 4, 4, 0, None) == -1


def _check_clip(cuda_ops, name, h, w, frames, t, seed, **over):
    """first, steady and forced-reset windows: forward_u8 / push_frame_u8 (both orders) against rv_eval_images of forward()"""
    lrs, refs = _u8_clip(frames, h, w, seed)
    nf, nu, np_ = (_engine(name, seed=seed, **over) for _ in range(3))
    assert nu.Network.use_graphs and nu.Network.overlap_branches
    for k, wl, wr, first in _windows(lrs, refs, t):
        res = nf(planar_f32(wl, False), planar_f32(wr, False), first)['result']
        want = _bgr_bytes(cuda_ops, res)
        got = nu.forward_u8(wl.flip(-1).contiguous(), wr.flip(-1).contiguous(), first, bgr=True)
        assert torch.equal(got, want), f'{name} window {k}: forward_u8 (BGR)'
        if first:
            got = np_.forward_u8(wl, wr, True)
        else:
            got = np_.push_frame_u8(wl[0, -1], wr[0, -1]).unsqueeze(0)
        assert torch.equal(got, want.flip(-1)), f'{name} window {k}: push_frame_u8 (RGB)'
    for net in (nu, np_):
        assert net.Network.reuse_fallbacks == 0
    assert any(key[-1] is True for key in nu.Network._graphs) and any(key[-1] is False for key in np_.Network._graphs)
    assert nf.Network.frame_itr_num == nu.Network.frame_itr_num == np_.Network.frame_itr_num


def test_forward_u8_mfid_270x480(cuda_ops):
    """RefVSR_MFID at the bench shape with graphs and branch overlap; reset_branch = 4 puts a forced reset inside the clip"""
    _check_clip(cuda_ops, 'RefVSR_MFID', 270, 480, 7, 7, 31, reset_branch=4)


def test_forward_u8_x2(cuda_ops):
    _check_clip(cuda_ops, 'RefVSR_MFID', 136, 240, 6, 7, 32, num_blocks=4, scale=2, matching_ksize=4, reset_branch=3)


def test_forward_u8_flag_hd_in(cuda_ops):
    _check_clip(cuda_ops, 'RefVSR_small_MFID_8K', 48, 64, 6, 3, 33, num_blocks=2, reset_branch=2)


def test_forward_u8_batch_equals_single_streams(cuda_ops):
    """n = 2 through one batched schedule (forward_u8, then push_frames_u8) equals two n = 1 streams, byte for byte"""
    h, w, t, frames = 40, 56, 7, 9
    clips = [_u8_clip(frames, h, w, 40 + i) for i in range(2)]
    wins = [list(_windows(*c, t)) for c in clips]
    batched = _engine('RefVSR_MFID', seed=40, num_blocks=3, reset_branch=5)
    singles = [_engine('RefVSR_MFID', seed=40, num_blocks=3, reset_branch=5) for _ in range(2)]
    for k in range(frames):
        first = wins[0][k][3]
        if first or k % 2:
            out = batched.forward_u8(torch.cat([wins[i][k][1] for i in range(2)]), torch.cat([wins[i][k][2] for i in range(2)]), first)
        else:
            out = batched.push_frames_u8(torch.stack([wins[i][k][1][0, -1] for i in range(2)]),
                                         torch.stack([wins[i][k][2][0, -1] for i in range(2)]))
        for i in range(2):
            exp = singles[i].forward_u8(wins[i][k][1], wins[i][k][2], first)[0]
            assert torch.equal(out[i], exp), f'window {k}, element {i}'
    assert batched.Network.batch_fallbacks == 0 and batched.Network.reuse_fallbacks == 0
    assert any(key[0] == 'batch' for key in batched.Network._graphs)
