"""-m gpu: every CUDA kernel behind the C ABI against the oracle (oracle/oracle_ops.py, CPU fp32) on the
same seeded inputs.  Tolerances are written next to each check: fp32 paths 1e-4 (accumulation order),
16-bit paths a few ulps of the storage type."""
import pytest
import torch

from refvsr_b200 import packing
from refvsr_b200.lib import (ACT_CLAMP3, ACT_LRELU01, ACT_LRELU02, ACT_NONE, ACT_RELU, IMPL_SIMT, IMPL_TC)

pytestmark = pytest.mark.gpu

DT = {'fp32': torch.float32, 'fp16': torch.float16, 'bf16': torch.bfloat16}
TOL = {torch.float32: 2e-4, torch.float16: 4e-3, torch.bfloat16: 3e-2}


def g(seed):
    return torch.Generator(device='cpu').manual_seed(seed)


def rnd(shape, seed, dtype=torch.float32, scale=1.0):
    return ((torch.rand(shape, generator=g(seed)) * 2 - 1) * scale).to(dtype)


def close(a, b, tol, what=''):
    a, b = a.float().cpu(), b.float().cpu()
    err = (a - b).abs().max().item()
    ref = b.abs().max().item() + 1e-6
    assert err <= tol * max(1.0, ref), f'{what}: max err {err:.3e} (ref max {ref:.3e}, tol {tol})'


# ---------------------------------------------------------------------------------------------
# convolution: SIMT and wgmma implementations against F.conv2d-based oracle
# ---------------------------------------------------------------------------------------------
CONV_CASES = [
    # name, H, W, srcs[(real,alloc)], cout, k, stride, pad, act_pre, act_post, gate, res, shuffle, out_f32
    ('rb3x3', 37, 53, [(48, 48)], 48, 3, 1, 1, ACT_RELU, ACT_NONE, False, True, False, False),
    ('gated', 19, 40, [(48, 48)], 48, 3, 1, 1, ACT_LRELU02, ACT_NONE, True, True, False, False),
    ('in_conv', 33, 47, [(3, 8), (48, 48)], 48, 3, 1, 1, ACT_LRELU01, ACT_NONE, False, False, False, False),
    ('cat96', 24, 32, [(48, 48), (48, 48)], 48, 3, 1, 1, ACT_LRELU02, ACT_NONE, False, False, False, False),
    ('small24', 21, 35, [(24, 24), (24, 24)], 24, 3, 1, 1, ACT_LRELU02, ACT_NONE, False, True, False, False),
    ('shuffle', 17, 29, [(48, 48)], 192, 3, 1, 1, ACT_LRELU01, ACT_NONE, False, False, True, False),
    ('shuffle24', 17, 29, [(24, 24)], 96, 3, 1, 1, ACT_NONE, ACT_NONE, False, False, True, False),
    ('spy0', 36, 60, [(8, 8)], 32, 7, 1, 3, ACT_RELU, ACT_NONE, False, False, False, False),
    ('spy1', 18, 30, [(32, 32)], 64, 7, 1, 3, ACT_RELU, ACT_NONE, False, False, False, False),
    ('spy2', 9, 15, [(64, 64)], 32, 7, 1, 3, ACT_RELU, ACT_NONE, False, False, False, False),
    ('spy4_flow', 36, 60, [(16, 16)], 2, 7, 1, 3, ACT_NONE, ACT_NONE, False, True, False, True),
    ('align5x5', 30, 44, [(3, 8)], 32, 5, 1, 2, ACT_LRELU02, ACT_NONE, False, False, False, False),
    ('post_act', 30, 44, [(32, 32)], 32, 3, 1, 1, ACT_NONE, ACT_LRELU02, False, True, False, False),
    ('vgg1x1', 25, 31, [(64, 64)], 16, 1, 1, 0, ACT_LRELU02, ACT_NONE, False, False, False, False),
    ('fusion1x1', 25, 31, [(48, 48), (48, 48)], 48, 1, 1, 0, ACT_NONE, ACT_NONE, False, False, False, False),
    ('conf16', 25, 31, [(2, 8)], 16, 3, 1, 1, ACT_LRELU02, ACT_NONE, False, False, False, False),
    ('last3', 40, 48, [(48, 48)], 3, 3, 1, 1, ACT_NONE, ACT_NONE, False, False, False, True),
    ('affine', 20, 28, [(32, 32)], 3, 1, 1, 0, ACT_NONE, ACT_CLAMP3, False, False, False, True),
    ('tiny', 2, 3, [(48, 48)], 48, 3, 1, 1, ACT_RELU, ACT_NONE, False, True, False, False),
    ('pconv_s2', 30, 44, [(32, 32), (32, 32)], 32, 5, 2, 2, ACT_LRELU02, ACT_NONE, False, False, False, False),
    ('enc_s2', 31, 45, [(48, 48)], 48, 3, 2, 1, ACT_LRELU02, ACT_NONE, False, False, False, False),
]


def _run_conv(ops, oracle, case, dtype, prefer_tc, tc_layout=None):
    name, H, W, srcs, cout, k, stride, pad, a_pre, a_post, use_gate, use_res, shuffle, out_f32 = case
    cin = sum(r for r, _ in srcs)
    w = rnd((cout, cin, k, k), 1, scale=(1.5 / (cin * k * k) ** 0.5)).to(dtype).float()   # representable in `dtype`
    b = rnd((cout,), 2, scale=0.1)
    xs = [rnd((H, W, a), 10 + i, dtype) for i, (_, a) in enumerate(srcs)]
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    odt = torch.float32 if out_f32 else dtype
    gate = rnd((Ho, Wo, cout), 3, dtype) if use_gate else None
    res = rnd((Ho, Wo, cout), 4, odt) if use_res else None
    oshape = (2 * Ho, 2 * Wo, cout // 4) if shuffle else (Ho, Wo, cout if not out_f32 else max(cout, 4))
    # oracle
    lo = oracle.pack_conv(name, w, b, srcs, stride, pad, dtype, 'cpu', False, 1.0 if a_post == ACT_CLAMP3 else 0.0)
    exp = torch.zeros(oshape, dtype=torch.float32)
    oracle.conv2d(lo, xs[0], xs[1] if len(xs) > 1 else None, exp, gate=gate, res=res, act_pre=a_pre,
                  act_post=a_post, pixel_shuffle=shuffle)
    # cuda
    lc = packing.pack_conv(name, w, b, srcs, stride, pad, dtype, 'cuda', prefer_tc, 1.0 if a_post == ACT_CLAMP3 else 0.0,
                           tc_layout=tc_layout)
    out = torch.zeros(oshape, dtype=odt, device='cuda')
    cx = [x.cuda() for x in xs]
    ops.conv2d(lc, cx[0], cx[1] if len(cx) > 1 else None, out, gate=None if gate is None else gate.cuda(),
               res=None if res is None else res.cuda(), act_pre=a_pre, act_post=a_post, pixel_shuffle=shuffle)
    torch.cuda.synchronize()
    return lc, out, exp


@pytest.mark.parametrize('case', CONV_CASES, ids=[c[0] for c in CONV_CASES])
@pytest.mark.parametrize('prec', ['fp32', 'fp16', 'bf16'])
def test_conv_simt(cuda_ops, oracle_ops, case, prec):
    lc, out, exp = _run_conv(cuda_ops, oracle_ops, case, DT[prec], prefer_tc=False)
    assert lc.impl == IMPL_SIMT
    close(out, exp, TOL[out.dtype] if out.dtype != torch.float32 else 2e-4, f'conv_simt[{case[0]},{prec}]')


@pytest.mark.parametrize('case', [c for c in CONV_CASES if c[6] == 1], ids=[c[0] for c in CONV_CASES if c[6] == 1])
@pytest.mark.parametrize('prec', ['fp16', 'bf16'])
@pytest.mark.parametrize('layout', [0, 1, 2, 3])
def test_conv_tc(cuda_ops, oracle_ops, case, prec, layout):
    """layout 0: one 128B-swizzled 64-channel TMA box per (kx, chunk) stage; layout 1: one box per (tile, chunk), taps
    as shifted UMMA descriptor views (only where all taps stay resident in shared memory); layout 2: 32B-swizzled
    16-channel quads (one UMMA_K slice per row)"""
    if layout in (1, 3) and not packing.layout1_fits(case[5], case[5], case[3], packing.choose_nb(case[4])):
        pytest.skip('weights of this conv are streamed (layout 0 only)')
    # layout 3 = the layout-1 weight image with the kx-folded 3x3 mode disabled (layout 1 folds when eligible)
    lc, out, exp = _run_conv(cuda_ops, oracle_ops, case, DT[prec], prefer_tc=True, tc_layout=layout)
    assert lc.impl == IMPL_TC and lc.layout == layout, 'stride-1 16-bit convs must take the tensor-core path'
    close(out, exp, TOL[out.dtype] if out.dtype != torch.float32 else 2e-4, f'conv_tc[{case[0]},{prec}]')


RB_CASES = [  # name, H, W, C(real), alloc, act_mid, act_post
    ('noBN48', 37, 53, 48, 48, ACT_RELU, ACT_NONE),
    ('res48', 64, 40, 48, 48, ACT_LRELU02, ACT_NONE),
    ('align32', 30, 44, 32, 32, ACT_LRELU02, ACT_LRELU02),
    ('small24', 33, 21, 24, 24, ACT_RELU, ACT_NONE),
    ('tiny', 3, 5, 48, 48, ACT_RELU, ACT_NONE),
    ('one_tile_exact', 16, 8, 48, 48, ACT_RELU, ACT_NONE),
]


@pytest.mark.parametrize('case', RB_CASES, ids=[c[0] for c in RB_CASES])
@pytest.mark.parametrize('prec', ['fp16', 'bf16'])
def test_resblock_fused(cuda_ops, oracle_ops, case, prec):
    """rv_resblock (one launch: conv -> act -> conv -> +x) against the oracle's two convolutions"""
    name, H, W, C, alloc, a_mid, a_post = case
    dt = DT[prec]
    w1 = rnd((C, C, 3, 3), 1, scale=1.5 / (C * 9) ** 0.5).to(dt).float()
    w2 = rnd((C, C, 3, 3), 2, scale=1.5 / (C * 9) ** 0.5).to(dt).float()
    b1, b2 = rnd((C,), 3, scale=0.2), rnd((C,), 4, scale=0.2)
    x = rnd((H, W, alloc), 5, dt)
    ro = oracle_ops.pack_resblock(name, w1, b1, w2, b2, alloc, dt, 'cpu')
    exp = torch.zeros((H, W, C))
    oracle_ops.resblock(ro, x, exp, a_mid, a_post)
    rc = packing.pack_resblock(name, w1, b1, w2, b2, alloc, dt, 'cuda')
    out = torch.zeros((H, W, alloc), dtype=dt, device='cuda')
    cuda_ops.resblock(rc, x.cuda(), out, a_mid, a_post)
    torch.cuda.synchronize()
    close(out[..., :C], exp, TOL[dt], f'resblock[{name},{prec}]')


def test_resblock_fused_full_size_matches_two_convs(cuda_ops):
    """270x480x48: fused kernel == conv_tc + conv_tc (same 16-bit intermediate rounding)"""
    H, W, C = 270, 480, 48
    dt = torch.bfloat16
    w1 = rnd((C, C, 3, 3), 1, scale=0.07).to(dt).float()
    w2 = rnd((C, C, 3, 3), 2, scale=0.07).to(dt).float()
    b1, b2 = rnd((C,), 3, scale=0.1), rnd((C,), 4, scale=0.1)
    x = rnd((H, W, C), 5, dt).cuda()
    l1 = packing.pack_conv('a', w1, b1, [(C, C)], 1, 1, dt, 'cuda', True)
    l2 = packing.pack_conv('b', w2, b2, [(C, C)], 1, 1, dt, 'cuda', True)
    t = torch.zeros((H, W, C), dtype=dt, device='cuda')
    ref = torch.zeros((H, W, C), dtype=dt, device='cuda')
    cuda_ops.conv2d(l1, x, None, t, act_pre=ACT_RELU)
    cuda_ops.conv2d(l2, t, None, ref, res=x)
    rb = packing.pack_resblock('rb', w1, b1, w2, b2, C, dt, 'cuda')
    out = torch.zeros((H, W, C), dtype=dt, device='cuda')
    cuda_ops.resblock(rb, x, out, ACT_RELU)
    torch.cuda.synchronize()
    close(out, ref, 1e-2, 'fused vs two convs')
    assert (out.float() - ref.float()).abs().mean().item() < 2e-3


def test_conv_tc_large_matches_simt(cuda_ops):
    """full-size property: tensor-core path == CUDA-core path on a 270x480x48 map (fp16 storage ulp)."""
    H, W, C = 270, 480, 48
    w = rnd((C, C, 3, 3), 1, scale=0.07).half().float()
    b = rnd((C,), 2, scale=0.1)
    x = rnd((H, W, C), 3, torch.float16).cuda()
    r = rnd((H, W, C), 4, torch.float16).cuda()
    outs = []
    for tc in (False, True):
        lc = packing.pack_conv('big', w, b, [(C, C)], 1, 1, torch.float16, 'cuda', tc)
        o = torch.zeros((H, W, C), dtype=torch.float16, device='cuda')
        cuda_ops.conv2d(lc, x, None, o, res=r, act_pre=ACT_RELU)
        outs.append(o)
    torch.cuda.synchronize()
    close(outs[1], outs[0], 2e-3, 'tc vs simt 270x480')


# ---------------------------------------------------------------------------------------------
# pointwise / gather kernels
# ---------------------------------------------------------------------------------------------
def both(oracle_fn, cuda_fn, ins, out_shape, out_dtype):
    exp = torch.zeros(out_shape, dtype=out_dtype)
    oracle_fn(*ins, exp)
    got = torch.zeros(out_shape, dtype=out_dtype, device='cuda')
    cuda_fn(*[i.cuda() if torch.is_tensor(i) else i for i in ins], got)
    torch.cuda.synchronize()
    return got, exp


@pytest.mark.parametrize('prec', ['fp32', 'fp16'])
@pytest.mark.parametrize('up2', [False, True])
def test_warp(cuda_ops, oracle_ops, prec, up2):
    dt = DT[prec]
    h, w, C = 27, 41, 48
    flow = rnd((h, w, 2), 1, scale=3.0)
    src = rnd((2 * h, 2 * w, C) if up2 else (h, w, C), 2, dt)
    oshape = (2 * h, 2 * w, C) if up2 else (h, w, C)
    got, exp = both(lambda s, f, o: oracle_ops.warp(s, f, o, flow_up2=up2),
                    lambda s, f, o: cuda_ops.warp(s, f, o, flow_up2=up2), (src, flow), oshape, dt)
    close(got, exp, 1e-4 if dt == torch.float32 else 2e-3, 'warp')


def test_warp_quirk_lr_source_on_2x_grid(cuda_ops, oracle_ops):
    """RefVSR.py:254: an LR-size feature warped onto the 2x grid with the upsampled flow."""
    h, w, C = 20, 28, 24
    flow = rnd((h, w, 2), 1, scale=2.0)
    src = rnd((h, w, C), 2)
    got, exp = both(lambda s, f, o: oracle_ops.warp(s, f, o, flow_up2=True),
                    lambda s, f, o: cuda_ops.warp(s, f, o, flow_up2=True), (src, flow), (2 * h, 2 * w, C), torch.float32)
    close(got, exp, 1e-4, 'warp quirk')


def test_warp_conf_plane_and_zero_flow(cuda_ops, oracle_ops):
    h, w = 30, 44
    conf = torch.rand((h, w), generator=g(5))
    flow = torch.zeros((h, w, 2))
    got, exp = both(lambda s, f, o: oracle_ops.warp(s, f, o), lambda s, f, o: cuda_ops.warp(s, f, o), (conf, flow),
                    (h, w), torch.float32)
    close(got, exp, 1e-5, 'conf warp')
    assert (got.cpu() - conf).abs().max() > 1e-3, 'zero flow is NOT the identity in the reference (SURVEY A1)'


def test_prep_image(cuda_ops, oracle_ops):
    img = torch.rand((3, 26, 38), generator=g(1))
    mat = [1 / 0.229, 0, 0, -0.485 / 0.229, 0, 1 / 0.224, 0, -0.456 / 0.224, 0, 0, 1 / 0.225, -0.406 / 0.225]
    for pool in (False, True):
        for m in (None, mat):
            shp = (13, 19, 8) if pool else (26, 38, 8)
            got, exp = both(lambda s, o: oracle_ops.prep_image(s, o, mat12=m, pool2=pool),
                            lambda s, o: cuda_ops.prep_image(s, o, mat12=m, pool2=pool), (img,), shp, torch.float32)
            close(got, exp, 1e-5, f'prep_image pool={pool}')


@pytest.mark.parametrize('prec', ['fp32', 'fp16', 'bf16'])
def test_maxpool2(cuda_ops, oracle_ops, prec):
    """vgg19.features[4] of the flag_HD_in matching path (odd sizes drop the last row / column like nn.MaxPool2d)"""
    dt = DT[prec]
    for (H, W, C) in ((26, 38, 64), (9, 7, 8)):
        x = rnd((H, W, C), 1, dt)
        got, exp = both(oracle_ops.maxpool2, cuda_ops.maxpool2, (x,), (H // 2, W // 2, C), dt)
        assert torch.equal(got.cpu(), exp), 'max of representable values is exact'


def test_resize_planes(cuda_ops, oracle_ops):
    """bicubic x4 (+clamp) of the relevance map, bicubic x0.5 (+clamp) of the LR frame, nearest x0.5 (attention.py:65-67,
    96-98; RefVSR.py:125)"""
    conf = torch.rand((1, 12, 17), generator=g(1)) * 1.2 - 0.1
    got, exp = both(lambda s, o: oracle_ops.resize_planes(s, o, 0.25, 'bicubic', True),
                    lambda s, o: cuda_ops.resize_planes(s, o, 0.25, 'bicubic', True), (conf,), (1, 48, 68), torch.float32)
    close(got, exp, 1e-5, 'bicubic x4 clamp')
    img = torch.rand((3, 26, 38), generator=g(2))
    for clamp in (False, True):
        got, exp = both(lambda s, o: oracle_ops.resize_planes(s, o, 2.0, 'bicubic', clamp),
                        lambda s, o: cuda_ops.resize_planes(s, o, 2.0, 'bicubic', clamp), (img,), (3, 13, 19), torch.float32)
        close(got, exp, 1e-5, f'bicubic x0.5 clamp={clamp}')
    got, exp = both(lambda s, o: oracle_ops.resize_planes(s, o, 2.0, 'nearest'),
                    lambda s, o: cuda_ops.resize_planes(s, o, 2.0, 'nearest'), (img,), (3, 13, 19), torch.float32)
    assert torch.equal(got.cpu(), exp)
    odd = torch.rand((3, 27, 39), generator=g(3))
    got, exp = both(lambda s, o: oracle_ops.resize_planes(s, o, 2.0, 'nearest'),
                    lambda s, o: cuda_ops.resize_planes(s, o, 2.0, 'nearest'), (odd,), (3, 13, 19), torch.float32)
    assert torch.equal(got.cpu(), exp)


def test_spynet_glue(cuda_ops, oracle_ops):
    img = torch.rand((3, 27, 45), generator=g(1))
    got, exp = both(oracle_ops.spynet_resize_norm, cuda_ops.spynet_resize_norm, (img,), (32, 64, 3), torch.float32)
    close(got, exp, 1e-5, 'resize_norm')
    lvl = exp
    got, exp = both(oracle_ops.avgpool2, cuda_ops.avgpool2, (lvl,), (16, 32, 3), torch.float32)
    close(got, exp, 1e-6, 'avgpool2')
    ref, supp = rnd((16, 32, 3), 3), rnd((16, 32, 3), 4)
    fprev = rnd((8, 16, 2), 5, scale=2.0)
    for fp in (None, fprev):
        e8, ef = torch.zeros((16, 32, 8)), torch.zeros((16, 32, 2))
        oracle_ops.spynet_level_input(ref, supp, fp, e8, ef)
        g8 = torch.zeros((16, 32, 8), device='cuda')
        gf = torch.zeros((16, 32, 2), device='cuda')
        cuda_ops.spynet_level_input(ref.cuda(), supp.cuda(), None if fp is None else fp.cuda(), g8, gf)
        torch.cuda.synchronize()
        close(g8, e8, 1e-5, 'level_input x8')
        close(gf, ef, 1e-5, 'level_input flow_up')
    flow = rnd((32, 64, 2), 6, scale=4.0)
    got, exp = both(oracle_ops.flow_resize, cuda_ops.flow_resize, (flow,), (27, 45, 2), torch.float32)
    close(got, exp, 1e-5, 'flow_resize')


def test_space_to_depth(cuda_ops, oracle_ops):
    x = rnd((14, 22, 48), 1, torch.float16)
    got, exp = both(oracle_ops.space_to_depth2, cuda_ops.space_to_depth2, (x,), (7, 11, 192), torch.float16)
    assert torch.equal(got.cpu(), exp)


def test_stride2_conv_via_space_to_depth_on_tensor_cores(cuda_ops, oracle_ops):
    """ref_encoder2.0.0 (3x3 s2) and aa2.align.p_conv.0 (5x5 s2, two sources) through s2d + wgmma"""
    for k, srcs in ((3, [(48, 48)]), (5, [(32, 32), (32, 32)])):
        cin = sum(r for r, _ in srcs)
        w = rnd((32, cin, k, k), 1, scale=1.5 / (cin * k * k) ** 0.5).half().float()
        b = rnd((32,), 2, scale=0.1)
        xs = [rnd((30, 44, a), 10 + i, torch.float16) for i, (_, a) in enumerate(srcs)]
        lo = oracle_ops.pack_conv('ref', w, b, srcs, 2, k // 2, torch.float16, 'cpu', False)
        exp = torch.zeros((15, 22, 32))
        oracle_ops.conv2d(lo, xs[0], xs[1] if len(xs) > 1 else None, exp, act_pre=ACT_LRELU02)
        w2, srcs2 = packing.s2d_weights(w, srcs, k // 2)
        lc = packing.pack_conv('s2d', w2, b, srcs2, 1, 1, torch.float16, 'cuda', True)
        assert lc.impl == IMPL_TC
        zs = []
        for x in xs:
            z = torch.empty((15, 22, 4 * x.shape[2]), dtype=torch.float16, device='cuda')
            cuda_ops.space_to_depth2(x.cuda(), z)
            zs.append(z)
        out = torch.zeros((15, 22, 32), dtype=torch.float16, device='cuda')
        cuda_ops.conv2d(lc, zs[0], zs[1] if len(zs) > 1 else None, out, act_pre=ACT_LRELU02)
        torch.cuda.synchronize()
        close(out, exp, 4e-3, f's2d conv k={k}')


@pytest.mark.parametrize('C', [48, 24, 40, 4])          # 6 / 3 vectors per row (compiled widths), 5 (run-time width), 8-byte rows
@pytest.mark.parametrize('ks', [1, 2])
def test_gather_blocks(cuda_ops, oracle_ops, ks, C):
    hq, wq = 14, 45
    Hv, Wv = 9 * ks, 13 * ks
    value = rnd((Hv, Wv, C), 1, torch.float16)
    idx = torch.randint(0, (Hv // ks) * (Wv // ks), (hq * wq,), generator=g(2), dtype=torch.int32)
    got, exp = both(lambda v, i, o: oracle_ops.gather_blocks(v, i, hq, wq, ks, o),
                    lambda v, i, o: cuda_ops.gather_blocks(v, i, hq, wq, ks, o), (value, idx), (ks * hq, ks * wq, C),
                    torch.float16)
    assert torch.equal(got.cpu(), exp), 'gather is a pure copy: must be bit exact'


@pytest.mark.parametrize('C', [48, 40])
@pytest.mark.parametrize('prec', ['fp32', 'fp16', 'bf16'])
def test_aligned_sample(cuda_ops, oracle_ops, prec, C):
    dt = DT[prec]
    h, w, ks = 13, 17, 2
    x = rnd((ks * h, ks * w, C), 1, dt)
    aff = (1.0 + rnd((h, w, 3), 2, scale=1.5)).clamp(-3, 3)
    got, exp = both(lambda a, b, o: oracle_ops.aligned_sample(a, b, ks, o), lambda a, b, o: cuda_ops.aligned_sample(a, b, ks, o),
                    (x, aff), (ks * h, ks * w, C), dt)
    close(got, exp, 2e-4 if dt == torch.float32 else (3e-3 if prec == 'fp16' else 2.5e-2), 'aligned_sample')
    # identity at affine == (1,1,1) (SURVEY 8c known-answer fact)
    one = torch.ones((h, w, 3))
    got, _ = both(lambda a, b, o: oracle_ops.aligned_sample(a, b, ks, o), lambda a, b, o: cuda_ops.aligned_sample(a, b, ks, o),
                  (x, one), (ks * h, ks * w, C), dt)
    close(got, x, 1e-6 if dt == torch.float32 else (1e-3 if prec == 'fp16' else 8e-3), 'aligned_sample identity')


def test_bicubic_conf_reconstruct(cuda_ops, oracle_ops):
    img = torch.rand((3, 21, 33), generator=g(1))
    got, exp = both(oracle_ops.bicubic_up2_image, cuda_ops.bicubic_up2_image, (img,), (42, 66, 8), torch.float32)
    close(got, exp, 1e-5, 'bicubic_up2_image')
    a, b = torch.rand((21, 33), generator=g(2)), torch.rand((21, 33), generator=g(3))
    for up2 in (False, True):
        shp = (42, 66, 8) if up2 else (21, 33, 8)
        got, exp = both(lambda x, y, o: oracle_ops.conf_pair(x, y, o, up2=up2), lambda x, y, o: cuda_ops.conf_pair(x, y, o, up2=up2),
                        (a, b), shp, torch.float32)
        close(got, exp, 1e-5, f'conf_pair up2={up2}')
    got, exp = both(oracle_ops.conf_max, cuda_ops.conf_max, (a, b), (21, 33), torch.float32)
    assert torch.equal(got.cpu(), exp)
    x = rnd((84, 132, 4), 4, scale=0.3)
    for clamp in (False, True):
        got, exp = both(lambda t, l, o: oracle_ops.reconstruct(t, l, 4, clamp, o), lambda t, l, o: cuda_ops.reconstruct(t, l, 4, clamp, o),
                        (x, img), (3, 84, 132), torch.float32)
        close(got, exp, 1e-5, f'reconstruct clamp={clamp}')


# ---------------------------------------------------------------------------------------------
# matching
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('mode', [0, 1, 2])
def test_patch_pack(cuda_ops, oracle_ops, mode):
    feat = rnd((19, 27, 16), 1, torch.float16)
    kpad = 192 if mode == 0 else 448
    got, exp = both(lambda f, o: oracle_ops.patch_pack(f, o, mode), lambda f, o: cuda_ops.patch_pack(f, o, mode), (feat,),
                    (19 * 27, kpad), torch.float16)
    # fp16 hi parts agree to 1 ulp, lo parts are tiny: compare the reconstructed values
    close(got, exp, 1e-3, 'patch_pack')


@pytest.mark.parametrize('split', [False, True])
@pytest.mark.parametrize('impl', [0, 1])
def test_match_argmax(cuda_ops, oracle_ops, split, impl):
    """argmax over reference patches; ragged sizes (P, R not multiples of the 128 x 256 tile)."""
    lr_f = rnd((37, 45, 16), 1)
    ref_f = rnd((23, 31, 16), 2)
    kpad = 448 if split else 192
    P, R = 37 * 45, 23 * 31
    A, B = torch.zeros((P, kpad), dtype=torch.float16), torch.zeros((R, kpad), dtype=torch.float16)
    oracle_ops.patch_pack(lr_f, A, 1 if split else 0)
    oracle_ops.patch_pack(ref_f, B, 2 if split else 0)
    conf_e, idx_e = torch.zeros(P), torch.zeros(P, dtype=torch.int32)
    oracle_ops.match_argmax(A, B, conf_e, idx_e)
    conf = torch.zeros(P, device='cuda')
    idx = torch.zeros(P, dtype=torch.int32, device='cuda')
    cuda_ops.match_argmax(A.cuda(), B.cuda(), conf, idx, impl=impl)
    torch.cuda.synchronize()
    close(conf, conf_e, 2e-5 if split else 1e-4, 'match conf')
    mism = (idx.cpu() != idx_e).float().mean().item()
    assert mism <= 2e-3, f'index mismatch rate {mism:.4f}'
    # where indices differ the scores must be ties within accumulation noise
    S = (B.float() @ A.float().t()) / 4096.0
    got_scores = S[idx.cpu().long(), torch.arange(P)]
    assert (conf_e - got_scores).max().item() <= 1e-5 + (0 if split else 1e-4)


def test_match_split_is_fp32_grade(cuda_ops, oracle_ops):
    """the [hi|lo|hi] x [hi|hi|lo] fp16 product reproduces the fp32 cosine similarity (attention.py:83-91)."""
    import torch.nn.functional as F
    from oracle import refvsr_oracle as O
    lr_f, ref_f = rnd((24, 40, 16), 1), rnd((16, 24, 16), 2)
    conf32, idx32 = O.match_argmax(lr_f.permute(2, 0, 1).unsqueeze(0), ref_f.permute(2, 0, 1).unsqueeze(0))
    P, R = 24 * 40, 16 * 24
    A = torch.zeros((P, 448), dtype=torch.float16, device='cuda')
    B = torch.zeros((R, 448), dtype=torch.float16, device='cuda')
    cuda_ops.patch_pack(lr_f.cuda(), A, 1)
    cuda_ops.patch_pack(ref_f.cuda(), B, 2)
    conf = torch.zeros(P, device='cuda')
    idx = torch.zeros(P, dtype=torch.int32, device='cuda')
    cuda_ops.match_argmax(A, B, conf, idx, impl=1)
    torch.cuda.synchronize()
    close(conf, conf32.flatten(), 5e-6, 'split conf vs fp32')
    assert (idx.cpu().long() != idx32.flatten()).float().mean().item() <= 2e-3


def test_errors_are_python_exceptions(cuda_ops):
    """error convention: Python exceptions, no crashes (SURVEY 8b)."""
    with pytest.raises(ValueError):
        cuda_ops.prep_image(torch.zeros((3, 5, 5), device='cuda'), torch.zeros((2, 2, 8), device='cuda'), pool2=True)
    w, b = torch.zeros((48, 48, 3, 3)), torch.zeros((48,))
    lc = packing.pack_conv('x', w, b, [(48, 48)], 1, 1, torch.float16, 'cuda', True)
    with pytest.raises(AssertionError):
        cuda_ops.conv2d(lc, torch.zeros((8, 8, 40), dtype=torch.float16, device='cuda'), None,
                        torch.zeros((8, 8, 48), dtype=torch.float16, device='cuda'))


# ---------------------------------------------------------------------------------------------------------------------
# rv_conv_chain: persistent cross-layer kernel (conv_chain.cu) == the same layers launched one by one, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
def _chain_case(cuda_ops, C, H, W, dt, kind, nblk, seed=0):
    from refvsr_b200 import packing
    from refvsr_b200.lib import ACT_LRELU02, ACT_NONE, ACT_RELU
    g = torch.Generator().manual_seed(seed)
    mk = lambda: torch.randn((H, W, C), generator=g).to(dt).cuda()
    nconv = 2 * nblk + (1 if kind == 'reslist' else 0)
    ws = [(torch.rand((C, C, 3, 3), generator=g) - 0.5) * (0.35 if i % 2 == 0 else 0.1) for i in range(nconv)]
    bs = [(torch.rand((C,), generator=g) - 0.5) * 0.1 for _ in range(nconv)]
    chain_l = [packing.pack_chain(f'c{i}', ws[i], bs[i], C, dt, 'cuda') for i in range(nconv)]
    # per-layer twin: layout 3 = the single-box image WITHOUT the kx-folded mode (whose fp32 summation order differs)
    conv_l = [packing.pack_conv(f'c{i}', ws[i], bs[i], [(C, C)], 1, 1, dt, 'cuda', True, tc_layout=3) for i in range(nconv)]
    x = mk()
    if kind == 'trunk':        # ResidualBlocksWithInputConv body: bufs [s0, s1, t, out]
        bufs = [x, torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)]
        layers, ci = [], 0
        for i in range(nblk):
            ni = 3 if i == nblk - 1 else 1 - ci
            layers.append((2 * i, ci, -1, 2, ACT_RELU, ACT_NONE))
            layers.append((2 * i + 1, 2, ci, ni, ACT_NONE, ACT_NONE))
            ci = ni
        out_idx = 3
    else:                      # ResList: bufs [x, s0, s1, t, out]
        bufs = [x] + [torch.empty_like(x) for _ in range(4)]
        layers, cur = [], 0
        for i in range(nblk):
            nxt = 1 + (i % 2)
            layers.append((2 * i, cur, -1, 3, ACT_LRELU02, ACT_NONE))
            layers.append((2 * i + 1, 3, cur, nxt, ACT_NONE, ACT_LRELU02 if i == 1 else ACT_NONE))   # one act_post for coverage
            cur = nxt
        layers.append((2 * nblk, cur, 0, 4, ACT_NONE, ACT_NONE))
        out_idx = 4
    return bufs, layers, chain_l, conv_l, out_idx


def _run_per_layer(cuda_ops, bufs, layers, conv_l):
    for li, src, res, dst, a0, a1 in layers:
        cuda_ops.conv2d(conv_l[li], bufs[src], None, bufs[dst], res=bufs[res] if res >= 0 else None, act_pre=a0, act_post=a1)


@pytest.mark.parametrize('C,H,W,kind,nblk', [(48, 16, 8, 'trunk', 2), (48, 37, 53, 'trunk', 3), (48, 64, 96, 'reslist', 4),
                                             (24, 40, 56, 'trunk', 3), (32, 33, 47, 'reslist', 2), (48, 135, 240, 'reslist', 4),
                                             (48, 270, 480, 'trunk', 30), (48, 540, 960, 'reslist', 4)],
                         ids=['1tile', 'odd', 'reslist', 'c24', 'c32', 'half', 'full_trunk', '2x_reslist'])
@pytest.mark.parametrize('prec', ['bf16', 'fp16'])
def test_conv_chain_matches_per_layer(cuda_ops, C, H, W, kind, nblk, prec):
    dt = DT[prec]
    bufs, layers, chain_l, conv_l, out_idx = _chain_case(cuda_ops, C, H, W, dt, kind, nblk)
    x0 = bufs[0].clone()
    _run_per_layer(cuda_ops, bufs, layers, conv_l)
    torch.cuda.synchronize()
    expect = bufs[out_idx].clone()
    assert torch.isfinite(expect.float()).all() and expect.float().abs().max() > 1e-3
    flags = torch.empty((((H + 15) // 16) * ((W + 7) // 8),), dtype=torch.int32, device='cuda')
    for rep in range(4 if H * W <= 270 * 480 else 2):             # repeated: a dependency race would not be deterministic
        for b in bufs[1:]:
            b.fill_(float('nan'))
        bufs[0].copy_(x0)
        cuda_ops.conv_chain(bufs, [(chain_l[li], src, res, dst, a0, a1) for li, src, res, dst, a0, a1 in layers], flags)
        torch.cuda.synchronize()
        assert torch.equal(bufs[out_idx], expect), \
            f'rep {rep}: {(bufs[out_idx].float() - expect.float()).abs().max().item():.3e} max abs, ' \
            f'{(bufs[out_idx] != expect).float().mean().item():.3e} of the elements differ'
        assert int(flags.min()) == len(layers) and int(flags.max()) == len(layers)


def test_conv_chain_more_than_64_layers_and_errors(cuda_ops):
    dt = torch.bfloat16
    bufs, layers, chain_l, conv_l, out_idx = _chain_case(cuda_ops, 48, 48, 64, dt, 'trunk', 40)      # 80 layers -> two launches
    x0 = bufs[0].clone()
    _run_per_layer(cuda_ops, bufs, layers, conv_l)
    expect = bufs[out_idx].clone()
    bufs[0].copy_(x0)
    flags = torch.empty((3 * 8,), dtype=torch.int32, device='cuda')
    cuda_ops.conv_chain(bufs, [(chain_l[li], src, res, dst, a0, a1) for li, src, res, dst, a0, a1 in layers], flags)
    assert torch.equal(bufs[out_idx], expect)
    with pytest.raises(ValueError, match='own source'):
        cuda_ops.conv_chain(bufs, [(chain_l[0], 0, -1, 0, 0, 0)], flags)


@pytest.mark.parametrize('prec', ['fp16', 'bf16'])
@pytest.mark.parametrize('h,w,C', [(24, 40, 48), (37, 53, 24), (19, 23, 64), (19, 23, 40), (270, 480, 48)])
def test_warp3_equals_three_warps(cuda_ops, prec, h, w, C):
    """rv_warp3 (one launch, one flow read, 2-D tiles) against the three rv_warp launches it replaces: same formulas; the LR
    feature and confidence are bit-identical, the 2x feature may differ in the last bit where the compiler contracts the
    flow-interpolation arithmetic differently in the two kernels"""
    dt = DT[prec]
    g = torch.Generator().manual_seed(5)
    feat = torch.randn((h, w, C), generator=g).to(dt).cuda()
    featUP = torch.randn((2 * h, 2 * w, C), generator=g).to(dt).cuda()
    conf = torch.rand((h, w), generator=g).cuda()
    flow = (torch.randn((h, w, 2), generator=g) * 3.0).cuda()
    flow[:4] *= 20.0                                       # some taps far outside the image (zeros padding)
    e_f, e_u, e_c = torch.empty_like(feat), torch.empty_like(featUP), torch.empty_like(conf)
    cuda_ops.warp(feat, flow, e_f)
    cuda_ops.warp(conf, flow, e_c)
    cuda_ops.warp(featUP, flow, e_u, flow_up2=True)
    o_f, o_u, o_c = torch.full_like(feat, float('nan')), torch.full_like(featUP, float('nan')), torch.full_like(conf, float('nan'))
    cuda_ops.warp3(feat, featUP, conf, flow, o_f, o_u, o_c)
    torch.cuda.synchronize()
    assert torch.equal(o_f, e_f) and torch.equal(o_c, e_c)
    d = (o_u.float() - e_u.float()).abs()
    assert float(d.max()) <= (8e-3 if prec == 'fp16' else 6e-2) and float((d > 0).float().mean()) < 0.05, (float(d.max()), float((d > 0).float().mean()))
