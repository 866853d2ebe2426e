"""Pixel-shuffle convs in the HR-row column order (packing.ps_rows_order, rv_conv_desc.ps_order = 1).

The upsampling convs (48 -> 192, 3 x 3, then a x2 pixel shuffle) are packed so that column block a is HR sub-row a of both
sub-pixels and all 48 channels.  Each CTA then writes whole HR pixels: the PSV kernel stages each half tile of HR rows in
shared memory and stores it with one TMA box (or, when the staging buffers do not fit, as 16-byte stores from registers).

Without a GPU: the order is a permutation that puts whole HR pixels in a block; the engine's upsample shapes plan the TMA
row store within an H100's shared memory with two A slots per consumer, and a smaller budget the 16-byte register stores;
the engine packs the upsampling convs, and only those, in this order; a desc whose order its kernel does not store (the
general epilogue: other shapes, misaligned outputs) is refused.
With a GPU: the TMA store, the 16-byte register stores and the conv's own column order give the same bits at every grid
cap, leave the NaN guards around the output and in channels >= cout alone, and pass test_conv_fp64's element-wise float64
bound."""
import ctypes as C

import pytest
import torch

from refvsr_b200 import packing
from refvsr_b200.lib import DTYPE_CODE, load_library, rv_conv_desc
from test_conv_fp64 import GUARD, _sig, check, make_operands, out_hw, reference

H100_SMEM, H100_SMS = 232448, 132
# out_store kinds (rv_conv2d_tc_out_store)
REGS, TMA_TILE, TMA_ROWS, VEC_ROWS = 0, 1, 2, 3
# the engine's upsample convs: (name, LR geometry)
UPSAMPLES = [('upsample1', (270, 480)), ('upsample1', (540, 960)), ('upsample2', (540, 960))]
# a budget whose rings fit but the TMA staging buffers do not (one A slot per consumer, 16-byte register stores)
SMALL_SMEM = 180 * 1024
DTYPES = ((torch.bfloat16, 'bf16'), (torch.float16, 'fp16'))


def test_ps_rows_order_puts_whole_hr_pixels_in_a_block():
    nb = 96
    order = packing.ps_rows_order(nb)
    assert sorted(order.tolist()) == list(range(2 * nb))
    c, a, b = order // 4, (order // 2) % 2, order % 2
    for blk in range(2):
        cols = slice(blk * nb, (blk + 1) * nb)
        assert (a[cols] == blk).all()
        assert sorted(zip(b[cols].tolist(), c[cols].tolist())) == [(bb, cc) for bb in range(2) for cc in range(nb // 2)]
        # lane q's column pairs j = 4g .. 4g + 3 (columns 8j + 2q, + 1) are 8 consecutive channels of one sub-pixel
        for g in range(nb // 32):
            for q in range(4):
                cols_q = [blk * nb + 8 * j + 2 * q + e for j in range(4 * g, 4 * g + 4) for e in range(2)]
                assert len({int(b[i]) for i in cols_q}) == 1
                cq = [int(c[i]) for i in cols_q]
                assert cq == list(range(cq[0], cq[0] + 8)) and cq[0] % 8 == 0


def _layer(name, dt, ps_rows=True, device='cpu', w=None, bias=None):
    sig = _sig(name)
    w = torch.zeros(sig.cout, 48, 3, 3) if w is None else w
    bias = torch.zeros(sig.cout) if bias is None else bias
    return packing.pack_conv_uncached(name, w, bias, list(sig.srcs), 1, sig.pad, dt, device, True, ps_rows=ps_rows)


def _plan(layer, dt, H, W, out_off=0, out_cs=48, max_smem=H100_SMEM):
    lib = load_library()
    base = 1 << 20
    d = rv_conv_desc()
    d.src0, d.c0, d.in_dtype, d.H, d.W = base, 48, DTYPE_CODE[dt], H, W
    d.wpack, d.bias, d.cout, d.kh, d.kw, d.stride, d.pad = base, base, 192, 3, 3, 1, 1
    d.out, d.out_cs, d.out_dtype = base + 2 * out_off, out_cs, DTYPE_CODE[dt]
    d.pixel_shuffle, d.impl, d.nb, d.k_real, d.layout = 1, layer.impl, layer.nb, layer.k_real, layer.layout
    d.ps_order = layer.ps_order
    plan, kind = (C.c_int32 * 8)(), C.c_int32(-1)
    rc = lib.rv_conv2d_tc_plan(C.byref(d), max_smem, H100_SMS, plan)
    if rc:
        return rc, lib.rv_last_error().decode(), None, None, d
    assert lib.rv_conv2d_tc_out_store(C.byref(d), max_smem, H100_SMS, C.byref(kind)) == 0, lib.rv_last_error()
    return rc, None, list(plan), kind.value, d


@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('case', UPSAMPLES, ids=[f'{n}-{g[0]}x{g[1]}' for n, g in UPSAMPLES])
def test_engine_upsample_plans_the_tma_row_store(case, dt):
    name, (H, W) = case
    layer = _layer(name, dt)
    assert (layer.nb, layer.layout, layer.ps_order) == (96, 1, 1)
    rc, err, plan, kind, _ = _plan(layer, dt, H, W)
    assert rc == 0, err
    assert kind == TMA_ROWS
    # 108 KB of resident weights, two 23 KB A slots and one 12 KB half-tile staging buffer per consumer
    assert plan[1] == 2 and plan[2] == 1 and plan[6] == 96
    assert plan[7] == 1024 + 9 * 96 * 128 + 2 * 2 * 23552 + 2 * 8 * 16 * 48 * 2 <= H100_SMEM - 1024
    # an output padded to 56 channels keeps 16-byte aligned pixel rows
    assert _plan(layer, dt, H, W, out_cs=56)[3] == TMA_ROWS
    # no room for the staging buffers: 16-byte stores from registers
    rc, err, plan, kind, _ = _plan(layer, dt, H, W, max_smem=SMALL_SMEM)
    assert rc == 0 and kind == VEC_ROWS and plan[1] == 1, (err, plan, kind)
    # the conv's own column order takes the general epilogue's 2-byte stores, also on an output 2 bytes off alignment
    for off in (0, 1):
        rc, err, plan, kind, _ = _plan(_layer(name, dt, ps_rows=False), dt, H, W, out_off=off)
        assert rc == 0 and kind == REGS, (err, kind)


def test_wrong_column_order_is_refused():
    dt = torch.bfloat16
    layer = _layer('upsample1', dt)
    lib = load_library()
    _, _, _, _, d = _plan(layer, dt, 270, 480)
    for field, value in (('pixel_shuffle', 0), ('cout', 96), ('nb', 48), ('ps_order', 2)):
        old = getattr(d, field)
        setattr(d, field, value)
        plan = (C.c_int32 * 8)()
        assert lib.rv_conv2d_tc_plan(C.byref(d), H100_SMEM, H100_SMS, plan) != 0, field
        assert b'ps_order' in lib.rv_last_error(), (field, lib.rv_last_error())
        setattr(d, field, old)
    # only the PSV kernel stores the order: an output 2 bytes off alignment, or a gate, is refused
    d.out += 2
    assert lib.rv_conv2d_tc_plan(C.byref(d), H100_SMEM, H100_SMS, plan) != 0 and b'ps_order' in lib.rv_last_error()
    d.out -= 2
    d.gate, d.gate_cs = d.out, 192
    assert lib.rv_conv2d_tc_plan(C.byref(d), H100_SMEM, H100_SMS, plan) != 0 and b'ps_order' in lib.rv_last_error()
    d.gate, d.gate_cs = None, 0
    # the CUDA-core conv has no column order of its own
    d.impl = 0
    assert lib.rv_conv2d(C.byref(d), None) != 0 and b'ps_order' in lib.rv_last_error()
    # convs the PSV kernel does not run are packed in their own order
    for cout, cin, k, layout in ((48, 48, 3, None), (128, 32, 3, None), (192, 48, 1, None), (192, 48, 3, 0)):
        w = torch.zeros(cout, cin, k, k)
        pc = packing.pack_conv_uncached('x', w, torch.zeros(cout), [(cin, cin)], 1, k // 2, dt, 'cpu', True, tc_layout=layout,
                                        ps_rows=True)
        assert pc.ps_order == 0, (cout, cin, k, layout)


class _PackOrders:
    """engine ops without a packer of their own, so that the engine packs its layers with packing.pack_conv, as it does for
    the CUDA ops; conv2d records each layer's column order, every other operator is a no-op"""
    def __init__(self):
        self.orders = {}

    def conv2d(self, layer, src0, src1, out, gate=None, res=None, act_pre=0, act_post=0, pixel_shuffle=False):
        self.orders[layer.name] = (layer.ps_order, bool(pixel_shuffle))

    def __getattr__(self, name):
        if name.startswith('__') or name == 'pack_conv':
            raise AttributeError(name)
        return lambda *a, **k: 0


@pytest.mark.parametrize('over', [dict(), dict(scale=2, matching_ksize=4)], ids=['x4', 'x2'])
def test_engine_packs_only_the_upsample_convs_in_hr_row_order(over):
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip, sliding_windows
    cfg = get_config('config_RefVSR_MFID', device='cpu', b200_precision='bf16', num_blocks=1, **over)
    net = SRNet(cfg).eval()
    seeded_test_weights(net, seed=5)
    ops = _PackOrders()
    net.Network.set_ops(ops)
    lrs, refs = make_clip(cfg.frame_num, 24, 32, 1, seed=5)
    for k, wl, wr, first in sliding_windows(lrs, refs, cfg.frame_num):
        net(wl, wr, first)
        break
    ups = {'upsample1.upsample_conv'} | ({'upsample2.upsample_conv'} if not over else set())
    assert {n for n, (_, ps) in ops.orders.items() if ps} == ups, ops.orders
    assert {n for n, (order, _) in ops.orders.items() if order} == ups, ops.orders


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
GPU_CASES = [('upsample1', (270, 480)), ('upsample1', (540, 960)), ('upsample2', (540, 960)), ('upsample1', (271, 483))]


@pytest.mark.gpu
@pytest.mark.parametrize('case', GPU_CASES, ids=[f'{n}-{g[0]}x{g[1]}' for n, g in GPU_CASES])
def test_store_paths_give_the_same_bits(cuda_ops, case):
    """the engine's packed layer (HR-row order) through the TMA row store at grid caps 0, 7 and 1 and through the 16-byte
    register stores (a shared-memory bound without room for the staging buffers), and the conv's own column order through
    the general epilogue (aligned and 2 bytes off): the same HR map, within test_conv_fp64's float64 bound, with the NaN
    guards around the output and in its channels >= cout intact"""
    name, (H, W) = case
    sig = _sig(name)
    ops = make_operands(sig, H, W, 'cuda', 1234 + H + W)
    ref, base = reference(sig, ops)
    Ho, Wo = out_hw(sig, H, W)
    ce, ocs = sig.cout // 4, 56
    n = Ho * Wo * ocs
    for dt, dtn in DTYPES:
        rows = _layer(name, dt, True, 'cuda', ops['w'], ops['b'])
        own = _layer(name, dt, False, 'cuda', ops['w'], ops['b'])
        assert rows.ps_order == 1 and own.ps_order == 0
        x = ops['xs'][0].to(dt)
        results = {}
        for tag, layer, cap, smem, off in (('tma cap0', rows, 0, 0, 0), ('tma cap7', rows, 7, 0, 0), ('tma cap1', rows, 1, 0, 0),
                                           ('vec16', rows, 0, SMALL_SMEM, 0), ('vec16 cap7', rows, 7, SMALL_SMEM, 0),
                                           ('own order', own, 0, 0, 0), ('own order offset 2B', own, 0, 0, 1)):
            buf = torch.full((n + 2 * GUARD + off,), float('nan'), dtype=dt, device='cuda')
            out = buf[GUARD + off:GUARD + off + n].view(Ho, Wo, ocs)
            old_cap, old_smem = cuda_ops.set_conv_cta_cap(cap), cuda_ops.set_conv_smem_cap(smem)
            try:
                cuda_ops.conv2d(layer, x, None, out, act_pre=sig.act_pre, act_post=sig.act_post, pixel_shuffle=True)
                torch.cuda.synchronize()
            finally:
                cuda_ops.set_conv_cta_cap(old_cap)
                cuda_ops.set_conv_smem_cap(old_smem)
            what = f'{name} {H}x{W} {dtn} {tag}'
            assert torch.isnan(buf[:GUARD + off]).all() and torch.isnan(buf[GUARD + off + n:]).all(), (what, 'wrote outside')
            assert torch.isnan(out[..., ce:]).all(), (what, 'wrote channels at or beyond cout')
            results[tag] = out[..., :ce].clone()
        check(results['tma cap0'], ref, base, dt, f'{name} {H}x{W} {dtn}', (16, 8), 96, True)
        for tag, y in results.items():
            assert torch.equal(y.view(torch.int16), results['tma cap0'].view(torch.int16)), (name, H, W, dtn, tag)


@pytest.mark.parametrize('srcs,cout,k,layout', [([(3, 8), (48, 48)], 48, 3, None), ([(48, 48)], 48, 1, None),
                                                 ([(16, 16)], 48, 3, 2), ([(48, 48)], 48, 3, 0)],
                         ids=['8+48-3x3', '48-48-1x1', '16-48-layout2', '48-48-layout0'])
def test_runtime_loop_convs_store_plain_tiles_by_tma(srcs, cout, k, layout):
    """the TMA tile store is not tied to the compile-time tap loop: runtime-loop convs up to NB = 48 with an aligned 16-bit
    output plan it too (rv_conv2d_tc_out_store 1), and an output 2 bytes off alignment keeps the register stores"""
    from refvsr_b200.lib import rv_conv_desc
    lib = load_library()
    dt = torch.bfloat16
    w = torch.zeros(cout, sum(r for r, _ in srcs), k, k)
    layer = packing.pack_conv_uncached('x', w, torch.zeros(cout), srcs, 1, k // 2, dt, 'cpu', True, tc_layout=layout)
    base = 1 << 20
    for off, want in ((0, TMA_TILE), (1, REGS)):
        d = rv_conv_desc()
        d.src0, d.src1 = base, (base if len(srcs) > 1 else None)
        d.c0, d.c1 = layer.alloc0, layer.alloc1
        d.in_dtype, d.H, d.W = DTYPE_CODE[dt], 270, 480
        d.wpack, d.bias, d.cout, d.kh, d.kw, d.stride, d.pad = base, base, cout, k, k, 1, k // 2
        d.out, d.out_cs, d.out_dtype = base + 2 * off, cout, DTYPE_CODE[dt]
        d.impl, d.nb, d.k_real, d.layout = layer.impl, layer.nb, layer.k_real, layer.layout
        kind = C.c_int32(-1)
        assert lib.rv_conv2d_tc_out_store(C.byref(d), H100_SMEM, H100_SMS, C.byref(kind)) == 0, lib.rv_last_error()
        assert kind.value == want, (srcs, cout, k, layout, off, kind.value)
