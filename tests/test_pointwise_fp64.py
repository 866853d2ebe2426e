"""Every sampling and pointwise operator the engine launches, checked element by element against a float64 reference at the
engine's shapes.

The reference is written from the model's semantics with torch's float64 primitives, not from the CPU operator set: grid_sample
(zeros, align_corners=False) on the linspace + flow / ((W - 1) / 2) grid for the warps, bilinear align_corners=True x 2 for the
up-sampled flow, grid_sample (border, align_corners=True) for SPyNet's level input, bicubic / bilinear F.interpolate for the
resizes and the reconstruction base, avg / max pooling, the ReflectionPad2d(1) + AlignedConv2d corner / clamp formula for
aligned_sample and reflect-padded, L2-normalised 3 x 3 patches x 64 for patch_pack.

The bound.  Operands are exact in bf16 and fp16 (maps k / 128, affine maps multiples of 1 / 64), so the kernels'
fp32 arithmetic works on exact inputs and rounds once to the output type (flows are fp32 operands in every precision).  Every output element y then satisfies

    |y - ref| <= ulp_T(ref) (16-bit outputs only) + C_AR * u * A + L * delta

  * u = 2^-24; A the float64 magnitude the fp32 arithmetic works on: sum |w_i x_i| over the taps the output blends (for the
    bicubic operators 2.25 max|x| + |ref|, which also covers the fp32 evaluation of the cubic weights); C_AR bounds the number
    of fp32 operations between the exact inputs and the rounded value, each erring by at most u of the magnitude it works on.
  * delta: the fp32 error of the sampling coordinate, derived from its expression.  For the warp grid
    px = ((lin + f / ((W - 1) / 2) + 1) W - 1) / 2 every operation errs by at most u of its operand, which sums to
    u (W / 2 + 1) (10 + 5 |g|) pixels (g the float64 grid value); the up-sampled flow adds 2 (2 |f|max 2u s + 6 u A_f) (its
    align_corners scale (n - 1) / (2n - 1) is inexact); the other resampling operators are derived the same way.
  * L: a slope bound of the output against its coordinate - the largest difference between the taps the element blends, or
    twice the map's largest magnitude where the coordinate is within delta of a cell edge, where the kernel may blend the
    neighbouring cell's taps.

Exact operators (gather_blocks, space_to_depth2, maxpool2, nearest resize_planes, conf_max) must match bit for bit.
aligned_sample's clamped corners make it discontinuous where a padded coordinate crosses 0 or Hp - 1: there the reference is
also evaluated at p +- delta and either side is accepted (the number of such elements is printed).  8-bit outputs must equal
round(clamp(ref) * 255) except within the bound of a .5 boundary, where either neighbour is accepted.

patch_pack writes each patch value v = 64 x / max(|patch|, 1e-12) as hi = fp16(v32) and, for the split modes the fp32 engine
uses, lo = fp16(v32 - hi), where v32 is the kernel's fp32 value.  |patch|^2 is a sum of K = 9 C non-negative fp32 squares (K
roundings and K - 1 additions, each within u of the partial sum: K u of |patch|^2), its square root halves that and adds u, the
division adds u and x 64 is exact, so |v32 - v| <= (K / 2 + 3) u |v| <= (K + C_AR) u |v|.  v32 - hi is exact in fp32 and lo is
its fp16 rounding, so

    |hi - v| <= ulp_fp16(v),    |hi + lo - v| <= ulp_fp16(v - hi) + (K + C_AR) u |v|,

with the arithmetic term added to - not multiplied by - the operation count: about 2^-16 |v| for K = 144, well below fp16's own
precision, so a missing, doubled or twice-rounded lo half fails.  Padding columns must be exactly zero.

C_AR = 64 is chosen once from this derivation (the longest chain, a bicubic tap sum with its weights, has about 30 operations)
and not tuned per case.  It is tight enough that a half-pixel shift, two swapped corner weights, the wrong padding mode, a
missing x 2 on the up-sampled flow, the wrong cubic coefficient, a second rounding of an fp32 output or the wrong image stride
in a batch fail (the CPU self-tests below plant each of them into a fake kernel).

Without a GPU: those self-tests, and the list of operator calls below against what the engine launches.  With a GPU: every
(signature, geometry) of the list in bf16 and fp16 (and fp32 where the fp32 engine launches it), plus cases named for the
kernel branch they force: batched, ragged tiles and misaligned outputs."""
import collections
import inspect
import re
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_conv_fp64 import ulp

U = 2.0 ** -24
C_AR = 64.0
GUARD = 4096

# ------------------------------------------------------------------------------------------------------------------
# the list: every non-conv, non-GEMM operator call of the engine
# ------------------------------------------------------------------------------------------------------------------
# A signature: operator, dtype of its activation-typed operand ('act': the engine's precision; 'fp32': always fp32), real and
# allocated channels, and flags.  Each entry also names the engine precisions that launch it ('16': bf16 / fp16, '32': fp32)
# and the input geometries of the x4 (LR 270x480) and x2 (LR 540x960) schedules:
#   warp: flow (h, w); spynet_resize_norm / flow_resize / resize_planes: input (H, W) + output (H, W); gather_blocks:
#   value (H, W) + cells (hq, wq); aligned_sample: affine cells (h, w); reconstruct*: LR (h, w); the others: input (H, W).
# Signatures only flag_HD_in launches (ks 8, nearest x0.5, bicubic x4 of the relevance map) run at the geometries of an
# HD model at LR 272x480.  test_engine_signatures_are_all_listed / test_engine_geometries_are_all_listed keep this complete.
Sig = collections.namedtuple('Sig', 'op dt real alloc flags')
Entry = collections.namedtuple('Entry', 'sig precs geoms')


def P(op, dt, real, alloc, precs, geoms, **flags):
    return Entry(Sig(op, dt, real, alloc, tuple(sorted(flags.items()))), precs, tuple(geoms))


X4, X2 = (270, 480), (540, 960)
LEVELS = [(18, 30), (36, 60), (72, 120), (144, 240), (288, 480), (34, 60), (68, 120), (136, 240), (272, 480), (544, 960)]
ENGINE_POINTWISE = [
    P('warp3', 'act', 48, 48, '16', [X4, X2]),
    P('warp', 'act', 48, 48, '16+32', [X4, X2], flow_up2=False, src_scale=1),
    P('warp', 'act', 48, 48, '16+32', [X4, X2], flow_up2=True, src_scale=1),      # the quirk: the LR feature onto the 2x grid
    P('warp', 'act', 48, 48, '32', [X4, X2], flow_up2=True, src_scale=2),
    P('warp', 'fp32', 1, 1, '16+32', [X4, X2], flow_up2=False, src_scale=1),
    P('spynet_resize_norm', 'fp32', 3, 3, '16+32', [(270, 480, 288, 480), (540, 960, 544, 960)]),
    P('avgpool2', 'fp32', 3, 3, '16+32', LEVELS),
    P('spynet_level_input', 'act', 8, 8, '16+32', [(9, 15), (17, 30)], flow_prev=False),
    P('spynet_level_input', 'act', 8, 8, '16+32', LEVELS, flow_prev=True),
    P('flow_resize', 'fp32', 2, 2, '16+32', [(288, 480, 270, 480), (544, 960, 540, 960)]),
    P('prep_image', 'act', 3, 8, '16+32', [X4, X2], mat=False, pool2=False),
    P('prep_image', 'act', 3, 8, '16+32', [X4, X2], mat=True, pool2=False),
    P('prep_image', 'act', 3, 8, '16+32', [X4, X2], mat=True, pool2=True),
    P('maxpool2', 'act', 64, 64, '16+32', [X4, X2]),
    P('resize_planes', 'fp32', 1, 1, '16+32', [(270, 480, 540, 960)], clamp01=True, inv_scale=0.5, mode='bicubic'),
    P('resize_planes', 'fp32', 3, 3, '16+32', [(540, 960, 270, 480)], clamp01=True, inv_scale=2.0, mode='bicubic'),
    P('resize_planes', 'fp32', 1, 1, '16+32', [(68, 120, 272, 480)], clamp01=True, inv_scale=0.25, mode='bicubic'),
    P('resize_planes', 'fp32', 3, 3, '16+32', [(272, 480, 136, 240)], clamp01=False, inv_scale=2.0, mode='nearest'),
    P('patch_pack', 'act', 16, 144, '16', [(135, 240), (270, 480)], mode=0),
    P('patch_pack', 'act', 16, 432, '32', [(270, 480)], mode=1),
    P('patch_pack', 'act', 16, 432, '32', [(135, 240)], mode=2),
    P('gather_blocks', 'act', 48, 48, '16+32', [(135, 240, 270, 480)], ks=1),
    P('gather_blocks', 'act', 48, 48, '16+32', [(270, 480, 270, 480)], ks=2),
    P('gather_blocks', 'act', 48, 48, '16+32', [(540, 960, 270, 480)], ks=4),
    P('gather_blocks', 'act', 48, 48, '16+32', [(544, 960, 68, 120)], ks=8),
    P('gather_blocks', 'act', 8, 8, '16+32', [(270, 480, 270, 480), (540, 960, 270, 480)], ks=2),
    P('gather_blocks', 'act', 8, 8, '16+32', [(540, 960, 270, 480)], ks=4),
    P('gather_blocks', 'act', 8, 8, '16+32', [(544, 960, 68, 120)], ks=8),
    P('space_to_depth2', 'act', 48, 48, '16', [X4, X2]),
    P('space_to_depth2', 'act', 32, 32, '16', [X2]),
    P('bicubic_up2_image', 'act', 3, 8, '16+32', [X4, X2]),
    P('aligned_sample', 'act', 48, 48, '16+32', [X4], ks=2),
    P('aligned_sample', 'act', 48, 48, '16+32', [X4], ks=4),
    P('aligned_sample', 'act', 48, 48, '16+32', [(68, 120)], ks=8),
    P('conf_pair', 'act', 2, 8, '16+32', [X4, X2], up2=False),
    P('conf_pair', 'act', 2, 8, '16+32', [X4, X2], up2=True),
    P('conf_max', 'fp32', 1, 1, '16+32', [X4, X2]),
    P('reconstruct', 'fp32', 3, 4, '16+32', [X4], clamp01=True, scale=4),
    P('reconstruct', 'fp32', 3, 4, '16+32', [X2], clamp01=True, scale=2),
    P('reconstruct_u8', 'fp32', 3, 4, '16+32', [X4], bgr=True, clamp01=True, scale=4),
    P('reconstruct_u8', 'fp32', 3, 4, '16+32', [X2], bgr=False, clamp01=True, scale=2),
]
DTN = {torch.float32: 'fp32', torch.float16: 'fp16', torch.bfloat16: 'bf16'}
DT = {v: k for k, v in DTN.items()}
POINTWISE_OPS = ('warp', 'warp3', 'spynet_resize_norm', 'avgpool2', 'spynet_level_input', 'flow_resize', 'prep_image', 'maxpool2',
                 'resize_planes', 'patch_pack', 'gather_blocks', 'space_to_depth2', 'bicubic_up2_image', 'aligned_sample', 'conf_pair',
                 'conf_max', 'reconstruct', 'reconstruct_u8')
# the other operators the engine calls: the convs (test_conv_fp64.py), the matching GEMM (test_match_fp64.py), the reuse guard
# (test_frames_differ.py) and the 8-bit input conversion (test_gpu_u8_frames.py)
ELSEWHERE = {'conv2d', 'pack_conv', 'match_argmax', 'frames_differ', 'frames_from_u8', 'launch_count'}


def _expand(entries, prec):
    """the concrete signatures an engine at precision `prec` ('bf16' | 'fp32') launches according to the list"""
    want = '16' if prec != 'fp32' else '32'
    return {e.sig._replace(dt=prec if e.sig.dt == 'act' else 'fp32') for e in entries if want in e.precs}


# ------------------------------------------------------------------------------------------------------------------
# CPU: the list above is what the engine launches
# ------------------------------------------------------------------------------------------------------------------
def _bind(op, a, k):
    from u8_ops import U8OracleOps
    b = inspect.signature(getattr(U8OracleOps, op)).bind(None, *a, **k)
    b.apply_defaults()
    return b.arguments


def _signature(op, a, k):
    """(Sig, geometry) of one operator call, in the engine's dtypes"""
    v = _bind(op, a, k)
    f = {}
    if op == 'warp':
        src, flow = v['src'], v['flow']
        c = src.shape[2] if src.dim() == 3 else 1
        f = dict(flow_up2=bool(v['flow_up2']), src_scale=src.shape[0] // flow.shape[0])
        return Sig(op, DTN[src.dtype], c, c, tuple(sorted(f.items()))), tuple(flow.shape[:2])
    if op == 'warp3':
        t = v['feat']
        return Sig(op, DTN[t.dtype], t.shape[2], t.shape[2], ()), tuple(t.shape[:2])
    if op == 'spynet_resize_norm':
        return Sig(op, 'fp32', 3, 3, ()), tuple(v['src'].shape[1:]) + tuple(v['out'].shape[:2])
    if op in ('avgpool2', 'maxpool2', 'space_to_depth2'):
        t = v['src']
        return Sig(op, DTN[t.dtype], t.shape[2], t.shape[2], ()), tuple(t.shape[:2])
    if op == 'spynet_level_input':
        return (Sig(op, DTN[v['out8'].dtype], 8, 8, (('flow_prev', v['flow_prev'] is not None),)),
                tuple(v['ref'].shape[:2]))
    if op == 'flow_resize':
        return Sig(op, 'fp32', 2, 2, ()), tuple(v['flow'].shape[:2]) + tuple(v['out'].shape[:2])
    if op == 'prep_image':
        o = v['out']
        f = dict(mat=v['mat12'] is not None, pool2=bool(v['pool2']))
        return Sig(op, DTN[o.dtype], 3, o.shape[2], tuple(sorted(f.items()))), tuple(v['src'].shape[1:])
    if op == 'resize_planes':
        s, o = v['src'], v['out']
        f = dict(mode=v['mode'], clamp01=bool(v['clamp01']), inv_scale=float(v['inv_scale']))
        return Sig(op, 'fp32', s.shape[0], s.shape[0], tuple(sorted(f.items()))), tuple(s.shape[1:]) + tuple(o.shape[1:])
    if op == 'patch_pack':
        t = v['feat']
        return Sig(op, DTN[t.dtype], t.shape[2], v['out'].shape[1], (('mode', v['mode']),)), tuple(t.shape[:2])
    if op == 'gather_blocks':
        t = v['value']
        return Sig(op, DTN[t.dtype], t.shape[2], t.shape[2], (('ks', v['ks']),)), tuple(t.shape[:2]) + (v['hq'], v['wq'])
    if op == 'bicubic_up2_image':
        o = v['out']
        return Sig(op, DTN[o.dtype], 3, o.shape[2], ()), tuple(v['src'].shape[1:])
    if op == 'aligned_sample':
        t = v['x']
        return Sig(op, DTN[t.dtype], t.shape[2], t.shape[2], (('ks', v['ks']),)), tuple(v['affine'].shape[:2])
    if op == 'conf_pair':
        o = v['out']
        return Sig(op, DTN[o.dtype], 2, o.shape[2], (('up2', bool(v['up2'])),)), tuple(v['a'].shape)
    if op == 'conf_max':
        return Sig(op, 'fp32', 1, 1, ()), tuple(v['a'].shape)
    if op in ('reconstruct', 'reconstruct_u8'):
        x = v['x']
        f = dict(scale=v['scale'], clamp01=bool(v['clamp01']))
        if op == 'reconstruct_u8':
            f['bgr'] = bool(v['bgr'])
        return Sig(op, DTN[x.dtype], 3, x.shape[2], tuple(sorted(f.items()))), tuple(v['lr'].shape[1:])
    raise AssertionError(op)


def _recording_ops(compute):
    """the CPU operator set (OracleOps and the 8-bit pair) recording (Sig, geometry) of every in-scope operator call and the name of
    every operator the engine looks up; compute=False: every operator is a no-op, so that a full-size schedule runs in seconds"""
    from u8_ops import U8OracleOps

    class Recording(U8OracleOps):
        def __init__(self):
            self.seen, self.called, self.depth = collections.Counter(), set(), 0

        def __getattribute__(self, name):
            attr = object.__getattribute__(self, name)
            if name.startswith('_') or name in ('seen', 'called', 'depth') or not callable(attr):
                return attr
            object.__getattribute__(self, 'called').add(name)
            if name in POINTWISE_OPS:
                def rec(*a, **k):
                    if self.depth == 0:                   # (OracleOps.warp3 is three OracleOps.warp calls: not the engine's)
                        self.seen[_signature(name, a, k)] += 1
                    if compute:
                        self.depth += 1
                        try:
                            return attr(*a, **k)
                        finally:
                            self.depth -= 1
                return rec
            if not compute and name != 'pack_conv':
                return lambda *a, **k: 0
            return attr
    return Recording()


def _run_engine(ops, h, w, prec, cfg_name='config_RefVSR_MFID', u8=None, ref_scale=1, **over):
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip, sliding_windows
    cfg = get_config(cfg_name, device='cpu', b200_precision=prec, **over)
    net = SRNet(cfg).eval()
    seeded_test_weights(net, seed=5)
    net.Network.set_ops(ops)
    lrs, refs = make_clip(cfg.frame_num, h, w, ref_scale, seed=5)
    with torch.no_grad():
        for n, (k, wl, wr, first) in enumerate(sliding_windows(lrs, refs, cfg.frame_num)):
            if u8 is None:
                net(wl, wr, first)
            else:
                q = lambda x: (x[0].clamp(0, 1) * 255).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous().unsqueeze(0)
                net.Network.forward_u8(q(wl), q(wr), first, bgr=u8)
            if n == 1:
                break
    return ops


_X2_MODEL = dict(scale=2, matching_ksize=4)


def _signature_runs():
    """{(Sig, precision)} of small x4, x2 and flag_HD_in models at bf16 and fp32 (OracleOps computes), fp32 / 8-bit output"""
    seen, called = set(), set()
    for prec in ('bf16', 'fp32'):
        runs = [dict(), dict(**_X2_MODEL), dict(cfg_name='config_RefVSR_MFID_8K', h=32, w=48),
                dict(u8=True), dict(u8=False, **_X2_MODEL)]
        for r in runs:
            r = dict(r)
            h, w = r.pop('h', 24), r.pop('w', 32)
            ops = _run_engine(_recording_ops(True), h, w, prec, num_blocks=1, **r)
            seen |= {(s, prec) for s, _ in ops.seen}
            called |= ops.called
    return seen, called


def _geometry_runs():
    """{precision: {(Sig, geometry)}} of the full-size x4 (LR 270x480) and x2 (LR 540x960) schedules, shapes only"""
    seen = collections.defaultdict(set)
    for h, w, over in ((270, 480, {}), (540, 960, _X2_MODEL)):
        for prec in ('bf16', 'fp32'):
            seen[prec] |= set(_run_engine(_recording_ops(False), h, w, prec, **over).seen)
    return seen


def test_engine_signatures_are_all_listed():
    """small x4, x2 and flag_HD_in models at bf16 and fp32, with fp32 and 8-bit output (OracleOps computes; the first window
    takes the quirk path's three warp calls): every in-scope operator call's signature is listed, every listed signature is
    launched, and the engine calls no operator outside the list and ELSEWHERE"""
    seen, called = _signature_runs()
    for prec in ('bf16', 'fp32'):
        got = {s for s, p in seen if p == prec}
        listed = _expand(ENGINE_POINTWISE, prec)
        assert not got - listed, f'{prec}: signatures the engine launches and ENGINE_POINTWISE does not list: {sorted(got - listed)}'
        assert not listed - got, f'{prec}: listed signatures the engine does not launch: {sorted(listed - got)}'
    assert called - ELSEWHERE == set(POINTWISE_OPS), f'operators outside the list: {sorted(called - ELSEWHERE - set(POINTWISE_OPS))}'
    assert {e.sig.op for e in ENGINE_POINTWISE} == set(POINTWISE_OPS)


def test_engine_geometries_are_all_listed():
    """the full-size x4 (LR 270x480) and x2 (LR 540x960) schedules at bf16 and fp32, shapes only: every (signature, geometry)
    they launch is a case of test_engine_pointwise"""
    for prec, seen in _geometry_runs().items():
        listed = {(e.sig._replace(dt=prec if e.sig.dt == 'act' else 'fp32'), g) for e in ENGINE_POINTWISE
                  if ('16' if prec != 'fp32' else '32') in e.precs for g in e.geoms}
        missing = seen - listed
        assert not missing, f'{prec}: (signature, geometry) pairs the engine launches and ENGINE_POINTWISE does not list: {sorted(missing)}'


# ------------------------------------------------------------------------------------------------------------------
# the float64 reference
# ------------------------------------------------------------------------------------------------------------------
def _nchw(t):
    """(H, W, C) or (H, W) -> (1, C, H, W) float64"""
    t = t.double()
    return (t.unsqueeze(-1) if t.dim() == 2 else t).permute(2, 0, 1).unsqueeze(0)


def _hwc(t):
    return t[0].permute(1, 2, 0)


def _lin(n, dev):
    return torch.linspace(-1.0, 1.0, n, dtype=torch.float64, device=dev)


def _taps(X, x0, y0, border):
    """the four bilinear taps nw, ne, sw, se of X (1, C, H, W) at integer corners (x0, y0) (Ho, Wo): zero outside the map
    (zeros padding) or clamped (border)"""
    _, C, H, W = X.shape
    out = []
    for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
        xi, yi = x0 + dx, y0 + dy
        ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
        idx = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)).view(1, 1, -1).expand(1, C, -1)
        v = X.reshape(1, C, H * W).gather(2, idx).view(1, C, *x0.shape)
        out.append(v if border else v * ok)
    return out


def _slope(X, px, py, border, dx, dy):
    """L_x delta_x + L_y delta_y: the local tap differences, or 2 max|X| where the coordinate is within delta of a cell edge"""
    x0, y0 = px.floor(), py.floor()
    nw, ne, sw, se = _taps(X, x0.long(), y0.long(), border)
    lx = torch.maximum((ne - nw).abs(), (se - sw).abs())
    ly = torch.maximum((sw - nw).abs(), (se - ne).abs())
    g = 2 * float(X.abs().max())
    fx, fy = px - x0, py - y0
    lx = torch.where(((fx <= dx) | (fx >= 1 - dx)), torch.full_like(lx, g), lx)
    ly = torch.where(((fy <= dy) | (fy >= 1 - dy)), torch.full_like(ly, g), ly)
    return lx * dx + ly * dy


def _up2_flow(flow):
    """F.interpolate(x 2, bilinear, align_corners=True) * 2 of an (h, w, 2) flow -> (1, 2, 2h, 2w) float64, and the fp32
    error bound of a kernel's evaluation of it (coordinate s = X (n - 1) / (2n - 1) with an inexact scale, 4-tap blend, x 2)"""
    f = _nchw(flow)
    up = F.interpolate(f, scale_factor=2, mode='bilinear', align_corners=True) * 2
    a = F.interpolate(f.abs(), scale_factor=2, mode='bilinear', align_corners=True) * 2
    h, w = flow.shape[:2]
    dev = flow.device
    sy = torch.arange(2 * h, dtype=torch.float64, device=dev).view(-1, 1) * ((h - 1) / max(2 * h - 1, 1))
    sx = torch.arange(2 * w, dtype=torch.float64, device=dev).view(1, -1) * ((w - 1) / max(2 * w - 1, 1))
    fmax = float(f.abs().max())
    err = 2 * (2 * fmax * 2 * U * (sy + sx)) + 6 * U * a
    return up, err


def ref_warp(src, flow, up2):
    """models/utils.py warp: grid_sample(bilinear, zeros, align_corners=False) on linspace + flow / ((W - 1) / 2).  Returns the
    output (Ho, Wo, C) and the bound without the output type's ulp"""
    X = _nchw(src)
    _, _, Hi, Wi = X.shape
    dev = src.device
    if up2:
        f, ef = _up2_flow(flow)
        efx, efy = ef[0, 0], ef[0, 1]
    else:
        f, efx, efy = _nchw(flow), 0.0, 0.0
    Ho, Wo = f.shape[-2:]
    gx = _lin(Wo, dev).view(1, Wo) + f[0, 0] / ((Wi - 1) / 2)
    gy = _lin(Ho, dev).view(Ho, 1) + f[0, 1] / ((Hi - 1) / 2)
    grid = torch.stack([gx, gy], -1).unsqueeze(0)
    ref = F.grid_sample(X, grid, mode='bilinear', padding_mode='zeros', align_corners=False)
    A = F.grid_sample(X.abs(), grid, mode='bilinear', padding_mode='zeros', align_corners=False)
    px, py = ((gx + 1) * Wi - 1) / 2, ((gy + 1) * Hi - 1) / 2
    dx = U * (Wi / 2 + 1) * (10 + 5 * gx.abs()) + efx
    dy = U * (Hi / 2 + 1) * (10 + 5 * gy.abs()) + efy
    base = C_AR * U * A + _slope(X, px, py, False, dx, dy)
    return _hwc(ref), _hwc(base)


def ref_level_input(ref_img, supp, flow_prev):
    """SPyNet level input: [ref, flow_warp(supp, flow_up, border, align_corners=True), flow_up] and flow_up"""
    H, W = ref_img.shape[:2]
    dev = ref_img.device
    if flow_prev is None:
        fu, ef = torch.zeros(1, 2, H, W, dtype=torch.float64, device=dev), torch.zeros(1, 2, H, W, dtype=torch.float64, device=dev)
    else:
        fu, ef = _up2_flow(flow_prev)
    X = _nchw(supp)
    xs = torch.arange(W, dtype=torch.float64, device=dev).view(1, W)
    ys = torch.arange(H, dtype=torch.float64, device=dev).view(H, 1)
    gx = 2 * (xs + fu[0, 0]) / max(W - 1, 1) - 1
    gy = 2 * (ys + fu[0, 1]) / max(H - 1, 1) - 1
    grid = torch.stack([gx, gy], -1).unsqueeze(0)
    wv = F.grid_sample(X, grid, mode='bilinear', padding_mode='border', align_corners=True)
    A = F.grid_sample(X.abs(), grid, mode='bilinear', padding_mode='border', align_corners=True)
    px = ((gx + 1) / 2 * (W - 1)).clamp(0, W - 1)
    py = ((gy + 1) / 2 * (H - 1)).clamp(0, H - 1)
    dx = U * (W / 2 + 1) * (8 + 4 * gx.abs()) + ef[0, 0]
    dy = U * (H / 2 + 1) * (8 + 4 * gy.abs()) + ef[0, 1]
    bw = C_AR * U * A + _slope(X, px, py, True, dx, dy)
    out = torch.cat([_nchw(ref_img), wv, fu], 1)
    base = torch.cat([torch.zeros_like(_nchw(ref_img)), bw, ef], 1)
    return _hwc(out), _hwc(base), _hwc(fu), _hwc(ef)


def ref_bilinear(x, size, mul=None):
    """F.interpolate(bilinear, align_corners=False) of (1, C, H, W) float64 to `size` (x mul per channel); the bound covers the
    fp32 source coordinate s = fl(H / Ho) (Y + 0.5) - 0.5 and the blend"""
    y = F.interpolate(x, size=size, mode='bilinear', align_corners=False)
    a = F.interpolate(x.abs(), size=size, mode='bilinear', align_corners=False)
    H, W = x.shape[-2:]
    dev = x.device
    sy = (torch.arange(size[0], dtype=torch.float64, device=dev).view(-1, 1) + 0.5) * (H / size[0])
    sx = (torch.arange(size[1], dtype=torch.float64, device=dev).view(1, -1) + 0.5) * (W / size[1])
    L = 2 * float(x.abs().max())
    base = C_AR * U * a + L * 4 * U * (sy + sx + 2)
    if mul is not None:
        m = torch.tensor(mul, dtype=torch.float64, device=dev).view(1, -1, 1, 1)
        y, base = y * m, base * m.abs() + 2 * U * (y * m).abs()
    return y, base


def bicubic(x, scale):
    """F.interpolate(bicubic, align_corners=False, scale_factor) of (1, C, H, W) float64 and its bound without the output ulp"""
    y = F.interpolate(x, scale_factor=scale, mode='bicubic', align_corners=False)
    return y, C_AR * U * (2.25 * x.abs().amax(dim=(2, 3), keepdim=True) + y.abs())


def ref_aligned(x, aff, ks, dr=0.0, dc=0.0):
    """AlignedConv2d sampling (alignment.py): ReflectionPad2d(1) of x (ks h, ks w, C); per cell and offset (a, b) the position
    p = R(theta) ((a - half) s_x, (b - half) s_y) + half + 1 + ks (i, j), its floor / floor + 1 corners and p itself clamped
    to the padded map, weights from the clamped values.  (dr, dc): offsets added to p.  Returns ref, A, p_r, p_c, max|x|."""
    H, W, C = x.shape
    h, w = aff.shape[:2]
    Hp, Wp = H + 2, W + 2
    dev = x.device
    xp = F.pad(_nchw(x), (1, 1, 1, 1), mode='reflect')
    a = aff.double()
    half = (ks - 1) // 2 + 0.5
    o = torch.arange(ks, dtype=torch.float64, device=dev) - half
    u = o.view(1, 1, ks, 1) * a[..., 0, None, None]
    v = o.view(1, 1, 1, ks) * a[..., 1, None, None]
    th = ((a[..., 2] - 1) * 1.0472)[..., None, None]
    rr, cc = u * th.cos() - v * th.sin(), u * th.sin() + v * th.cos()
    i = torch.arange(h, dtype=torch.float64, device=dev).view(h, 1, 1, 1)
    j = torch.arange(w, dtype=torch.float64, device=dev).view(1, w, 1, 1)
    pr = (rr + half + 1 + ks * i).permute(0, 2, 1, 3).reshape(H, W) + dr
    pc = (cc + half + 1 + ks * j).permute(0, 2, 1, 3).reshape(H, W) + dc
    ltr, ltc = pr.floor(), pc.floor()
    rbr, rbc = (ltr + 1).clamp(0, Hp - 1), (ltc + 1).clamp(0, Wp - 1)
    ltr, ltc = ltr.clamp(0, Hp - 1), ltc.clamp(0, Wp - 1)
    qr, qc = pr.clamp(0, Hp - 1), pc.clamp(0, Wp - 1)
    g = [(1 + (ltr - qr)) * (1 + (ltc - qc)), (1 - (rbr - qr)) * (1 - (rbc - qc)),
         (1 + (ltr - qr)) * (1 - (rbc - qc)), (1 - (rbr - qr)) * (1 + (ltc - qc))]
    flat = xp.reshape(C, Hp * Wp)
    ref = torch.zeros(C, H, W, dtype=torch.float64, device=dev)
    A = torch.zeros_like(ref)
    for gi, (r, c) in zip(g, ((ltr, ltc), (rbr, rbc), (ltr, rbc), (rbr, ltc))):
        t = flat[:, (r * Wp + c).long().view(-1)].view(C, H, W)
        ref += gi * t
        A += (gi * t).abs()
    return ref.permute(1, 2, 0), A.permute(1, 2, 0), pr, pc, aff


def aligned_delta(pr, pc, aff, ks, H, W):
    """the fp32 error of the kernel's padded coordinates: the rotation of offsets up to |u| + |v| with cos / sin of an fp32 angle,
    then the additions of half, 1 and ks * i"""
    h, w = aff.shape[:2]
    a = aff.double()
    half = (ks - 1) // 2 + 0.5
    m = (half * (a[..., 0].abs() + a[..., 1].abs()) * (1 + ((a[..., 2] - 1) * 1.0472).abs()))
    m = m.repeat_interleave(ks, 0).repeat_interleave(ks, 1)
    return 4 * U * m + 2 * U * (pr.abs() + 1), 4 * U * m + 2 * U * (pc.abs() + 1)


def ref_patches(feat):
    """reflect-padded 3 x 3 patches of (H, W, C) (channel-major, c * 9 + ky * 3 + kx), L2-normalised, x 64 -> (H W, 9 C)"""
    p = F.unfold(F.pad(_nchw(feat), (1, 1, 1, 1), mode='reflect'), kernel_size=3)[0].t()
    return p / p.norm(dim=1, keepdim=True).clamp(min=1e-12) * 64


# ------------------------------------------------------------------------------------------------------------------
# checks
# ------------------------------------------------------------------------------------------------------------------
def check(y, ref, base, dtype, what, tile=(16, 16), alt=None):
    """|y - ref| <= ulp_dtype(ref) (16-bit) + base element by element on (H, W, C) views, y finite wherever ref is.  alt: (mask,
    [refs]) - where mask is set, any of refs is also accepted (aligned_sample's either-side rule).  Prints the largest
    |y - ref| / bound; a failure names where the failing elements sit within their tiles.  Returns (worst, either-side count)."""
    y = y.double()
    bnd = base if dtype == torch.float32 else base + ulp(ref, dtype)
    fin = torch.isfinite(ref)
    bad_fin = fin & ~torch.isfinite(y)
    err = (y - ref).abs()
    ratio = torch.where(fin & (err > 0), err / bnd, torch.zeros_like(ref))
    either = 0
    if alt is not None:
        mask, refs = alt
        best = ratio
        for r in refs:
            e = (y - r).abs()
            best = torch.minimum(best, torch.where(mask, torch.where(e > 0, e / bnd, torch.zeros_like(e)), best))
        either = int(((ratio > 1) & (best <= 1)).sum())
        ratio = best
    worst = float(ratio.max()) if ratio.numel() else 0.0
    print(f'[pointwise_fp64] {what}: max |y - ref| / bound = {worst:.4f}' + (f', either-side elements {either}' if alt else ''))
    if bad_fin.any() or not worst <= 1.0:
        pytest.fail(_explain(y, ref, ratio, bad_fin, what, tile))
    return worst, either


def check_exact(y, ref, what, tile=(16, 16)):
    same = (y == ref) | (torch.isnan(y.double()) & torch.isnan(ref.double()))
    print(f'[pointwise_fp64] {what}: bit-exact {bool(same.all())}')
    if not same.all():
        d = (y.double() - ref.double()).abs()
        bad_fin = torch.isfinite(ref.double()) & ~torch.isfinite(y.double())
        pytest.fail(_explain(y.double(), ref.double(), torch.where(same | bad_fin, torch.zeros_like(d), d + 2), bad_fin,
                             what + ' (exact)', tile))
    return 0.0, 0


def _explain(y, ref, ratio, bad_fin, what, tile):
    bad = (ratio > 1.0) | bad_fin | torch.isnan(ratio)
    idx = bad.nonzero()
    i = int(torch.nan_to_num(ratio, nan=1e30).flatten().argmax())
    yy, xx, c = [int(v) for v in torch.unravel_index(torch.tensor(i), ratio.shape)]
    th, tw = tile
    msg = [f'{what}: {idx.shape[0]} of {ratio.numel()} elements outside the bound ({int(bad_fin.sum())} non-finite)',
           f'worst at ({yy}, {xx}, channel {c}): y = {float(y[yy, xx, c])!r}, ref = {float(ref[yy, xx, c])!r}, '
           f'{float(ratio[yy, xx, c]):.3g} x bound',
           f'within its {th} x {tw} tile: y % {th} = {yy % th}, x % {tw} = {xx % tw}; tile ({yy // th}, {xx // tw})']
    if idx.shape[0]:
        for label, v in (('channels', idx[:, 2]), (f'y % {th}', idx[:, 0] % th), (f'x % {tw}', idx[:, 1] % tw),
                         ('image rows', idx[:, 0]), ('image columns', idx[:, 1])):
            u, cnt = torch.unique(v, return_counts=True)
            top = cnt.argsort(descending=True)[:8]
            msg.append(f'  failing elements by {label}: ' + ', '.join(f'{int(u[j])}: {int(cnt[j])}' for j in top))
    return '\n'.join(msg)


def check_u8(y, v, base, what, tile=(16, 16)):
    """y: uint8 bytes of the float64 values v (same layout); round(clamp(v) * 255) except within base (in v units, plus the fp32
    product's rounding) of a .5 boundary, where either neighbour is accepted.  The ratio printed and returned is
    |y - clamp(255 v)| / (0.5 + e), e the bound in byte units: at most 1 for every accepted byte."""
    s = v * 255
    e = base * 255 + 255 * U * (v.abs() + 1)
    lo = (s - e).clamp(0, 255).round()
    hi = (s + e).clamp(0, 255).round()
    yd = y.double()
    ok = (yd >= lo) & (yd <= hi)
    either = int((ok & (yd != s.clamp(0, 255).round())).sum())
    ratio = (yd - s.clamp(0, 255)).abs() / (0.5 + e)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    print(f'[pointwise_fp64] {what}: 8-bit, max |y - 255 ref| / (0.5 + bound) = {worst:.4f}, {int((~ok).sum())} outside, '
          f'{either} took the neighbour of a .5 boundary')
    if not ok.all():
        pytest.fail(_explain(yd, s.clamp(0, 255).round(), torch.where(ok, torch.minimum(ratio, torch.ones_like(ratio)), ratio + 2),
                             torch.zeros_like(ok), what, tile))
    return worst, either


# ------------------------------------------------------------------------------------------------------------------
# operands that reach the edges: maps k / 128 (exact in bf16 and fp16), fp32 flows, affine maps multiples of 1 / 64
# ------------------------------------------------------------------------------------------------------------------
def _ints(g, shape, lo, hi, dev):
    return torch.randint(lo, hi, shape, generator=g, device=dev).float()


def make_map(g, shape, dev, channels=None):
    x = _ints(g, shape, -255, 256, dev) / 128
    if channels is not None:
        x[..., channels:] = 0
    return x


def make_flow(g, h, w, dev):
    """(h, w, 2) fp32 in nine row bands: random +-3 px; integers and half-integers, which put SPyNet's align_corners=True
    coordinate X + f on cell edges and centres; zero (not the identity of the align_corners=False grid); bands that push the
    warp's taps partly and wholly off the left, right, top and bottom borders (by 0 .. 2 px); and flows whose align_corners=False
    warp coordinate (X + f) W / (W - 1) - 0.5 of a same-size source lands on a cell edge k (up to the flow's fp32 rounding)"""
    f = _ints(g, (h, w, 2), -192, 193, dev) / 64
    band = (torch.arange(h, device=dev) * 9 // h).view(h, 1).expand(h, w)
    X = torch.arange(w, device=dev, dtype=torch.float32).view(1, w).expand(h, w)
    Y = torch.arange(h, device=dev, dtype=torch.float32).view(h, 1).expand(h, w)
    r = _ints(g, (h, w), 0, 129, dev) / 64
    ints = _ints(g, (h, w, 2), -3, 4, dev)
    f = torch.where((band == 1)[..., None], ints, f)
    f = torch.where((band == 2)[..., None], ints + 0.5, f)
    f = torch.where((band == 3)[..., None], torch.zeros_like(f), f)
    f[..., 0] = torch.where(band == 4, -(X + r), f[..., 0])
    f[..., 0] = torch.where(band == 5, (w - 1 - X) + r, f[..., 0])
    f[..., 1] = torch.where(band == 6, -(Y + r), f[..., 1])
    f[..., 1] = torch.where(band == 7, (h - 1 - Y) + r, f[..., 1])
    kx, ky = (X.double() + ints[..., 0]).clamp(0, w - 1), (Y.double() + ints[..., 1]).clamp(0, h - 1)
    f[..., 0] = torch.where(band == 8, ((kx + 0.5) * (w - 1) / w - X.double()).float(), f[..., 0])
    f[..., 1] = torch.where(band == 8, ((ky + 0.5) * (h - 1) / h - Y.double()).float(), f[..., 1])
    return f.contiguous()


def make_affine(g, h, w, dev):
    """(h, w, 3) in [-3, 3]: random, both clamp limits, and the identity (1, 1, 1)"""
    a = _ints(g, (h, w, 3), -192, 193, dev) / 64
    band = (torch.arange(h, device=dev) * 4 // h).view(h, 1, 1).expand(h, w, 3)
    lim = (_ints(g, (h, w, 3), 0, 2, dev) * 6 - 3)
    a = torch.where(band == 1, lim, a)
    a = torch.where(band == 2, torch.ones_like(a), a)
    return a.contiguous()


def make_conf(g, shape, dev):
    """confidence values k / 128 in [-0.5, 1.5]: outside [0, 1] where a clamp follows"""
    return _ints(g, shape, -64, 193, dev) / 128


def _seed(*parts):
    return zlib.crc32('/'.join(map(str, parts)).encode())


# ------------------------------------------------------------------------------------------------------------------
# one case: operands, the call, the reference check
# ------------------------------------------------------------------------------------------------------------------
Case = collections.namedtuple('Case', 'outs run verify tile')


def _fl(sig):
    return dict(sig.flags)


def build_case(sig, geom, dt, dev, seed, n=0, C=None):
    """the operator call of `sig` at input geometry `geom` with activation dtype `dt` on `dev`; n > 0: a batch of n distinct
    images through the batched entry.  Case.outs: [(shape, dtype)]; Case.run(ops, *outs); Case.verify(*outs) -> (worst,
    either-side count)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    op, fl = sig.op, _fl(sig)
    C = C or sig.alloc
    lead = (n,) if n else ()
    imgs = range(max(n, 1))
    at = (lambda t, k: t[k] if n else t)

    if op == 'warp':
        h, w = geom
        up2, ss = fl['flow_up2'], fl['src_scale']
        Hs, Ws = ss * h, ss * w
        Ho, Wo = (2 * h, 2 * w) if up2 else (h, w)
        src = make_map(g, lead + ((Hs, Ws) if C == 1 else (Hs, Ws, C)), dev).to(dt)
        flow = torch.stack([make_flow(g, h, w, dev) for _ in imgs]) if n else make_flow(g, h, w, dev)
        shape = lead + ((Ho, Wo) if C == 1 else (Ho, Wo, C))
        return Case([(shape, dt)], lambda ops, o: ops.warp(src, flow, o, flow_up2=up2),
                    lambda o: _worst([check(_v3(at(o, k)), *ref_warp(at(src, k), at(flow, k), up2), dt, f'image {k}', (16, 16))
                                      for k in imgs]), (16, 16))
    if op == 'warp3':
        h, w = geom
        feat = make_map(g, lead + (h, w, C), dev).to(dt)
        featUP = make_map(g, lead + (2 * h, 2 * w, C), dev).to(dt)
        conf = make_conf(g, lead + (h, w), dev)
        flow = torch.stack([make_flow(g, h, w, dev) for _ in imgs]) if n else make_flow(g, h, w, dev)

        def verify(of, ou, oc):
            r = []
            for k in imgs:
                r.append(check(_v3(at(of, k)), *ref_warp(at(feat, k), at(flow, k), False), dt, f'image {k} feat', (8, 16)))
                r.append(check(_v3(at(ou, k)), *ref_warp(at(featUP, k), at(flow, k), True), dt, f'image {k} featUP', (16, 32)))
                r.append(check(_v3(at(oc, k)), *ref_warp(at(conf, k), at(flow, k), False), torch.float32, f'image {k} conf', (8, 16)))
            return _worst(r)
        return Case([(lead + (h, w, C), dt), (lead + (2 * h, 2 * w, C), dt), (lead + (h, w), torch.float32)],
                    lambda ops, of, ou, oc: ops.warp3(feat, featUP, conf, flow, of, ou, oc), verify, (8, 16))
    if op == 'spynet_resize_norm':
        H, W, Ho, Wo = geom
        src = _ints(g, (3, H, W), 0, 256, dev) / 255
        mean = torch.tensor([0.485, 0.456, 0.406], dtype=torch.float32).double().to(dev).view(1, 3, 1, 1)
        std = torch.tensor([0.229, 0.224, 0.225], dtype=torch.float32).double().to(dev).view(1, 3, 1, 1)

        def verify(o):
            y, b = ref_bilinear(src.double().unsqueeze(0), (Ho, Wo))
            r = (y - mean) / std
            return check(o, _hwc(r), _hwc((b + C_AR * U * (y.abs() + mean)) / std), torch.float32, 'resize_norm')
        return Case([((Ho, Wo, 3), torch.float32)], lambda ops, o: ops.spynet_resize_norm(src, o), verify, (16, 16))
    if op == 'avgpool2':
        H, W = geom
        src = make_map(g, (H, W, 3), dev)
        return Case([((H // 2, W // 2, 3), torch.float32)], lambda ops, o: ops.avgpool2(src, o),
                    lambda o: check(o, _hwc(F.avg_pool2d(_nchw(src), 2)), _hwc(C_AR * U * F.avg_pool2d(_nchw(src).abs(), 2)),
                                    torch.float32, 'avgpool2'), (16, 16))
    if op == 'spynet_level_input':
        H, W = geom
        ref_img, supp = make_map(g, (H, W, 3), dev), make_map(g, (H, W, 3), dev)
        fp = make_flow(g, H // 2, W // 2, dev) if fl['flow_prev'] else None

        def verify(o8, ofu):
            r, b, fu, ef = ref_level_input(ref_img, supp, fp)
            a = check(o8, r, b, dt, 'out8')
            return _worst([a, check(ofu, fu, ef, torch.float32, 'flow_up')])
        return Case([((H, W, 8), dt), ((H, W, 2), torch.float32)],
                    lambda ops, o8, ofu: ops.spynet_level_input(ref_img, supp, fp, o8, ofu), verify, (16, 16))
    if op == 'flow_resize':
        H, W, h, w = geom
        flow = make_flow(g, H, W, dev)

        def verify(o):
            y, b = ref_bilinear(_nchw(flow), (h, w), mul=[w / W, h / H])
            return check(o, _hwc(y), _hwc(b), torch.float32, 'flow_resize')
        return Case([((h, w, 2), torch.float32)], lambda ops, o: ops.flow_resize(flow, o), verify, (16, 16))
    if op == 'prep_image':
        H, W = geom
        src = _ints(g, (3, H, W), 0, 256, dev) / 255
        mat = (_ints(g, (12,), -128, 129, dev) / 64).tolist() if fl['mat'] else None
        pool = fl['pool2']
        Ho, Wo = (H // 2, W // 2) if pool else (H, W)

        def verify(o):
            x = src.double().unsqueeze(0)
            y, a = x, x.abs()
            if mat is not None:
                m = torch.tensor(mat, dtype=torch.float64, device=dev).view(3, 4)
                y = F.conv2d(x, m[:, :3].reshape(3, 3, 1, 1), m[:, 3])
                a = F.conv2d(x.abs(), m[:, :3].abs().reshape(3, 3, 1, 1), m[:, 3].abs())
            if pool:
                y, a = F.avg_pool2d(y, 2), F.avg_pool2d(a, 2)
            assert torch.equal(o[..., 3:].float(), torch.zeros_like(o[..., 3:].float())), 'padding channels not zero'
            return check(o[..., :3], _hwc(y), _hwc(C_AR * U * a), dt, 'prep_image')
        return Case([((Ho, Wo, sig.alloc), dt)], lambda ops, o: ops.prep_image(src, o, mat12=mat, pool2=pool), verify, (16, 16))
    if op == 'maxpool2':
        H, W = geom
        src = make_map(g, (H, W, C), dev).to(dt)
        return Case([((H // 2, W // 2, C), dt)], lambda ops, o: ops.maxpool2(src, o),
                    lambda o: check_exact(o, _hwc(F.max_pool2d(_nchw(src), 2)).to(dt), 'maxpool2'), (16, 16))
    if op == 'resize_planes':
        H, W, Ho, Wo = geom
        src = make_conf(g, (sig.alloc, H, W), dev)
        inv, mode, cl = fl['inv_scale'], fl['mode'], fl['clamp01']

        def verify(o):
            o3 = o.permute(1, 2, 0)
            if mode == 'nearest':
                return check_exact(o3, src[:, ::2, ::2].permute(1, 2, 0), 'nearest')
            y, b = bicubic(src.double().unsqueeze(0), 1.0 / inv)
            if cl:
                y = y.clamp(0, 1)
            return check(o3, _hwc(y), _hwc(b.expand_as(y)), torch.float32, 'resize_planes')
        return Case([((sig.alloc, Ho, Wo), torch.float32)],
                    lambda ops, o: ops.resize_planes(src, o, inv, mode=mode, clamp01=cl), verify, (16, 16))
    if op == 'patch_pack':
        H, W = geom
        feat = make_map(g, (H, W, sig.real), dev).to(dt)
        feat[0, 0] = 0                                               # one zero pixel: a patch with a zero tap
        mode, kpad = fl['mode'], sig.alloc

        def verify(o):
            v = ref_patches(feat)
            K = v.shape[1]
            hi_, lo_ = o[:, :K].double(), None        # (every hi copy is checked on its own below)
            segs = {0: [('hi', 0)], 1: [('hi', 0), ('lo', K), ('hi', 2 * K)], 2: [('hi', 0), ('hi', K), ('lo', 2 * K)]}[mode]
            res = []
            for kind, s in segs:
                seg = o[:, s:s + K].double()
                if kind == 'hi':
                    res.append(check(seg.view(H, W, K), v.view(H, W, K), torch.zeros_like(v).view(H, W, K), torch.float16,
                                     f'hi at column {s}'))
                else:
                    lo_ = seg
            if lo_ is not None:
                base = ulp(v - hi_, torch.float16) + (K + C_AR) * U * v.abs()
                res.append(check((hi_ + lo_).view(H, W, K), v.view(H, W, K), base.view(H, W, K), torch.float32, 'hi + lo'))
            used = K * (1 if mode == 0 else 3)
            assert bool((o[:, used:] == 0).all()), 'padding columns not zero'
            return _worst(res)
        return Case([((H * W, kpad), torch.float16)], lambda ops, o: ops.patch_pack(feat, o, mode), verify, (16, 16))
    if op == 'gather_blocks':
        Hv, Wv, hq, wq = geom
        ks = fl['ks']
        value = make_map(g, (Hv, Wv, C), dev).to(dt)
        idx = torch.randint(0, (Hv // ks) * (Wv // ks), (hq * wq,), generator=g, device=dev, dtype=torch.int32)

        def verify(o):
            wvk = Wv // ks
            ry, rx = (idx.long() // wvk).view(hq, wq), (idx.long() % wvk).view(hq, wq)
            a = torch.arange(ks, device=dev)
            iy = (ry.view(hq, 1, wq, 1) * ks + a.view(1, ks, 1, 1)).expand(hq, ks, wq, ks).reshape(hq * ks, wq * ks)
            ix = (rx.view(hq, 1, wq, 1) * ks + a.view(1, 1, 1, ks)).expand(hq, ks, wq, ks).reshape(hq * ks, wq * ks)
            return check_exact(o, value[iy, ix], 'gather_blocks', (ks, ks))
        return Case([((ks * hq, ks * wq, C), dt)], lambda ops, o: ops.gather_blocks(value, idx, hq, wq, ks, o), verify, (ks, ks))
    if op == 'space_to_depth2':
        H, W = geom
        src = make_map(g, (H, W, C), dev).to(dt)
        return Case([((H // 2, W // 2, 4 * C), dt)], lambda ops, o: ops.space_to_depth2(src, o),
                    lambda o: check_exact(o, src.view(H // 2, 2, W // 2, 2, C).permute(0, 2, 1, 3, 4).reshape(H // 2, W // 2, 4 * C),
                                          's2d'), (16, 16))
    if op == 'bicubic_up2_image':
        H, W = geom
        src = make_conf(g, (3, H, W), dev)

        def verify(o):
            assert torch.equal(o[..., 3:].float(), torch.zeros_like(o[..., 3:].float())), 'padding channels not zero'
            y, b = bicubic(src.double().unsqueeze(0), 2)
            return check(o[..., :3], _hwc(y), _hwc(b.expand_as(y)), dt, 'bicubic_up2_image')
        return Case([((2 * H, 2 * W, sig.alloc), dt)], lambda ops, o: ops.bicubic_up2_image(src, o), verify, (16, 16))
    if op == 'aligned_sample':
        h, w = geom
        ks = fl['ks']
        x = make_map(g, (ks * h, ks * w, C), dev).to(dt)
        aff = make_affine(g, h, w, dev)
        return Case([((ks * h, ks * w, C), dt)], lambda ops, o: ops.aligned_sample(x, aff, ks, o),
                    lambda o: verify_aligned(o, x, aff, ks, dt, 'aligned_sample'), (2 * ks, 16 * ks))
    if op == 'conf_pair':
        h, w = geom
        up2 = fl['up2']
        a, b = make_conf(g, lead + (h, w), dev), make_conf(g, lead + (h, w), dev)
        Ho, Wo = (2 * h, 2 * w) if up2 else (h, w)

        def verify(o):
            r = []
            for k in imgs:
                ok = at(o, k)
                assert torch.equal(ok[..., 2:].float(), torch.zeros_like(ok[..., 2:].float())), f'image {k}: padding channels not zero'
                x = torch.stack([at(a, k), at(b, k)]).double().unsqueeze(0)
                if up2:
                    y, bb = bicubic(x, 2)
                    y, bb = y.clamp(0, 1), bb.expand_as(y)
                else:
                    y, bb = x, torch.zeros_like(x)
                r.append(check(ok[..., :2], _hwc(y), _hwc(bb), dt, f'image {k}'))
            return _worst(r)
        return Case([(lead + (Ho, Wo, sig.alloc), dt)], lambda ops, o: ops.conf_pair(a, b, o, up2=up2), verify, (16, 16))
    if op == 'conf_max':
        h, w = geom
        a, b = make_conf(g, (h, w), dev), make_conf(g, (h, w), dev)
        return Case([((h, w), torch.float32)], lambda ops, o: ops.conf_max(a, b, o),
                    lambda o: check_exact(_v3(o), _v3(torch.maximum(a, b)), 'conf_max'), (16, 16))
    if op in ('reconstruct', 'reconstruct_u8'):
        h, w = geom
        s, cl = fl['scale'], fl['clamp01']
        xdt = DT[sig.dt] if sig.dt != 'act' else dt
        x = (_ints(g, lead + (s * h, s * w, sig.alloc), -128, 129, dev) / 128).to(xdt)
        lr = _ints(g, lead + (3, h, w), -64, 321, dev) / 256

        def ref_rec(k):
            base, bb = bicubic(at(lr, k).double().unsqueeze(0), s)
            base = base.clamp(0, 1)
            v = _hwc(base) + at(x, k)[..., :3].double()
            if cl:
                v = v.clamp(0, 1)
            return v, _hwc(bb.expand_as(base)) + C_AR * U * (v.abs() + 1)
        if op == 'reconstruct':
            return Case([(lead + (3, s * h, s * w), torch.float32)], lambda ops, o: ops.reconstruct(x, lr, s, cl, o),
                        lambda o: _worst([check(at(o, k).permute(1, 2, 0), *ref_rec(k), torch.float32, f'image {k}', (s, 16 * s))
                                          for k in imgs]), (s, 16 * s))
        bgr = fl['bgr']

        def verify_u8(o):
            r = []
            for k in imgs:
                v, b = ref_rec(k)
                if bgr:
                    v, b = v.flip(-1), b.flip(-1)
                r.append(check_u8(at(o, k), v, b, f'image {k}', (s, 16)))
            return _worst(r)
        return Case([(lead + (s * h, s * w, 3), torch.uint8)], lambda ops, o: ops.reconstruct_u8(x, lr, s, cl, o, bgr), verify_u8,
                    (s, 16))
    raise AssertionError(op)


def verify_aligned(o, x, aff, ks, dt, what):
    """aligned_sample's check with the either-side rule at the clamped padded border"""
    H, W = x.shape[:2]
    ref, A, pr, pc, _ = ref_aligned(x, aff, ks)
    drr, dcc = aligned_delta(pr, pc, aff, ks, H, W)
    L = 4 * float(x.double().abs().max())
    base = C_AR * U * A + (L * (drr + dcc)).unsqueeze(-1)
    near = torch.zeros_like(pr, dtype=torch.bool)
    for p, d, m in ((pr, drr, H + 1), (pc, dcc, W + 1)):
        near |= (p.abs() <= d) | ((p - m).abs() <= d)
    alts = []
    if near.any():
        for sr in (-1, 1):
            for sc in (-1, 1):
                alts.append(ref_aligned(x, aff, ks, sr * drr, sc * dcc)[0])
    return check(o, ref, base, dt, what, (2 * ks, 16 * ks), alt=(near.unsqueeze(-1), alts))


def _v3(t):
    return t.unsqueeze(-1) if t.dim() == 2 else t


def _worst(results):
    return max(r[0] for r in results), sum(r[1] for r in results)


def run_guarded(ops, case, dev, off=0, prof_kernels=None):
    """Case.run with every output `off` elements into a buffer filled with NaN (0xA5 for bytes) and GUARD sentinels on either
    side: the guards must be intact afterwards.  Returns the outputs."""
    bufs, outs = [], []
    for shape, dtp in case.outs:
        nel = int(np.prod(shape))
        buf = torch.empty(nel + 2 * GUARD + off, dtype=dtp, device=dev)
        buf.fill_(0xA5 if dtp == torch.uint8 else float('nan'))
        bufs.append((buf, nel))
        outs.append(buf[GUARD + off:GUARD + off + nel].view(shape))
    case.run(ops, *outs)
    if dev != 'cpu':
        torch.cuda.synchronize()
    for buf, nel in bufs:
        head, tail = buf[:GUARD + off], buf[GUARD + off + nel:]
        if buf.dtype == torch.uint8:
            assert bool((head == 0xA5).all()) and bool((tail == 0xA5).all()), 'wrote outside its output'
        else:
            assert bool(torch.isnan(head).all()) and bool(torch.isnan(tail).all()), 'wrote outside its output'
    return outs


# ------------------------------------------------------------------------------------------------------------------
# CPU: the bound separates a correct kernel from subtly wrong ones
# ------------------------------------------------------------------------------------------------------------------
def _entry(op, **flags):
    return next(e for e in ENGINE_POINTWISE if e.sig.op == op and all(dict(e.sig.flags).get(k) == v for k, v in flags.items()))


def _cpu_sig(e, dt):
    return e.sig._replace(dt='fp32' if e.sig.dt == 'fp32' else DTN[dt])


# (id, entry, geometry): a subset of the list at CPU-sized geometries, with one full 270x480 warp
# patch_pack into rows wider than its values (kpad 160 > 144): the padding columns must be written as zeros
PP_PAD = _entry('patch_pack', mode=0)._replace(sig=_entry('patch_pack', mode=0).sig._replace(alloc=160))
FAKE_CASES = [
    ('warp-270x480', _entry('warp', flow_up2=False, src_scale=1), (270, 480)),
    ('warp-conf', _entry('warp', flow_up2=False, src_scale=1)._replace(sig=_entry('warp', src_scale=1).sig._replace(real=1, alloc=1)), (37, 53)),
    ('warp-up2', _entry('warp', flow_up2=True, src_scale=2), (19, 27)),
    ('warp-up2-quirk', _entry('warp', flow_up2=True, src_scale=1), (19, 27)),
    ('level-input', _entry('spynet_level_input', flow_prev=True), (36, 60)),
    ('resize-norm', _entry('spynet_resize_norm'), (45, 60, 48, 64)),
    ('flow-resize', _entry('flow_resize'), (48, 64, 45, 64)),
    ('prep-pool', _entry('prep_image', mat=True, pool2=True), (30, 44)),
    ('bicubic-up2', _entry('bicubic_up2_image'), (21, 33)),
    ('resize-x2-clamp', _entry('resize_planes', inv_scale=0.5), (21, 33, 42, 66)),
    ('aligned-ks2', _entry('aligned_sample', ks=2), (13, 17)),
    ('aligned-ks4', _entry('aligned_sample', ks=4), (7, 9)),
    ('patch-pack', _entry('patch_pack', mode=0), (19, 27)),
    ('patch-pack-split-lo-mid', _entry('patch_pack', mode=1), (19, 27)),
    ('patch-pack-split-lo-last', _entry('patch_pack', mode=2), (19, 27)),
    ('patch-pack-padding-columns', PP_PAD, (19, 27)),
    ('conf-pair-up2', _entry('conf_pair', up2=True), (21, 33)),
    ('reconstruct-x4', _entry('reconstruct', scale=4), (21, 33)),
    ('reconstruct-u8-x2', _entry('reconstruct_u8', scale=2), (21, 33)),
    ('gather-ks4', _entry('gather_blocks', ks=4, ), (32, 48, 7, 9)),
]


def _oracle():
    from u8_ops import U8OracleOps
    return U8OracleOps()


@pytest.mark.parametrize('dt', [torch.float32, torch.bfloat16, torch.float16], ids=['fp32', 'bf16', 'fp16'])
@pytest.mark.parametrize('cid,entry,geom', FAKE_CASES, ids=[c[0] for c in FAKE_CASES])
def test_bound_passes_a_correct_kernel(cid, entry, geom, dt):
    """OracleOps (fp32 arithmetic, one rounding to the output type) passes the bound: the float64 reference and OracleOps agree on
    the operators' semantics"""
    if entry.sig.dt == 'fp32' and dt != torch.float32:
        pytest.skip('fp32-only operator')
    if entry.sig.op == 'patch_pack' and (dt == torch.float32) != ('32' in entry.precs):
        pytest.skip('the engine packs 16-bit features with mode 0 and fp32 features with the split modes')
    case = build_case(_cpu_sig(entry, dt), geom, dt, 'cpu', _seed(cid))
    case.verify(*run_guarded(_oracle(), case, 'cpu'))


class _Mutant:
    """OracleOps with one planted defect"""

    def __init__(self, mutation):
        self.o, self.m = _oracle(), mutation

    def __getattr__(self, name):
        return getattr(self.o, name)

    def warp(self, src, flow, out, flow_up2=False):
        m = self.m
        if m == 'half-pixel-shift':
            flow = flow + 0.5
        if m == 'up2-without-x2' and flow_up2:
            flow = flow / 2
        if m in ('swap-ne-sw', 'border-padding'):
            x = _nchw(src).float()
            f = _nchw(flow).float()
            Hi, Wi = x.shape[-2:]
            Ho, Wo = f.shape[-2:]
            gx = torch.linspace(-1, 1, Wo).view(1, Wo) + f[0, 0] / ((Wi - 1) / 2)
            gy = torch.linspace(-1, 1, Ho).view(Ho, 1) + f[0, 1] / ((Hi - 1) / 2)
            px, py = ((gx + 1) * Wi - 1) / 2, ((gy + 1) * Hi - 1) / 2
            x0, y0 = px.floor(), py.floor()
            taps = _taps(x, x0.long(), y0.long(), m == 'border-padding')
            fx, fy = px - x0, py - y0
            wts = [(1 - fx) * (1 - fy), fx * (1 - fy), (1 - fx) * fy, fx * fy]
            if m == 'swap-ne-sw':
                wts[1], wts[2] = wts[2], wts[1]
            y = sum(t * wq for t, wq in zip(taps, wts))
            out.copy_((_hwc(y) if out.dim() == 3 else _hwc(y)[..., 0]).to(out.dtype))
            return
        self.o.warp(src, flow, out, flow_up2)

    def patch_pack(self, feat, out, mode):
        self.o.patch_pack(feat, out, mode)
        K = 9 * feat.shape[2]
        lo = out[:, K:2 * K] if mode == 1 else out[:, 2 * K:3 * K]
        if self.m == 'dropped-lo':
            lo.zero_()
        if self.m == 'doubled-lo':
            lo.mul_(2)

    def aligned_sample(self, x, affine, ks, out):
        if self.m != 'replicate-padding':
            return self.o.aligned_sample(x, affine, ks, out)
        import oracle.refvsr_oracle as O
        pad = O.F.pad
        O.F.pad = lambda t, p, mode='constant', value=None: pad(t, p, mode='replicate')
        try:
            self.o.aligned_sample(x, affine, ks, out)
        finally:
            O.F.pad = pad

    def reconstruct(self, x, lr, scale, clamp01, out):
        import oracle.refvsr_oracle as O
        if self.m == 'cubic-a-0.5':
            cw = O._cubic_weights

            def w05(t):
                A = -0.5
                return torch.stack([((A * (t + 1) - 5 * A) * (t + 1) + 8 * A) * (t + 1) - 4 * A, ((A + 2) * t - (A + 3)) * t * t + 1,
                                    ((A + 2) * (1 - t) - (A + 3)) * (1 - t) * (1 - t) + 1,
                                    ((A * (2 - t) - 5 * A) * (2 - t) + 8 * A) * (2 - t) - 4 * A], -1)
            O._cubic_weights = w05
            try:
                return self._reconstruct(x, lr, scale, clamp01, out)
            finally:
                O._cubic_weights = cw
        return self._reconstruct(x, lr, scale, clamp01, out)

    def _reconstruct(self, x, lr, scale, clamp01, out):
        if lr.dim() == 4:                                        # a batch: image k's output from image k's operands
            for k in range(lr.shape[0]):
                src = 0 if self.m == 'batch-stride' else k       # the wrong image stride: every image reads image 0
                self.o.reconstruct(x[src], lr[src], scale, clamp01, out[k])
            return
        self.o.reconstruct(x, lr, scale, clamp01, out)
        if self.m == 'double-rounding':
            out.copy_(out.to(torch.bfloat16).float())


_16 = ((torch.bfloat16, 'bf16'), (torch.float16, 'fp16'))
_32 = ((torch.float32, 'fp32'),)
MUTATIONS = [
    ('half-pixel-shift', 'warp', dict(flow_up2=False, src_scale=1), (27, 41), 0, _16),
    ('swap-ne-sw', 'warp', dict(flow_up2=False, src_scale=1), (27, 41), 0, _16),
    ('border-padding', 'warp', dict(flow_up2=False, src_scale=1), (27, 41), 0, _16),
    ('up2-without-x2', 'warp', dict(flow_up2=True, src_scale=2), (19, 27), 0, _16),
    ('replicate-padding', 'aligned_sample', dict(ks=2), (13, 17), 0, _16),
    ('cubic-a-0.5', 'reconstruct', dict(scale=4), (21, 33), 0, _16),
    ('double-rounding', 'reconstruct', dict(scale=2), (21, 33), 0, _16),
    ('batch-stride', 'reconstruct', dict(scale=4), (21, 33), 3, _16),
    ('dropped-lo', 'patch_pack', dict(mode=1), (19, 27), 0, _32),
    ('dropped-lo', 'patch_pack', dict(mode=2), (19, 27), 0, _32),
    ('doubled-lo', 'patch_pack', dict(mode=1), (19, 27), 0, _32),
]
_MUTATION_CASES = [m[:5] + (dt,) for m in MUTATIONS for dt, _ in m[5]]


@pytest.mark.parametrize('mutation,op,flags,geom,n,dt', _MUTATION_CASES,
                         ids=[f'{m[0]}-{"-".join(f"{k}{v}" for k, v in m[2].items())}-{DTN[m[5]]}' for m in _MUTATION_CASES])
def test_bound_fails_a_subtly_wrong_kernel(mutation, op, flags, geom, n, dt):
    """each planted defect fails, with a report that names where the failing elements sit within their tiles"""
    case = build_case(_cpu_sig(_entry(op, **flags), dt), geom, dt, 'cpu', _seed(mutation), n=n)
    outs = run_guarded(_Mutant(mutation), case, 'cpu')
    with pytest.raises(pytest.fail.Exception, match=r'outside the bound(.|\n)*within its \d+ x \d+ tile'):
        case.verify(*outs)


def test_flow_bands_reach_every_border():
    """the flow operands move the warp's taps partly and wholly off each border and put its align_corners=False coordinate on
    cell edges; they put SPyNet's align_corners=True coordinate X + f on edges and centres; and they include zero"""
    h, w = 64, 96
    f = make_flow(torch.Generator().manual_seed(0), h, w, 'cpu').double()
    X = torch.arange(w, dtype=torch.float64).view(1, w)
    Y = torch.arange(h, dtype=torch.float64).view(h, 1)
    px, py = (X + f[..., 0]) * w / (w - 1) - 0.5, (Y + f[..., 1]) * h / (h - 1) - 0.5       # the warp of a same-size source
    for m in (px < -1, (px > -1) & (px < 0), px > w, (px > w - 1) & (px < w), py < -1, (py > -1) & (py < 0), py > h,
              (py > h - 1) & (py < h)):
        assert bool(m.any())
    on_edge = ((px - px.round()).abs() < 1e-4) & ((py - py.round()).abs() < 1e-4)
    assert int(on_edge.sum()) >= w * (h // 9)
    assert bool((f == 0).all(-1).any()) and bool((f.frac() == 0.5).any()) and bool(((f.frac() == 0) & (f != 0)).any())
    a = make_affine(torch.Generator().manual_seed(0), 16, 16, 'cpu')
    assert float(a.min()) == -3 and float(a.max()) == 3 and bool((a == 1).all(-1).any())


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _dtypes(e):
    if e.sig.dt == 'fp32':
        return [torch.float32]
    return ([torch.bfloat16, torch.float16] if '16' in e.precs else []) + ([torch.float32] if '32' in e.precs else [])


def _flag_id(e):
    return ','.join(f'{k}={v}' for k, v in e.sig.flags)


_ENGINE_CASES = [(e, g, dt) for e in ENGINE_POINTWISE for g in e.geoms for dt in _dtypes(e)]


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        r = fn()
        torch.cuda.synchronize()
    return r, {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}


@pytest.mark.gpu
@pytest.mark.parametrize('case', _ENGINE_CASES, ids=[f'{e.sig.op}-{e.sig.real}of{e.sig.alloc}[{_flag_id(e)}]-{DTN[dt]}-{"x".join(map(str, g))}'
                                                     for e, g, dt in _ENGINE_CASES])
def test_engine_pointwise(cuda_ops, case):
    e, geom, dt = case
    c = build_case(_cpu_sig(e, dt), geom, dt, 'cuda', _seed(e.sig, geom, DTN[dt]))
    c.verify(*run_guarded(cuda_ops, c, 'cuda'))


W48, WC = _entry('warp', flow_up2=False, src_scale=1), _entry('warp', src_scale=1)
# kernel branches, forced: (id, entry, geometry, dtype, options: n batch, off output offset in elements (1: 2 bytes off a
# 16-byte boundary in a 16-bit map), C channels,
# expect: a regular expression one of the launched kernels must match)
BRANCH_CASES = [
    ('batched-warp', W48, (67, 121), torch.bfloat16, dict(n=3, expect=r'warp_vec_kernel')),
    ('batched-warp-conf', WC._replace(sig=WC.sig._replace(real=1, alloc=1, dt='fp32')), (67, 121), torch.float32,
     dict(n=3, expect=r'warp_kernel<float, 1>')),
    ('batched-warp3', _entry('warp3'), (67, 121), torch.bfloat16, dict(n=3, expect=r'warp3_kernel')),
    ('batched-conf-pair-up2', _entry('conf_pair', up2=True), (67, 121), torch.float16, dict(n=3, expect=r'conf_pair_kernel')),
    ('batched-reconstruct-x4', _entry('reconstruct', scale=4), (67, 121), torch.float32, dict(n=3, expect=r'reconstruct4_kernel')),
    ('batched-reconstruct-x2', _entry('reconstruct', scale=2), (67, 121), torch.float32, dict(n=3, expect=r'reconstruct2_kernel')),
    ('batched-reconstruct-u8-x4', _entry('reconstruct_u8', scale=4), (68, 120), torch.float32,
     dict(n=3, expect=r'reconstruct4_u8_kernel')),
    ('batched-reconstruct-u8-x2', _entry('reconstruct_u8', scale=2), (68, 120), torch.float32,
     dict(n=3, expect=r'reconstruct2_u8_kernel')),
    ('ragged-271x483-warp3', _entry('warp3'), (271, 483), torch.bfloat16, dict(expect=r'warp3_kernel')),
    ('ragged-271x483-warp3-fp16', _entry('warp3'), (271, 483), torch.float16, dict(expect=r'warp3_kernel')),
    ('ragged-warp3-c24-cv3', _entry('warp3'), (37, 53), torch.bfloat16, dict(C=24, expect=r'warp3_kernel<__nv_bfloat16, 3>')),
    ('ragged-aligned-ks2', _entry('aligned_sample', ks=2), (135, 241), torch.bfloat16, dict(expect=r'aligned_sample2_kernel')),
    ('ragged-aligned-ks4', _entry('aligned_sample', ks=4), (67, 121), torch.float16, dict(expect=r'aligned_sample4_kernel')),
    ('ragged-gather-cells-ks4', _entry('gather_blocks', ks=4, ), (540, 964, 67, 121), torch.bfloat16,
     dict(expect=r'gather_cells_kernel<4, 6>')),
    ('ragged-gather-cells-ks2-c8', _entry('gather_blocks', ks=2), (270, 482, 135, 241), torch.bfloat16, dict(C=8, expect=r'gather_cells_kernel<2, 0>')),
    ('ragged-reconstruct-u8-x4-vec', _entry('reconstruct_u8', scale=4), (67, 124), torch.float32, dict(expect=r'reconstruct4_u8_kernel')),
    ('ragged-reconstruct-u8-x4-novec', _entry('reconstruct_u8', scale=4), (67, 121), torch.float32, dict(expect=r'reconstruct4_u8_kernel')),
    ('ragged-reconstruct-u8-x2-novec', _entry('reconstruct_u8', scale=2), (67, 121), torch.float32, dict(expect=r'reconstruct2_u8_kernel')),
    ('ragged-reconstruct-x2', _entry('reconstruct', scale=2), (67, 121), torch.float32, dict(expect=r'reconstruct2_kernel')),
    ('misaligned-warp', W48, (67, 121), torch.bfloat16, dict(off=1, expect=r'warp_kernel<__nv_bfloat16, 1>')),
    ('misaligned-warp-up2', _entry('warp', flow_up2=True, src_scale=2), (33, 61), torch.float16, dict(off=1, expect=r'warp_kernel<__half, 1>')),
    ('misaligned-aligned-ks2', _entry('aligned_sample', ks=2), (67, 121), torch.bfloat16,
     dict(off=1, expect=r'aligned_sample_kernel<__nv_bfloat16, 1>')),
    ('misaligned-gather-blocks-4', _entry('gather_blocks', ks=4), (540, 964, 67, 121), torch.bfloat16,
     dict(off=2, expect=r'gather_blocks_kernel<4>')),
    # a 2-byte offset once took the 4-byte-word copy and faulted on a misaligned store: 16-bit words are the widest it can move
    ('misaligned-2B-gather-blocks-takes-16bit-words', _entry('gather_blocks', ks=4), (540, 964, 67, 121), torch.bfloat16,
     dict(off=1, expect=r'gather_blocks_kernel<2>')),
    ('misaligned-gather-blocks-2', _entry('gather_blocks', ks=2), (270, 482, 135, 241), torch.bfloat16,
     dict(C=3, expect=r'gather_blocks_kernel<2>')),
    ('patch-pack-padding-columns', PP_PAD, (270, 480), torch.bfloat16, dict(expect=r'patch_pack_kernel')),
    ('misaligned-reconstruct', _entry('reconstruct', scale=4), (67, 121), torch.float32, dict(off=1, expect=r'reconstruct_kernel<float>')),
    ('misaligned-reconstruct-u8', _entry('reconstruct_u8', scale=2), (67, 121), torch.float32, dict(off=1, expect=r'reconstruct2_u8_kernel')),
]


@pytest.mark.gpu
@pytest.mark.parametrize('case', BRANCH_CASES, ids=[c[0] for c in BRANCH_CASES])
def test_pointwise_branch(cuda_ops, case):
    cid, e, geom, dt, opt = case
    sig = _cpu_sig(e, dt)
    c = build_case(sig, geom, dt, 'cuda', _seed(cid), n=opt.get('n', 0), C=opt.get('C'))
    outs, names = _kernels(lambda: run_guarded(cuda_ops, c, 'cuda', off=opt.get('off', 0)))
    assert any(re.search(opt['expect'], k) for k in names), (cid, sorted(names))
    c.verify(*outs)
