"""Every convolution the engine launches, checked element by element against a float64 reference at the engine's shapes.

The kernels' arithmetic has a tight bound.  Inputs and weights are 16-bit values, so their products are exact in fp32; the
accumulator is fp32; the epilogue (v = act_pre(acc + bias); v *= gate; v += res; act_post; clamp3) runs in fp32 and
rounds once to the output type.  Against a float64 reference `ref` every output element y therefore satisfies

    16-bit outputs:  |y - ref| <= ulp_T(ref) + C_ACC * K * u * A * max(1, |gate|) + 2u |ref|
    fp32 outputs:    |y - ref| <=              C_ACC * K * u * A * max(1, |gate|) + 2u |ref|

with u = 2^-24, K the reduction length (kernel taps x real input channels), A = conv(|x|, |w|) + |b| in float64 and
ulp_T(ref) the spacing of the output type at |ref| (fp16 subnormals included).  That is tight enough to catch one dropped
tap, a tile or channel written from the wrong place, a shifted residual or a second rounding (the CPU tests below show it
on a fake kernel), where a max-abs tolerance relative to max|ref| lets them through.

Without a GPU: the bound's self-tests, and the list of convolutions below against what the engine's schedule launches
(x4 RefVSR_MFID at LR 270x480 and the x2 model at LR 540x960).  With a GPU: every one of them in bf16 and fp16 at every
geometry the two schedules run it at, and each launch-plan branch of the tensor-core kernel at full-size maps."""
import collections
import ctypes as C
import functools
import zlib

import pytest
import torch
import torch.nn.functional as F

from refvsr_b200 import packing
from refvsr_b200.lib import ACT_CLAMP3, ACT_LRELU01, ACT_LRELU02, ACT_NONE, ACT_RELU, IMPL_SIMT, IMPL_TC

U = 2.0 ** -24
# C_ACC: each fp32 operation between the exact products and the value the kernel rounds - the K - 1 additions of the
# accumulation (wgmma does not specify their order, hence the worst-case K * u form and not sqrt(K) * u), the bias add,
# the activation's multiply and the gate multiply - errs by at most 2u of the magnitude it works on if it truncates (u if
# it rounds to nearest; the tensor cores' rounding is not specified either).  To first order these add up to at most
# 2 (K + 2) u A max(1, |gate|) <= 3 K u A max(1, |gate|) for K >= 4 (every conv here has K >= 18).  The residual add and
# the clamp work on values of the size of |ref|: the 2u |ref| term.  Chosen once from this derivation, not per case.
C_ACC = 3.0
GUARD = 4096

# the activations as the kernel applies them: max(v, v * slope) with the slope as an fp32 number
_SLOPE = {ACT_NONE: 1.0, ACT_RELU: 0.0, ACT_LRELU01: float(torch.tensor(0.1, dtype=torch.float32)),
          ACT_LRELU02: float(torch.tensor(0.2, dtype=torch.float32)), ACT_CLAMP3: 1.0}
_MANT_EMIN = {torch.bfloat16: (7, -126), torch.float16: (10, -14)}

# A conv signature: sources [(real, allocated channels)], cout, square kernel size, padding, stride, activations, gate,
# residual ('' none, 'act' in the activation type, 'f32'), 2x pixel shuffle, output type ('act' | 'f32') and the
# channels of the output buffer (cout, cout / 4 after the pixel shuffle, or wider)
Sig = collections.namedtuple('Sig', 'srcs cout k pad stride act_pre act_post gate res ps out out_cs')
N, R, L1, L2, C3 = ACT_NONE, ACT_RELU, ACT_LRELU01, ACT_LRELU02, ACT_CLAMP3
X4, X2 = ((270, 480), (135, 240)), ((540, 960), (1080, 1920))

# SPyNet pyramid levels: the LR frame padded up to a multiple of 32, halved five times (x4: 270x480, x2: 540x960)
SPY = [(9, 15), (18, 30), (36, 60), (72, 120), (144, 240), (288, 480),
       (17, 30), (34, 60), (68, 120), (136, 240), (272, 480), (544, 960)]

# Every conv signature the engine launches (network.py, Network._conv) with the input geometries (H, W) it runs it at in the
# x4 (LR 270x480, Ref 270x480) and x2 (LR 540x960, Ref 540x960) schedules.  The stride-2 convs run as stride-1 3x3 convs over
# the space-to-depth map (s2d): that is what the kernel sees and what is listed.  test_engine_convs_are_all_listed keeps this
# list complete.
ENGINE_CONVS = [
    ('spynet.0', Sig(((8, 8),), 32, 7, 3, 1, R, N, False, '', False, 'act', 32), SPY),
    ('spynet.1', Sig(((32, 32),), 64, 7, 3, 1, R, N, False, '', False, 'act', 64), SPY),
    ('spynet.2', Sig(((64, 64),), 32, 7, 3, 1, R, N, False, '', False, 'act', 32), SPY),
    ('spynet.3', Sig(((32, 32),), 16, 7, 3, 1, R, N, False, '', False, 'act', 16), SPY),
    ('spynet.4+flow_up', Sig(((16, 16),), 2, 7, 3, 1, N, N, False, 'f32', False, 'f32', 2), SPY),
    ('feature_extract.0', Sig(((3, 8),), 64, 3, 1, 1, R, N, False, '', False, 'act', 64), [(270, 480), (135, 240), (540, 960)]),
    ('feature_extract.2', Sig(((64, 64),), 64, 3, 1, 1, R, N, False, '', False, 'act', 64), [(270, 480), (135, 240), (540, 960)]),
    ('feature_extract.5', Sig(((64, 64),), 128, 3, 1, 1, R, N, False, '', False, 'act', 128), [(270, 480), (135, 240)]),
    ('map64', Sig(((64, 64),), 16, 1, 0, 1, L2, N, False, '', False, 'act', 16), [(270, 480), (135, 240)]),
    ('map128', Sig(((128, 128),), 16, 1, 0, 1, L2, N, False, '', False, 'act', 16), [(270, 480), (135, 240)]),
    ('ref_encoder1.0', Sig(((3, 8),), 48, 3, 1, 1, L2, N, False, '', False, 'act', 48), [(270, 480), (540, 960)]),
    ('ref_encoder2.0.s2d', Sig(((192, 192),), 48, 3, 1, 1, L2, N, False, '', False, 'act', 48), [(135, 240), (270, 480)]),
    ('conv48.lrelu', Sig(((48, 48),), 48, 3, 1, 1, L2, N, False, '', False, 'act', 48), X4 + X2),
    ('conv48.relu', Sig(((48, 48),), 48, 3, 1, 1, R, N, False, '', False, 'act', 48), [(270, 480), (540, 960)]),
    ('conv48.res', Sig(((48, 48),), 48, 3, 1, 1, N, N, False, 'act', False, 'act', 48), X4 + X2),
    ('main.0', Sig(((3, 8), (48, 48)), 48, 3, 1, 1, L1, N, False, '', False, 'act', 48), [(270, 480), (540, 960)]),
    ('align.conv1.0', Sig(((3, 8),), 32, 5, 2, 1, L2, N, False, '', False, 'act', 32), [(540, 960), (1080, 1920)]),
    ('align.rb.conv1', Sig(((32, 32),), 32, 3, 1, 1, L2, N, False, '', False, 'act', 32), [(270, 480)] + list(X2)),
    ('align.rb.conv2', Sig(((32, 32),), 32, 3, 1, 1, N, L2, False, 'act', False, 'act', 32), [(270, 480)] + list(X2)),
    ('align.p_conv.0.s2d', Sig(((128, 128), (128, 128)), 32, 3, 1, 1, L2, N, False, '', False, 'act', 32), [(270, 480)]),
    ('align.p_conv.4', Sig(((32, 32),), 3, 1, 0, 1, N, C3, False, '', False, 'f32', 3), [(270, 480)]),
    ('conf_fusion.0', Sig(((2, 8),), 16, 3, 1, 1, L2, N, False, '', False, 'act', 16), [(270, 480)] + list(X2)),
    ('conf_fusion.1', Sig(((16, 16),), 48, 3, 1, 1, L2, N, False, '', False, 'act', 48), [(270, 480)] + list(X2)),
    ('feat_fusion.0', Sig(((48, 48), (48, 48)), 48, 3, 1, 1, L2, N, False, '', False, 'act', 48), [(270, 480)] + list(X2)),
    ('feat_fusion.1', Sig(((48, 48),), 48, 3, 1, 1, L2, N, True, 'act', False, 'act', 48), [(270, 480)] + list(X2)),
    ('upsample1', Sig(((48, 48),), 192, 3, 1, 1, N, N, False, '', True, 'act', 48), [(270, 480), (540, 960)]),
    ('upsample2', Sig(((48, 48),), 192, 3, 1, 1, L1, N, False, '', True, 'act', 48), [(540, 960)]),
    ('fusion_UP', Sig(((48, 48), (48, 48)), 48, 1, 0, 1, N, N, False, '', False, 'act', 48), list(X2)),
    ('conv_hr', Sig(((48, 48),), 48, 3, 1, 1, L1, N, False, '', False, 'act', 48), [(1080, 1920)]),
    ('conv_last', Sig(((48, 48),), 3, 3, 1, 1, N, N, False, '', False, 'f32', 4), [(1080, 1920)]),
    # x2 aa2 (blocks of 4): a stride-4 5x5 conv, which only the CUDA-core kernel (conv_simt.cu) runs
    ('align.p_conv.0.stride4', Sig(((32, 32), (32, 32)), 32, 5, 2, 4, L2, N, False, '', False, 'act', 32), [(1080, 1920)]),
]


# ------------------------------------------------------------------------------------------------------------------
# reference and bound
# ------------------------------------------------------------------------------------------------------------------
def ulp(ref, dtype):
    """spacing of `dtype` (bf16 / fp16) at |ref|, float64; below the smallest normal the subnormal spacing"""
    mant, emin = _MANT_EMIN[dtype]
    _, e = torch.frexp(ref.abs())                       # |ref| = m 2^e, m in [0.5, 1)
    e = torch.where(ref == 0, torch.full_like(e, emin), (e - 1).clamp(min=emin))
    return torch.ldexp(torch.ones_like(ref), e - mant)


def _act(v, code):
    if code == ACT_CLAMP3:
        return v.clamp(-3.0, 3.0)
    s = _SLOPE[code]
    return v if s == 1.0 else torch.maximum(v, v * s)


def _nchw(t):
    return t.permute(2, 0, 1).unsqueeze(0)


def _nhwc(t):
    return t[0].permute(1, 2, 0)


def reference(sig, ops, k_acc=None):
    """float64 (ref, base) in the output's NHWC layout: ref = the conv, then the epilogue in the kernel's order, then the
    pixel shuffle; base = C_ACC K u A max(1, |gate|) + 2u |ref|, the bound without the output type's ulp.  k_acc: the
    number of products that can round in the accumulation, if fewer than K (weights that are exact zeros add nothing)"""
    x = torch.cat([t[..., :r] for t, (r, _) in zip(ops['xs'], sig.srcs)], 2).double()
    w, b = ops['w'].double(), ops['b'].double()
    y = F.conv2d(_nchw(x), w, b, stride=sig.stride, padding=sig.pad)
    a = F.conv2d(_nchw(x).abs(), w.abs(), b.abs(), stride=sig.stride, padding=sig.pad)
    y = _act(y, sig.act_pre)
    if sig.gate:
        g = _nchw(ops['gate'][..., :sig.cout].double())
        y = y * g
        a = a * g.abs().clamp(min=1.0)
    if sig.res:
        y = y + _nchw(ops['res'][..., :sig.cout].double())
    y = _act(y, sig.act_post)
    if sig.ps:
        y, a = F.pixel_shuffle(y, 2), F.pixel_shuffle(a, 2)
    y, a = _nhwc(y), _nhwc(a)
    K = k_acc or sig.k * sig.k * sum(r for r, _ in sig.srcs)
    return y, C_ACC * K * U * a + 2 * U * y.abs()


def bound(ref, base, out_dtype):
    return base if out_dtype == torch.float32 else base + ulp(ref, out_dtype)


def out_hw(sig, H, W):
    Ho, Wo = (H + 2 * sig.pad - sig.k) // sig.stride + 1, (W + 2 * sig.pad - sig.k) // sig.stride + 1
    return (2 * Ho, 2 * Wo) if sig.ps else (Ho, Wo)


def make_operands(sig, H, W, device, seed, gate_cs=None, res_cs=None):
    """fp32 tensors whose values are exact in both bf16 and fp16 (at most 8 significant bits, exponents well inside both
    ranges), so that one float64 reference serves both types: inputs k / 128 and weights k 2^-e with |k| < 256, gates
    in [0, 2), residuals k / 64.  Padding channels of the sources are zero, as the engine keeps them; gate / residual
    channels beyond cout are NaN, which a kernel that reads them would carry into its output."""
    g = torch.Generator(device=device).manual_seed(seed)

    def ints(shape, lo, hi):
        return torch.randint(lo, hi, shape, generator=g, device=device).float()
    cin = sum(r for r, _ in sig.srcs)
    K = sig.k * sig.k * cin
    e = max(0, round(float(torch.tensor(73.0 * K ** 0.5).log2())))     # weight std ~ 1 / sqrt(K)
    ops = {'w': ints((sig.cout, cin, sig.k, sig.k), -255, 256) * 2.0 ** -e,
           'b': torch.randn(sig.cout, generator=g, device=device) * 0.1}
    ops['xs'] = []
    for r, a in sig.srcs:
        x = ints((H, W, a), -255, 256) / 128
        x[..., r:] = 0
        ops['xs'].append(x)
    Ho, Wo = (H + 2 * sig.pad - sig.k) // sig.stride + 1, (W + 2 * sig.pad - sig.k) // sig.stride + 1
    if sig.gate:
        ops['gate'] = torch.full((Ho, Wo, gate_cs or sig.cout), float('nan'), device=device)
        ops['gate'][..., :sig.cout] = ints((Ho, Wo, sig.cout), 0, 256) / 128
    if sig.res:
        ops['res'] = torch.full((Ho, Wo, res_cs or sig.cout), float('nan'), device=device)
        ops['res'][..., :sig.cout] = (torch.randn((Ho, Wo, sig.cout), generator=g, device=device) if sig.res == 'f32'
                                      else ints((Ho, Wo, sig.cout), -255, 256) / 64)
    return ops


def check(y, ref, base, out_dtype, what, tile=(16, 8), nb=None, ps=False):
    """assert |y - ref| <= bound element by element (y: the output's first cout channels) and that y is finite wherever
    ref is; prints the largest |y - ref| / bound.  A failure names where the failing elements sit within their tiles."""
    y = y.double()
    bnd = bound(ref, base, out_dtype)
    fin = torch.isfinite(ref)
    bad_fin = fin & ~torch.isfinite(y)
    ratio = torch.where(fin, (y - ref).abs() / bnd, torch.zeros_like(ref))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    print(f'[conv_fp64] {what}: max |y - ref| / bound = {worst:.4f}')
    if bad_fin.any() or not worst <= 1.0:
        pytest.fail(_explain(y, ref, ratio, bad_fin, out_dtype, what, tile, nb, ps))
    return worst


def _explain(y, ref, ratio, bad_fin, out_dtype, what, tile, nb, ps):
    bad = (ratio > 1.0) | bad_fin | torch.isnan(ratio)
    idx = bad.nonzero()
    i = int(bad_fin.flatten().nonzero()[0, 0]) if bad_fin.any() else int(torch.nan_to_num(ratio, nan=1e30).flatten().argmax())
    yy, xx, c = [int(v) for v in torch.unravel_index(torch.tensor(i), ratio.shape)]
    oy, ox, n = (yy // 2, xx // 2, 4 * c + 2 * (yy % 2) + xx % 2) if ps else (yy, xx, c)
    th, tw = tile
    e_ulp = ((y - ref).abs() / ulp(ref, out_dtype))[yy, xx, c] if out_dtype != torch.float32 else float('nan')
    msg = [f'{what}: {idx.shape[0]} of {ratio.numel()} elements outside the bound ({int(bad_fin.sum())} non-finite)',
           f'worst at output ({yy}, {xx}, channel {c}) = conv pixel ({oy}, {ox}) channel {n}: y = {float(y[yy, xx, c])!r}, '
           f'ref = {float(ref[yy, xx, c])!r}, {float(ratio[yy, xx, c]):.3g} x bound, {float(e_ulp):.3g} output ulp',
           f'within its {th} x {tw} tile: oy % {th} = {oy % th}, ox % {tw} = {ox % tw}' + (f', channel block {n // nb}' if nb else '')]
    if idx.shape[0]:
        py, px, pc = idx[:, 0], idx[:, 1], idx[:, 2]
        if ps:
            py, px, pc = py // 2, px // 2, 4 * pc + 2 * (idx[:, 0] % 2) + idx[:, 1] % 2
        for label, v in (('channels', pc), (f'oy % {th}', py % th), (f'ox % {tw}', px % tw)):
            u, cnt = torch.unique(v, return_counts=True)
            top = cnt.argsort(descending=True)[:8]
            msg.append(f'  failing elements by {label}: ' + ', '.join(f'{int(u[j])}: {int(cnt[j])}' for j in top))
    return '\n'.join(msg)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the bound separates a correct kernel from subtly wrong ones
# ------------------------------------------------------------------------------------------------------------------
def _fake_kernel(sig, ops, dt, mutation=None):
    """what the kernel computes, on the CPU: fp32 conv, fp32 epilogue, one rounding to the output type; `mutation` plants
    one defect: 'tap' drops tap (0, 2) of output channel 5, 'shift' takes the residual one pixel to the left, 'double'
    rounds the pre-activation to bf16 first.  (A second fp16 rounding in an fp16 conv stays below the bound wherever the
    worst-case accumulation term K u A is as large as the fp16 ulp, i.e. for K of a few hundred.)"""
    w = ops['w'].clone()
    if mutation == 'tap':
        w[5, :, 0, 2] = 0
    x = torch.cat([t[..., :r] for t, (r, _) in zip(ops['xs'], sig.srcs)], 2)
    y = F.conv2d(_nchw(x), w, ops['b'], stride=sig.stride, padding=sig.pad)
    if mutation == 'double':
        y = y.to(torch.bfloat16).float()
    y = _act(y, sig.act_pre)
    if sig.gate:
        y = y * _nchw(ops['gate'][..., :sig.cout])
    if sig.res:
        r = ops['res'][..., :sig.cout]
        y = y + _nchw(torch.roll(r, 1, dims=1) if mutation == 'shift' else r)
    y = _act(y, sig.act_post)
    if sig.ps:
        y = F.pixel_shuffle(y, 2)
    odt = torch.float32 if sig.out == 'f32' else dt
    return _nhwc(y).to(odt)


def _sig(name):
    return next(s for n, s, _ in ENGINE_CONVS if n == name)


@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('name', ['feat_fusion.1', 'main.0', 'upsample2', 'spynet.4+flow_up', 'conv_last', 'align.p_conv.4',
                                  'align.rb.conv2'])
def test_bound_passes_a_correct_kernel(name, dt):
    sig = _sig(name)
    ops = make_operands(sig, 20, 28, 'cpu', seed=zlib.crc32(name.encode()))
    ref, base = reference(sig, ops)
    y = _fake_kernel(sig, ops, dt)
    assert tuple(y.shape[:2]) == out_hw(sig, 20, 28)
    check(y, ref, base, y.dtype, f'fake kernel {name}', ps=sig.ps)


@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('mutation', ['tap', 'shift', 'double'])
def test_bound_fails_a_subtly_wrong_kernel(mutation, dt):
    sig = _sig('feat_fusion.1')
    ops = make_operands(sig, 20, 28, 'cpu', seed=7)
    ref, base = reference(sig, ops)
    y = _fake_kernel(sig, ops, dt, mutation)
    with pytest.raises(pytest.fail.Exception, match='outside the bound'):
        check(y, ref, base, dt, f'fake kernel with mutation {mutation}')


def test_ulp_spacing():
    v = torch.tensor([1.0, 1.5, 2.0, -3.0, 0.0, 2.0 ** -20, 6e4], dtype=torch.float64)
    assert ulp(v, torch.bfloat16).tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -6, 2.0 ** -6, 2.0 ** -133, 2.0 ** -27, 256.0]
    assert ulp(v, torch.float16).tolist() == [2.0 ** -10, 2.0 ** -10, 2.0 ** -9, 2.0 ** -9, 2.0 ** -24, 2.0 ** -24, 32.0]
    g = torch.Generator().manual_seed(0)
    for dt in (torch.bfloat16, torch.float16):
        # values of the type, normal and fp16-subnormal: one ulp up is the next value of the type, a quarter ulp rounds back
        x = (torch.randn(4000, generator=g) * torch.exp2(torch.randint(-22, 8, (4000,), generator=g).float())).abs().to(dt).double()
        x = x[x > 0]
        u = ulp(x, dt)
        assert torch.equal((x + u).to(dt).double(), x + u) and torch.equal((x + u / 4).to(dt).double(), x)


@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('layout', [0, 1, 2])
def test_packed_weights_are_the_weights_rounded_to_the_activation_type(layout, dt):
    """the tensor-core weight image holds w.to(activation type) and zeros: the reference takes the weights so rounded"""
    w = torch.randn(48, 56, 3, 3, generator=torch.Generator().manual_seed(1))
    img = (packing.pack_tc_sw32(w, [(8, 8), (48, 48)], dt, 48) if layout == 2
           else packing.pack_tc(w, [(8, 8), (48, 48)], dt, 48, layout))
    assert img.dtype == dt
    vals = img.float().flatten()
    assert torch.equal(vals[vals != 0].sort().values, w.to(dt).float().flatten().sort().values)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the list above is what the engine launches
# ------------------------------------------------------------------------------------------------------------------
def _signature(layer, src0, out, gate, res, act_pre, act_post, pixel_shuffle):
    assert gate is None or gate.shape[2] == layer.cout, (layer.name, 'gate channel stride')
    assert res is None or res.shape[2] == layer.cout, (layer.name, 'residual channel stride')
    return Sig(tuple(tuple(s) for s in layer.srcs), layer.cout, layer.weight.shape[2], layer.pad, layer.stride, act_pre,
               act_post, gate is not None, '' if res is None else ('f32' if res.dtype == torch.float32 else 'act'),
               bool(pixel_shuffle), 'f32' if out.dtype == torch.float32 else 'act', out.shape[2])


@functools.lru_cache(maxsize=None)
def kernel_of(weight_shape, srcs, stride, pad, act_dtype, prefer_tc):
    """the conv kernel the engine's packing picks for a layer: 'tc' (conv_tc.cu) or 'simt' (conv_simt.cu), from
    packing.pack_conv_uncached on zero weights on the CPU"""
    w = torch.zeros(weight_shape)
    pc = packing.pack_conv_uncached('kernel_of', w, torch.zeros(weight_shape[0]), [tuple(s) for s in srcs], stride, pad,
                                    act_dtype, 'cpu', prefer_tc)
    return 'tc' if pc.impl == IMPL_TC else 'simt'


def _recording_ops(compute, kernels=False):
    """OracleOps whose conv2d records (signature, input H, W) of every call; compute=False: every other operator (and the conv
    itself) is a no-op, so that a full-size schedule runs on the CPU in a second.  kernels=True: the record is (signature,
    kernel, precision class, input H, W), with the kernel of kernel_of and the class '16' (bf16 / fp16 activations) or '32'"""
    from oracle.oracle_ops import OracleOps

    class Recording(OracleOps):
        def __init__(self):
            self.seen = collections.Counter()

        def pack_conv(self, name, weight, bias, srcs, stride, pad, act_dtype, device, prefer_tc, bias_add=0.0):
            layer = super().pack_conv(name, weight, bias, srcs, stride, pad, act_dtype, device, prefer_tc, bias_add)
            if kernels:
                layer.kernel = kernel_of(tuple(weight.shape), tuple(tuple(s) for s in srcs), stride, pad, act_dtype,
                                         bool(prefer_tc))
                layer.prec = '32' if act_dtype == torch.float32 else '16'
            return layer

        def conv2d(self, layer, src0, src1, out, gate=None, res=None, act_pre=0, act_post=0, pixel_shuffle=False):
            sig = _signature(layer, src0, out, gate, res, act_pre, act_post, pixel_shuffle)
            self.seen[(sig, layer.kernel, layer.prec, tuple(src0.shape[:2])) if kernels else (sig, tuple(src0.shape[:2]))] += 1
            if compute:
                super().conv2d(layer, src0, src1, out, gate, res, act_pre, act_post, pixel_shuffle)

    if compute:
        return Recording()

    class ShapesOnly(Recording):
        def __getattribute__(self, name):
            if name in ('conv2d', 'pack_conv', 'seen') or name.startswith('__'):
                return object.__getattribute__(self, name)
            return lambda *a, **k: 0
    return ShapesOnly()


def _run_engine(ops, h, w, **over):
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip, sliding_windows
    cfg = get_config('config_RefVSR_MFID', device='cpu', b200_precision='bf16', **over)
    net = SRNet(cfg).eval()
    seeded_test_weights(net, seed=5)
    net.Network.set_ops(ops)
    lrs, refs = make_clip(cfg.frame_num, h, w, 1, seed=5)
    for n, (k, wl, wr, first) in enumerate(sliding_windows(lrs, refs, cfg.frame_num)):
        net(wl, wr, first)
        if n == 1:
            break
    return ops.seen


_X2_MODEL = dict(scale=2, matching_ksize=4)


def test_engine_convs_are_all_listed():
    """a small x4 and x2 case through the engine (OracleOps computes): every conv signature it launches is in ENGINE_CONVS"""
    listed = {s for _, s, _ in ENGINE_CONVS}
    seen = set()
    for over in (dict(num_blocks=1), dict(num_blocks=1, **_X2_MODEL)):
        seen |= {s for s, _ in _run_engine(_recording_ops(True), 24, 32, **over)}
    missing = seen - listed
    assert not missing, f'conv signatures the engine launches and ENGINE_CONVS does not list: {sorted(missing)}'
    assert len(seen) == len(listed) == len(ENGINE_CONVS)


def test_engine_geometries_are_all_listed():
    """the full-size x4 (LR 270x480) and x2 (LR 540x960) schedules, shapes only: every (signature, input geometry) they launch
    is a case of test_engine_conv"""
    listed = {(s, g) for _, s, geoms in ENGINE_CONVS for g in geoms}
    seen = set(_run_engine(_recording_ops(False), 270, 480)) | set(_run_engine(_recording_ops(False), 540, 960, **_X2_MODEL))
    missing = seen - listed
    assert not missing, f'(signature, geometry) pairs the engine launches and ENGINE_CONVS does not list: {sorted(missing)}'


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
DTYPES = ((torch.bfloat16, 'bf16'), (torch.float16, 'fp16'))
_REF = {}


def _reference_cached(key, sig, ops):
    """float64 references of the most recent case (one full-size case holds a few GB); reused across types and grid caps"""
    if key not in _REF:
        _REF.clear()
        torch.cuda.empty_cache()
        _REF[key] = reference(sig, ops)
    return _REF[key]


def run_case(cuda_ops, name, sig, H, W, caps=(0,), layout=None, gate_cs=None, res_cs=None, out_cs=None, out_off=0):
    """the conv `sig` on an H x W input through CudaOps.conv2d in bf16 and fp16 at each grid cap, against the float64
    reference.  The output sits `out_off` elements into a NaN-filled buffer with GUARD NaNs on either side; output channels
    at or beyond cout of a wider buffer (out_cs) must stay NaN, as must the guards."""
    ops = make_operands(sig, H, W, 'cuda', zlib.crc32(f'{name}/{H}x{W}'.encode()), gate_cs, res_cs)
    ref, base = _reference_cached((name, H, W, gate_cs, res_cs), sig, ops)
    Ho, Wo = out_hw(sig, H, W)
    ce = sig.cout // 4 if sig.ps else sig.cout
    ocs = out_cs or sig.out_cs
    worst = {}
    for dt, dtn in DTYPES:
        layer = packing.pack_conv_uncached(name, ops['w'], ops['b'], list(sig.srcs), sig.stride, sig.pad, dt, 'cuda', True,
                                           tc_layout=layout)
        assert layer.impl == (IMPL_TC if sig.stride == 1 else IMPL_SIMT), (name, layer.impl)
        xs = [x.to(dt) for x in ops['xs']]
        gate = ops['gate'].to(dt) if sig.gate else None
        res = ops['res'].to(torch.float32 if sig.res == 'f32' else dt) if sig.res else None
        odt = torch.float32 if sig.out == 'f32' else dt
        n = Ho * Wo * ocs
        buf = torch.empty(n + 2 * GUARD + out_off, dtype=odt, device='cuda')
        out = buf[GUARD + out_off:GUARD + out_off + n].view(Ho, Wo, ocs)
        x1 = xs[1] if len(xs) > 1 else None
        tile = (16, 8) if layer.layout in (1, 3) else (8, 16)
        for cap in caps:
            buf.fill_(float('nan'))
            old = cuda_ops.set_conv_cta_cap(cap)
            try:
                cuda_ops.conv2d(layer, xs[0], x1, out, gate=gate, res=res, act_pre=sig.act_pre, act_post=sig.act_post,
                                pixel_shuffle=sig.ps)
                torch.cuda.synchronize()
            finally:
                cuda_ops.set_conv_cta_cap(old)
            what = f'{name} {H}x{W} {dtn} cap {cap}'
            assert torch.isnan(buf[:GUARD + out_off]).all() and torch.isnan(buf[GUARD + out_off + n:]).all(), \
                (what, 'wrote outside its output')
            assert torch.isnan(out[..., ce:]).all(), (what, 'wrote output-buffer channels at or beyond cout')
            worst[(dtn, cap)] = check(out[..., :ce], ref, base, odt, what, tile, layer.nb or None, sig.ps)
    return worst


_ENGINE_CASES = [(n, s, g) for n, s, geoms in ENGINE_CONVS for g in geoms]


@pytest.mark.gpu
@pytest.mark.parametrize('case', _ENGINE_CASES, ids=[f'{n}-{g[0]}x{g[1]}' for n, _, g in _ENGINE_CASES])
def test_engine_conv(cuda_ops, case):
    name, sig, (H, W) = case
    run_case(cuda_ops, name, sig, H, W)


RES48 = _sig('conv48.res')
LRELU48 = _sig('conv48.lrelu')
# launch-plan branches of the tensor-core kernel (conv_tc.cu, plan_tc), forced at full-size maps so that every ring wraps
# many times: (id, signature, input geometry, run_case options)
BRANCH_CASES = [
    ('layout0', RES48, (270, 480), dict(layout=0, expect_mode=0, expect_depth=2)),
    ('layout1', RES48, (270, 480), dict(layout=1, expect_mode=1, expect_depth=2)),
    ('layout2', RES48, (270, 480), dict(layout=2, expect_mode=2, expect_depth=2)),
    ('layout3', RES48, (270, 480), dict(layout=3, expect_mode=1, expect_depth=2)),
    ('taps-runtime-8+48', _sig('main.0'), (270, 480), dict(expect_mode=1)),
    ('taps-fixed-48+48', _sig('feat_fusion.0'), (270, 480), dict(expect_mode=1)),
    ('no-epi-tma-f32-residual', RES48._replace(res='f32', out='f32'), (270, 480), dict(expect_depth=0)),
    ('no-epi-tma-gate-cs52', _sig('feat_fusion.1'), (270, 480), dict(gate_cs=52, expect_depth=0)),
    ('no-epi-tma-res-cs52', RES48, (270, 480), dict(res_cs=52, expect_depth=0)),
    ('epi-depth2-res', RES48, (270, 480), dict(expect_depth=2)),
    ('epi-depth2-gate', LRELU48._replace(gate=True), (270, 480), dict(expect_depth=2)),
    ('epi-depth1-gate+res', _sig('feat_fusion.1'), (270, 480), dict(expect_depth=1)),
    ('no-out-tma-offset2B', LRELU48, (270, 480), dict(out_off=1)),
    ('no-ps-vec-offset2B', _sig('upsample1'), (270, 480), dict(out_off=1)),
    ('out-cs56', LRELU48, (270, 480), dict(out_cs=56)),
    ('out-cs56-res', RES48, (270, 480), dict(out_cs=56)),
    ('cout192-nb96-two-blocks', LRELU48._replace(cout=192, out_cs=192), (270, 480), dict(expect_mode=1)),
    ('ragged-271x483-res', RES48, (271, 483), {}),
    ('ragged-271x483-gate+res', _sig('feat_fusion.1'), (271, 483), {}),
    ('ragged-271x483-upsample1', _sig('upsample1'), (271, 483), {}),
    ('ragged-271x483-f32-out', _sig('conv_last'), (271, 483), {}),
]


H100_SMEM, H100_SMS = 232448, 132


def test_branch_cases_take_their_branch():
    """rv_conv2d_tc_plan / rv_conv2d_tc_epi_depth for each branch case on an H100, with pointers aligned as run_case's
    tensors are (fresh allocations; the output GUARD + out_off elements into its buffer): the layout mode and the number of
    gate / residual TMA buffers per consumer (0: the epilogue loads them itself) are the ones the case is named for"""
    from refvsr_b200.lib import DTYPE_CODE, load_library, rv_conv_desc
    lib = load_library()
    base = 1 << 20
    for name, sig, (H, W), opt in BRANCH_CASES:
        want_mode, want_depth = opt.get('expect_mode'), opt.get('expect_depth')
        for dt in (torch.bfloat16, torch.float16):
            w = torch.zeros(sig.cout, sum(r for r, _ in sig.srcs), sig.k, sig.k)
            layer = packing.pack_conv_uncached(name, w, torch.zeros(sig.cout), list(sig.srcs), 1, sig.pad, dt, 'cpu', True,
                                               tc_layout=opt.get('layout'))
            odt = torch.float32 if sig.out == 'f32' else dt
            d = rv_conv_desc()
            d.src0, d.src1 = base, (base if len(sig.srcs) > 1 else None)
            d.c0, d.c1 = layer.alloc0, layer.alloc1
            d.in_dtype, d.H, d.W = DTYPE_CODE[dt], H, W
            d.wpack, d.bias, d.cout, d.kh, d.kw, d.stride, d.pad = base, base, sig.cout, sig.k, sig.k, 1, sig.pad
            d.act_pre, d.act_post = sig.act_pre, sig.act_post
            d.gate, d.gate_cs = (base, opt.get('gate_cs') or sig.cout) if sig.gate else (None, 0)
            d.res, d.res_cs = (base, opt.get('res_cs') or sig.cout) if sig.res else (None, 0)
            d.res_dtype = DTYPE_CODE[torch.float32 if sig.res == 'f32' else dt] if sig.res else 0
            d.out = base + (GUARD + opt.get('out_off', 0)) * odt.itemsize
            d.out_cs, d.out_dtype = opt.get('out_cs') or sig.out_cs, DTYPE_CODE[odt]
            d.pixel_shuffle, d.impl, d.nb, d.k_real, d.layout = int(sig.ps), layer.impl, layer.nb, layer.k_real, layer.layout
            plan, depth = (C.c_int32 * 8)(), C.c_int32(-1)
            assert lib.rv_conv2d_tc_plan(C.byref(d), H100_SMEM, H100_SMS, plan) == 0, lib.rv_last_error()
            assert lib.rv_conv2d_tc_epi_depth(C.byref(d), H100_SMEM, H100_SMS, C.byref(depth)) == 0, lib.rv_last_error()
            assert want_mode is None or plan[0] == want_mode, (name, 'layout mode', plan[0])
            assert want_depth is None or depth.value == want_depth, (name, 'gate / residual buffers per consumer', depth.value)
            if 'two-blocks' in name:
                assert plan[6] == 96 and sig.cout == 2 * 96


@pytest.mark.gpu
@pytest.mark.parametrize('cap', [0, 7], ids=['cap0', 'cap7'])
@pytest.mark.parametrize('case', BRANCH_CASES, ids=[c[0] for c in BRANCH_CASES])
def test_plan_branch(cuda_ops, case, cap):
    """each branch at grid cap 0 (one CTA per SM) and 7 (few CTAs, each with many tiles)"""
    name, sig, (H, W), opt = case
    opt = {k: v for k, v in opt.items() if not k.startswith('expect_')}
    run_case(cuda_ops, name, sig, H, W, caps=(cap,), **opt)
