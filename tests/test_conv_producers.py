"""Per-consumer producer warps of the tensor-core convolution (conv_tc.cu): producer warp c fills consumer c's A ring and
warp 2 + c its ring of gate / residual buffers.

Without a GPU: every conv shape of a RefVSR_MFID window plans within the H100's budget, and the gate / residual convs keep
two A slots per consumer with their epilogue buffers (rv_conv2d_tc_plan, rv_conv2d_tc_epi_depth).
With a GPU: outputs do not depend on the grid.  A capped grid changes which consumer and which producer warps handle each
tile and how often each ring wraps, so the same conv at rv_set_conv_cta_cap 0, 7 and 1 must give the same bits; at one to
three tiles some consumers and their producer warps have no work, which must neither hang nor write anything."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from refvsr_b200 import packing
from refvsr_b200.lib import ACT_RELU

H100_SMEM, H100_SMS = 232448, 132
GEOMS = ((270, 480), (540, 960), (1080, 1920), (37, 53))

# conv shapes of a RefVSR_MFID window: (name, srcs [(real, alloc)], cout, k, pad, pixel shuffle, gate, residual, fp32 out)
WINDOW_CONVS = [
    ('resblock conv1', [(48, 48)], 48, 3, 1, False, False, False, False),
    ('resblock conv2', [(48, 48)], 48, 3, 1, False, False, True, False),
    ('feat_fusion.0', [(48, 48), (48, 48)], 48, 3, 1, False, False, False, False),
    ('feat_fusion.1', [(48, 48)], 48, 3, 1, False, True, True, False),
    ('conf_fusion.0', [(2, 8)], 16, 3, 1, False, False, False, False),
    ('conf_fusion.1', [(16, 16)], 48, 3, 1, False, False, False, False),
    ('in_conv', [(3, 8), (48, 48)], 48, 3, 1, False, False, False, False),
    ('ref_encoder1.0', [(3, 8)], 48, 3, 1, False, False, False, False),
    ('upsample', [(48, 48)], 192, 3, 1, True, False, False, False),
    ('fusion_UP', [(48, 48), (48, 48)], 48, 3, 0, False, False, False, False),
    ('conv_last', [(48, 48)], 3, 3, 1, False, False, True, True),
    ('feature_extract.0', [(3, 8)], 64, 3, 1, False, False, False, False),
    ('feature_extract.2', [(64, 64)], 64, 3, 1, False, False, False, False),
    ('feature_extract.5', [(64, 64)], 128, 3, 1, False, False, False, False),
    ('map128', [(128, 128)], 16, 1, 0, False, False, False, False),
    ('spynet.0', [(8, 8)], 32, 7, 3, False, False, False, False),
    ('spynet.1', [(32, 32)], 64, 7, 3, False, False, False, False),
    ('spynet.2', [(64, 64)], 32, 7, 3, False, False, False, False),
    ('spynet.3', [(32, 32)], 16, 7, 3, False, False, False, False),
    ('spynet.4', [(16, 16)], 2, 7, 3, False, False, False, False),
]


def _desc(srcs, cout, k, pad, ps, gate, res, out_f32, H, W):
    from refvsr_b200.lib import rv_conv_desc
    buf = (C.c_char * 4096)()
    ptr = (C.addressof(buf) + 255) & ~255
    nb = packing.choose_nb(cout)
    d = rv_conv_desc()
    d.src0, d.src1 = ptr, (ptr if len(srcs) > 1 else None)
    d.c0, d.c1 = srcs[0][1], (srcs[1][1] if len(srcs) > 1 else 0)
    d.in_dtype, d.H, d.W = 2, H, W
    d.wpack, d.bias, d.cout, d.kh, d.kw, d.stride, d.pad = ptr, ptr, cout, k, k, 1, pad
    d.gate, d.gate_cs = (ptr if gate else None), (cout if gate else 0)
    d.res, d.res_cs, d.res_dtype = (ptr if res else None), (cout if res else 0), (0 if out_f32 else 2)
    d.out, d.out_cs, d.out_dtype = ptr, (cout // 4 if ps else (4 if out_f32 else cout)), (0 if out_f32 else 2)
    d.pixel_shuffle, d.impl, d.nb = int(ps), 1, nb
    d.k_real, d.layout = k * k * sum(r for r, _ in srcs), packing.choose_layout(k, k, srcs, nb)
    return d, buf


def _plan(lib, d):
    out, depth = (C.c_int32 * 8)(), C.c_int32(-1)
    rc = lib.rv_conv2d_tc_plan(C.byref(d), H100_SMEM, H100_SMS, out)
    assert rc == 0, lib.rv_last_error()
    assert lib.rv_conv2d_tc_epi_depth(C.byref(d), H100_SMEM, H100_SMS, C.byref(depth)) == 0, lib.rv_last_error()
    return list(out), depth.value


def test_window_convs_plan_within_the_h100_budget():
    from refvsr_b200.lib import load_library
    lib = load_library()
    for name, srcs, cout, k, pad, ps, gate, res, out_f32 in WINDOW_CONVS:
        for H, W in GEOMS:
            d, _keep = _desc(srcs, cout, k, pad, ps, gate, res, out_f32, H, W)
            (mode, slots, resident, S, ncons, nacc, nb, smem), depth = _plan(lib, d)
            assert ncons == nacc == 2 and slots >= 1 and smem <= H100_SMEM, (name, H, W, slots, smem)
            assert depth in (0, 1, 2), (name, depth)
            assert depth == 0 or (gate or res), (name, depth)


def test_gate_and_residual_convs_get_their_epilogue_ring():
    """16-bit gate / residual convs at NB 48: two A slots per consumer; a residual or a gate alone also gets two epilogue
    buffers per consumer.  Gate + residual cannot hold both next to the output buffer, and the plan keeps the two A slots."""
    from refvsr_b200.lib import load_library
    lib = load_library()
    for gate, res, want in ((False, True, 2), (True, False, 2), (True, True, 1)):
        for H, W in GEOMS:
            d, _keep = _desc([(48, 48)], 48, 3, 1, False, gate, res, False, H, W)
            (mode, slots, *_), depth = _plan(lib, d)
            assert slots >= 2 and depth == want, (gate, res, H, W, slots, depth)
    d, _keep = _desc([(48, 48)], 48, 3, 1, False, False, False, False, 270, 480)
    assert _plan(lib, d)[1] == 0          # no gate / residual: no epilogue buffers


# ------------------------------------------------------------------------------------------------------------------
# GPU: bit-equal outputs whatever the grid
# ------------------------------------------------------------------------------------------------------------------
# (name, srcs, cout, pixel shuffle, gate, residual, fp32 residual / output)
GPU_CONVS = [
    ('gate+res', [(48, 48)], 48, False, True, True, False),
    ('res', [(48, 48)], 48, False, False, True, False),
    ('plain', [(48, 48)], 48, False, False, False, False),
    ('two-source', [(48, 48), (48, 48)], 48, False, False, False, False),
    ('fp32 res', [(48, 48)], 3, False, False, True, True),
    ('pixel shuffle', [(48, 48)], 192, True, False, False, False),
]
GUARD = 4096


class Conv:
    def __init__(self, ops, srcs, cout, ps, gate, res, f32, H, W, dt=torch.float16, seed=0):
        gen = torch.Generator().manual_seed(seed)
        cin = sum(r for r, _ in srcs)
        self.w = torch.randn(cout, cin, 3, 3, generator=gen) * 0.05
        self.b = torch.randn(cout, generator=gen) * 0.1
        self.layer = packing.pack_conv('x', self.w, self.b, srcs, 1, 1, dt, 'cuda', True)
        self.xs = [torch.randn(H, W, a, generator=gen).to(dt).cuda() for _, a in srcs]
        for x, (r, a) in zip(self.xs, srcs):
            x[..., r:] = 0
        self.gate = torch.rand(H, W, cout, generator=gen).to(dt).cuda() if gate else None
        odt = torch.float32 if f32 else dt
        self.res = torch.randn(H, W, cout, generator=gen).to(odt).cuda() if res else None
        self.oshape = (2 * H, 2 * W, cout // 4) if ps else (H, W, cout)
        self.odt, self.ps, self.srcs, self.ops = odt, ps, srcs, ops

    def run(self, cap):
        """output, and whether the NaN guards on either side of it are intact"""
        n = 1
        for s in self.oshape:
            n *= s
        buf = torch.full((n + 2 * GUARD,), float('nan'), dtype=self.odt, device='cuda')
        out = buf[GUARD:GUARD + n].view(self.oshape)
        old = self.ops.set_conv_cta_cap(cap)
        try:
            self.ops.conv2d(self.layer, self.xs[0], self.xs[1] if len(self.xs) > 1 else None, out, gate=self.gate,
                            res=self.res, act_pre=ACT_RELU, pixel_shuffle=self.ps)
            torch.cuda.synchronize()
        finally:
            self.ops.set_conv_cta_cap(old)
        guards = torch.cat([buf[:GUARD], buf[GUARD + n:]])
        return out.clone(), bool(torch.isnan(guards).all())

    def reference(self):
        x = torch.cat([x[..., :r].float() for x, (r, _) in zip(self.xs, self.srcs)], 2).cpu().permute(2, 0, 1)[None]
        w = self.w.to(self.xs[0].dtype).float()
        y = F.conv2d(x, w, self.b.float(), padding=1)[0].permute(1, 2, 0)
        y = torch.relu(y)
        if self.gate is not None:
            y = y * self.gate.float().cpu()
        if self.res is not None:
            y = y + self.res.float().cpu()
        if self.ps:
            y = F.pixel_shuffle(y.permute(2, 0, 1)[None], 2)[0].permute(1, 2, 0)
        return y


@pytest.mark.gpu
@pytest.mark.parametrize('geom', [(270, 480), (37, 53)], ids=['270x480', '37x53'])
@pytest.mark.parametrize('case', GPU_CONVS, ids=[c[0] for c in GPU_CONVS])
def test_outputs_do_not_depend_on_the_grid(cuda_ops, case, geom):
    name, srcs, cout, ps, gate, res, f32 = case
    conv = Conv(cuda_ops, srcs, cout, ps, gate, res, f32, *geom)
    base, ok = conv.run(0)
    assert ok and not torch.isnan(base).any(), name
    for cap in (7, 1):
        y, ok = conv.run(cap)
        assert ok, (name, cap, 'wrote outside its output')
        assert torch.equal(y, base), (name, cap, (y.float() - base.float()).abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize('hw', [(16, 8), (16, 16), (16, 24), (9, 5), (20, 13)], ids=['1tile', '2tiles', '3tiles', '1ragged', '4ragged'])
@pytest.mark.parametrize('case', GPU_CONVS, ids=[c[0] for c in GPU_CONVS])
def test_tiny_grids_with_idle_consumers(cuda_ops, case, hw):
    """one to three tiles: at cap 0 every CTA has one tile, so consumer 1 and its producer warps have none; at cap 1 one
    CTA takes all of them.  Every output element is written once, nothing outside, and the values match F.conv2d."""
    name, srcs, cout, ps, gate, res, f32 = case
    conv = Conv(cuda_ops, srcs, cout, ps, gate, res, f32, *hw, seed=1)
    base, ok = conv.run(0)
    assert ok and not torch.isnan(base).any(), name
    y, ok = conv.run(1)
    assert ok and torch.equal(y, base), name
    ref = conv.reference()
    err = (base.float().cpu() - ref).abs().max().item()
    assert err <= 1e-2 * max(1.0, ref.abs().max().item()), (name, err)

