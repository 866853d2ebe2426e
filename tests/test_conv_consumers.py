"""Three consumer warpgroups in the single-source 48 -> 48 3x3 tensor-core conv (conv_tc.cu, conv_tc3_kernel).

On the CPU, with an H100's limits: the plan (rv_conv2d_tc_consumers) sends exactly the plain and residual 48 -> 48 convs to
three consumers, within the opt-in shared memory; a smaller budget, a gate, two sources, other NB or an fp32 output keep
two, and rv_set_conv_consumers(2) forces two.  The three-consumer kernels issue each tile as one 54-HGMMA batch and do not
spill.  With a GPU: the three-consumer kernel gives the bits of the forced two-consumer kernel for every epilogue variant,
in bf16 and fp16, at the window's map sizes and a ragged one, at grid caps 0, 7 and 1 (one CTA walks every tile on all
three consumers), and batched with loud data in the neighbouring image.  (test_conv_fp64.test_engine_conv holds the
default plan, three consumers included, to the fp64 element-wise bound.)"""
import ctypes as C
import os
import re
import subprocess
import zlib
from collections import defaultdict

import pytest
import torch

from refvsr_b200 import packing
from refvsr_b200.lib import ACT_CLAMP3, ACT_LRELU01, ACT_LRELU02, ACT_NONE, ACT_RELU
from test_conv_fp64 import DTYPES, H100_SMEM, H100_SMS, Sig, _sig, make_operands, out_hw
from test_conv_sass import LIB, _cuobjdump

N, R, L1, L2, C3 = ACT_NONE, ACT_RELU, ACT_LRELU01, ACT_LRELU02, ACT_CLAMP3
_INT = {2: torch.int16, 4: torch.int32}

# (id, signature, consumers on an H100)
PLAN_CASES = [
    ('plain', _sig('conv48.lrelu'), 3),
    ('residual', _sig('conv48.res'), 3),
    ('conv_hr', _sig('conv_hr'), 3),
    ('gate', _sig('conv48.lrelu')._replace(gate=True), 2),
    ('gate+res', _sig('feat_fusion.1'), 2),
    ('two-source', _sig('feat_fusion.0'), 2),
    ('upsample', _sig('upsample1'), 2),
    ('fp32-out', _sig('conv_last'), 2),
    ('nb16', Sig(((16, 16),), 16, 3, 1, 1, R, N, False, '', False, 'act', 16), 2),
]


def _desc(sig, H, W, dt, n=1):
    from refvsr_b200.lib import DTYPE_CODE, rv_conv_desc
    base = 1 << 20
    w = torch.zeros(sig.cout, sum(r for r, _ in sig.srcs), sig.k, sig.k)
    layer = packing.pack_conv_uncached('x', w, torch.zeros(sig.cout), list(sig.srcs), 1, sig.pad, dt, 'cpu', True, ps_rows=sig.ps)
    odt = torch.float32 if sig.out == 'f32' else dt
    d = rv_conv_desc()
    d.src0, d.src1 = base, (base if len(sig.srcs) > 1 else None)
    d.c0, d.c1 = layer.alloc0, layer.alloc1
    d.in_dtype, d.H, d.W = DTYPE_CODE[dt], H, W
    d.wpack, d.bias, d.cout, d.kh, d.kw, d.stride, d.pad = base, base, sig.cout, sig.k, sig.k, 1, sig.pad
    d.act_pre, d.act_post = sig.act_pre, sig.act_post
    d.gate, d.gate_cs = (base, sig.cout) if sig.gate else (None, 0)
    d.res, d.res_cs = (base, sig.cout) if sig.res else (None, 0)
    d.res_dtype = DTYPE_CODE[torch.float32 if sig.res == 'f32' else dt] if sig.res else 0
    d.out, d.out_cs, d.out_dtype = base, sig.out_cs, DTYPE_CODE[odt]
    d.pixel_shuffle, d.impl, d.nb, d.k_real, d.layout = int(sig.ps), layer.impl, layer.nb, layer.k_real, layer.layout
    d.ps_order = getattr(layer, 'ps_order', 0)
    d.n = n
    if n > 1:
        d.bs_src0 = d.bs_src1 = d.bs_gate = d.bs_res = d.bs_out = H * W * 256
    return d


def _consumers(lib, d, smem=H100_SMEM):
    out = (C.c_int32 * 4)()
    assert lib.rv_conv2d_tc_consumers(C.byref(d), smem, H100_SMS, out) == 0, lib.rv_last_error()
    return list(out)


@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
def test_plan_sends_the_48_channel_single_source_convs_to_three_consumers(dt):
    from refvsr_b200.lib import load_library
    lib = load_library()
    for name, sig, want in PLAN_CASES:
        for H, W in ((270, 480), (540, 960), (1080, 1920), (271, 483)):
            for n in (1, 2):
                ncons, slots, depth, smem = _consumers(lib, _desc(sig, H, W, dt, n))
                assert ncons == want and slots >= 1 and smem <= H100_SMEM, (name, H, W, n, ncons, slots, smem)
                if ncons == 3:
                    # weights, one A slot, the output buffer and (residual) one residual buffer per consumer
                    assert slots == 1 and depth == (1 if sig.res else 0), (name, slots, depth)
                    assert smem == 1024 + 9 * 48 * 128 + 3 * (23552 + 12288 + (12288 if sig.res else 0)), (name, smem)


def test_smaller_budget_and_the_switch_keep_two_consumers():
    from refvsr_b200.lib import load_library
    lib = load_library()
    for name, sig, want in PLAN_CASES[:3]:
        d = _desc(sig, 270, 480, torch.bfloat16)
        assert _consumers(lib, d)[0] == 3, name
        # the A slots, output and residual buffers of three consumers no longer fit next to the weights
        assert _consumers(lib, d, smem=163840)[0] == 2, name
        old = lib.rv_set_conv_consumers(2)
        try:
            assert _consumers(lib, d)[0] == 2, name
        finally:
            lib.rv_set_conv_consumers(old)
        assert _consumers(lib, d)[0] == 3, name


def test_three_consumer_kernels_issue_one_batch_per_tile_and_do_not_spill():
    tool = _cuobjdump()
    if not os.path.isfile(LIB) or tool is None:
        pytest.skip('library or cuobjdump missing')
    sass = subprocess.run([tool, '-sass', LIB], capture_output=True, text=True, check=True).stdout
    res = subprocess.run([tool, '-res-usage', LIB], capture_output=True, text=True, check=True).stdout
    funcs, cur = defaultdict(list), None
    for line in sass.splitlines():
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            cur = m.group(1)
        elif cur and re.search(r'/\*[0-9a-f]{4,}\*/', line):
            funcs[cur].append(line)
    stack = {m.group(1): int(m.group(2)) for m in re.finditer(r'Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)', res)}
    names = [f for f in funcs if 'conv_tc3_kernel' in f]
    assert len(names) == 4 and any('bfloat16' in f for f in names) and any('6__half' in f for f in names), names
    for name in names:
        assert stack.get(name) == 0 and not any(re.search(r'\b(LDL|STL)\b', line) for line in funcs[name]), name
        stages, cur = [], None
        for line in funcs[name]:
            if 'WARPGROUP.ARRIVE' in line:
                cur = []
                stages.append(cur)
            elif 'HGMMA' in line:
                cur.append('gsb0' in line)
        assert stages and all(len(st) == 54 and st[-1] and not any(st[:-1]) for st in stages), name


# ------------------------------------------------------------------------------------------------------------------
# GPU: three consumers against the forced two-consumer kernel, bit for bit
# ------------------------------------------------------------------------------------------------------------------
GPU_CASES = [
    ('plain', _sig('conv48.lrelu')),
    ('residual', _sig('conv48.res')),
    ('residual-lrelu-post', _sig('conv48.res')._replace(act_post=L2)),
    ('relu-clamp3', _sig('conv48.relu')._replace(act_post=C3)),
    ('residual-clamp3', _sig('conv48.res')._replace(act_pre=L1, act_post=C3)),
    ('gate', _sig('conv48.lrelu')._replace(gate=True)),
    ('gate+res', _sig('feat_fusion.1')),
]
GEOMS = [(270, 480), (540, 960), (1080, 1920), (271, 483)]


def _run(cuda_ops, layer, sig, xs, gate, res, out, cap, consumers):
    old_cap, old_cons = cuda_ops.set_conv_cta_cap(cap), cuda_ops.set_conv_consumers(consumers)
    try:
        cuda_ops.conv2d(layer, xs, None, out, gate=gate, res=res, act_pre=sig.act_pre, act_post=sig.act_post)
        torch.cuda.synchronize()
    finally:
        cuda_ops.set_conv_cta_cap(old_cap)
        cuda_ops.set_conv_consumers(old_cons)


@pytest.mark.gpu
@pytest.mark.parametrize('hw', GEOMS, ids=[f'{h}x{w}' for h, w in GEOMS])
@pytest.mark.parametrize('case', GPU_CASES, ids=[c[0] for c in GPU_CASES])
def test_three_consumers_equal_two(cuda_ops, case, hw):
    name, sig = case
    H, W = hw
    Ho, Wo = out_hw(sig, H, W)
    for n in (1, 2):
        seed = zlib.crc32(f'{name}/{H}x{W}/consumers'.encode())
        per = [make_operands(sig, H, W, 'cuda', seed + i) for i in range(n)]
        for dt, dtn in DTYPES:
            layer = packing.pack_conv_uncached(name, per[0]['w'], per[0]['b'], list(sig.srcs), 1, sig.pad, dt, 'cuda', True)
            # the odd images hold inputs 64 x larger: a tile that read across an image border would change its neighbour
            xs = torch.stack([p['xs'][0] * (64.0 if i % 2 else 1.0) for i, p in enumerate(per)]).to(dt)
            gate = torch.stack([p['gate'] for p in per]).to(dt) if sig.gate else None
            res = torch.stack([p['res'] for p in per]).to(dt) if sig.res else None
            if n == 1:
                xs, gate, res = xs[0], None if gate is None else gate[0], None if res is None else res[0]
            shape = (n, Ho, Wo, sig.out_cs) if n > 1 else (Ho, Wo, sig.out_cs)
            for cap in (0, 7, 1):
                two = torch.full(shape, float('nan'), dtype=dt, device='cuda')
                three = torch.full_like(two, float('nan'))
                _run(cuda_ops, layer, sig, xs, gate, res, two, cap, 2)
                _run(cuda_ops, layer, sig, xs, gate, res, three, cap, 0)
                assert torch.equal(two.view(_INT[2]), three.view(_INT[2])), f'{name} {H}x{W} n={n} {dtn} cap {cap}'
