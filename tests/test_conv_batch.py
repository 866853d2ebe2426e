"""rv_conv2d with n > 1 images (rv_conv_desc::n and the image strides): the batched launch against one launch per image, bit
for bit, for every conv signature the engine launches (test_conv_fp64.ENGINE_CONVS), with distinct data in every image.  On
the CPU: the ctypes mirror of the extended descriptor against the compiled header, and the host-only launch plan with a
batch."""
import ctypes as C
import os
import shutil
import subprocess
import zlib

import pytest
import torch

from refvsr_b200 import packing
from test_conv_fp64 import BRANCH_CASES, DTYPES, ENGINE_CONVS, H100_SMEM, H100_SMS, _sig, make_operands, out_hw

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_INT = {2: torch.int16, 4: torch.int32}


def _bits(t):
    return t.view(_INT[t.element_size()])


def run_batch(cuda_ops, name, sig, H, W, n, cap=0, loud=False, smem_cap=0):
    """the conv on n different H x W images as ONE launch (n, H, W, C) and as n launches, at grid cap `cap`, in bf16 and fp16.
    loud: the odd images hold inputs 64 x larger, so a tile that read across an image border would change its neighbour's
    output.  Output channels beyond cout start as NaN in both runs and must come out the same."""
    seed = zlib.crc32(f'{name}/{H}x{W}/batch'.encode())
    per = [make_operands(sig, H, W, 'cuda', seed + i) for i in range(n)]
    Ho, Wo = out_hw(sig, H, W)
    for dt, dtn in DTYPES:
        layer = packing.pack_conv_uncached(name, per[0]['w'], per[0]['b'], list(sig.srcs), sig.stride, sig.pad, dt, 'cuda', True,
                                           ps_rows=sig.ps)
        xs = [torch.stack([p['xs'][j] * (64.0 if loud and i % 2 else 1.0) for i, p in enumerate(per)]).to(dt)
              for j in range(len(sig.srcs))]
        gate = torch.stack([p['gate'] for p in per]).to(dt) if sig.gate else None
        res = torch.stack([p['res'] for p in per]).to(torch.float32 if sig.res == 'f32' else dt) if sig.res else None
        odt = torch.float32 if sig.out == 'f32' else dt
        out = torch.full((n, Ho, Wo, sig.out_cs), float('nan'), dtype=odt, device='cuda')
        alone = torch.full_like(out, float('nan'))
        x1 = xs[1] if len(xs) > 1 else None
        old = cuda_ops.set_conv_cta_cap(cap)
        old_smem = cuda_ops.set_conv_smem_cap(smem_cap)
        try:
            cuda_ops.conv2d(layer, xs[0], x1, out, gate=gate, res=res, act_pre=sig.act_pre, act_post=sig.act_post,
                            pixel_shuffle=sig.ps)
            for i in range(n):
                cuda_ops.conv2d(layer, xs[0][i], None if x1 is None else x1[i], alone[i],
                                gate=None if gate is None else gate[i], res=None if res is None else res[i],
                                act_pre=sig.act_pre, act_post=sig.act_post, pixel_shuffle=sig.ps)
            torch.cuda.synchronize()
        finally:
            cuda_ops.set_conv_cta_cap(old)
            cuda_ops.set_conv_smem_cap(old_smem)
        for i in range(n):
            assert torch.equal(_bits(out[i]), _bits(alone[i])), f'{name} {H}x{W} {dtn} n={n} cap {cap}: image {i} differs'


_ENGINE_CASES = [(nm, s, g) for nm, s, geoms in ENGINE_CONVS for g in geoms]


@pytest.mark.gpu
@pytest.mark.parametrize('case', _ENGINE_CASES, ids=[f'{nm}-{g[0]}x{g[1]}' for nm, _, g in _ENGINE_CASES])
def test_batched_engine_conv_equals_separate_launches(cuda_ops, case):
    name, sig, (H, W) = case
    run_batch(cuda_ops, name, sig, H, W, 2)


RAGGED = [(c[0], c[1], c[2]) for c in BRANCH_CASES if c[0].startswith('ragged')]


@pytest.mark.gpu
@pytest.mark.parametrize('cap', [1, 7], ids=['cap1', 'cap7'])
@pytest.mark.parametrize('case', RAGGED, ids=[c[0] for c in RAGGED])
def test_batched_ragged_tiles_cross_images_in_one_cta(cuda_ops, case, cap):
    """271 x 483 maps (partial edge tiles) and 3 images on 1 or 7 CTAs: each CTA's tile loop walks across image borders"""
    name, sig, (H, W) = case
    run_batch(cuda_ops, name, sig, H, W, 3, cap=cap)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['conv48.res', 'feat_fusion.1', 'main.0', 'upsample1', 'conv_last', 'spynet.0',
                                  'align.p_conv.0.stride4'])
def test_batched_padding_does_not_read_the_neighbouring_image(cuda_ops, name):
    run_batch(cuda_ops, name, _sig(name), 37, 53, 3, cap=7, loud=True)


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
def test_descriptor_layout_matches_the_compiled_header(tmp_path):
    """offset of every rv_conv_desc field and the struct size, as a C compiler lays out include/refvsr_b200.h, against the
    ctypes mirror in lib.py"""
    from refvsr_b200.lib import rv_conv_desc
    cc = shutil.which('cc') or shutil.which('gcc') or shutil.which('g++')
    if cc is None:
        pytest.skip('no C compiler')
    names = [f[0] for f in rv_conv_desc._fields_]
    src = tmp_path / 'layout.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "refvsr_b200.h"\nint main(void) {\n' +
                   ''.join(f'  printf("%zu\\n", offsetof(rv_conv_desc, {nm}));\n' for nm in names) +
                   '  printf("%zu\\n", sizeof(rv_conv_desc));\n  return 0;\n}\n')
    exe = tmp_path / 'layout'
    subprocess.run([cc, '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [getattr(rv_conv_desc, nm).offset for nm in names] + [C.sizeof(rv_conv_desc)]


def _desc(sig, H, W, dt, base, n=0, strides=None):
    from refvsr_b200.lib import DTYPE_CODE, rv_conv_desc
    w = torch.zeros(sig.cout, sum(r for r, _ in sig.srcs), sig.k, sig.k)
    layer = packing.pack_conv_uncached('plan', w, torch.zeros(sig.cout), list(sig.srcs), 1, sig.pad, dt, 'cpu', True, ps_rows=sig.ps)
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
    if strides is not None:
        d.bs_src0 = d.bs_src1 = d.bs_gate = d.bs_res = d.bs_out = strides
    return d


def _plan(lib, d):
    plan, depth, store = (C.c_int32 * 8)(), C.c_int32(-1), C.c_int32(-1)
    rc = lib.rv_conv2d_tc_plan(C.byref(d), H100_SMEM, H100_SMS, plan)
    assert rc == 0, lib.rv_last_error()
    assert lib.rv_conv2d_tc_epi_depth(C.byref(d), H100_SMEM, H100_SMS, C.byref(depth)) == 0, lib.rv_last_error()
    assert lib.rv_conv2d_tc_out_store(C.byref(d), H100_SMEM, H100_SMS, C.byref(store)) == 0, lib.rv_last_error()
    return list(plan), depth.value, store.value


_TC = [(nm, s) for nm, s, _ in ENGINE_CONVS if s.stride == 1]


@pytest.mark.parametrize('dt', [torch.bfloat16, torch.float16], ids=['bf16', 'fp16'])
def test_batch_plan_keeps_ownership_and_zero_n_is_one_image(dt):
    """for every tensor-core conv of the engine: n = 0 plans as n = 1 whatever the stride fields hold; n = 4 with 16-byte
    aligned image strides takes the same plan (rings, resident weights, gate / residual buffers, output store), and every
    consumer owns its slots and accumulators; a src0 stride TMA cannot address, or a missing stride, is refused"""
    from refvsr_b200.lib import load_library
    lib = load_library()
    base = 1 << 20
    for name, sig in _TC:
        H, W = 270, 480
        one = _plan(lib, _desc(sig, H, W, dt, base, n=1))
        assert _plan(lib, _desc(sig, H, W, dt, base, n=0)) == one, name
        assert _plan(lib, _desc(sig, H, W, dt, base, n=0, strides=12345)) == one, name
        four = _plan(lib, _desc(sig, H, W, dt, base, n=4, strides=H * W * 256))
        assert four == one, (name, four, one)
        mode, slots, resident, S, ncons, nacc, nb, smem = four[0]
        assert ncons == nacc == 2 and slots >= 1 and smem <= H100_SMEM and (resident or mode != 1), (name, four)
        d = _desc(sig, H, W, dt, base, n=4, strides=H * W * 256 + 4)
        assert lib.rv_conv2d_tc_plan(C.byref(d), H100_SMEM, H100_SMS, (C.c_int32 * 8)()) != 0, name
        d = _desc(sig, H, W, dt, base, n=4, strides=0)
        assert lib.rv_conv2d_tc_plan(C.byref(d), H100_SMEM, H100_SMS, (C.c_int32 * 8)()) == -1, name


def _psv_register_store_cap(dt):
    """the largest shared-memory budget at which the upsampling conv still runs the pixel-shuffle kernel but stores its HR rows
    as 16-byte register stores (rv_conv2d_tc_out_store kind 3) instead of TMA boxes, for a batch of 3"""
    from refvsr_b200.lib import load_library
    lib = load_library()
    sig = _sig('upsample1')
    for smem in range(H100_SMEM, 100 * 1024, -1024):
        d = _desc(sig, 37, 53, dt, 1 << 20, n=3, strides=37 * 53 * 48 * 4)
        kind = C.c_int32(-1)
        if lib.rv_conv2d_tc_out_store(C.byref(d), smem, H100_SMS, C.byref(kind)) == 0 and kind.value == 3:
            return smem
    return None


def test_psv_register_store_budget_exists():
    for dt in (torch.bfloat16, torch.float16):
        assert _psv_register_store_cap(dt) is not None


@pytest.mark.gpu
def test_batched_psv_register_stores(cuda_ops):
    """the batched pixel-shuffle kernel's 16-byte register-store path (out_tma off under a smaller shared-memory budget), with
    loud neighbouring images"""
    cap = min(_psv_register_store_cap(dt) for dt in (torch.bfloat16, torch.float16))
    run_batch(cuda_ops, 'upsample1', _sig('upsample1'), 37, 53, 3, cap=7, loud=True, smem_cap=cap)
