"""Machine code of the tensor-core convolution's compile-time 3x3 tap loop (conv_tc.cu, MODE 1 with KS = 3, KST = 3).

Each pipeline stage of those kernels must reach the tensor cores as one unbroken run of 9 taps x 2 halves x 3 K-steps = 54
HGMMAs: a single WARPGROUP.ARRIVE in front of it and the scoreboard (gsb0) only on its last HGMMA.  A runtime loop makes ptxas
fence and wait on every HGMMA instead.  The unrolled loop must not spill either: its stack frame and local-memory traffic are
those of the runtime-loop kernel of the same types and NB (the producer's per-consumer slot / phase arrays).  The NB = 96
pixel-shuffle twin (PSV) writes its 16-bit output rows only as 16-byte vectors.
Reads the built library with cuobjdump; needs no GPU."""
import os
import re
import shutil
import subprocess
from collections import defaultdict

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'refvsr_b200', 'librefvsr_b200.so')
MMAS_PER_STAGE = 9 * 2 * 3
FIXED = re.compile(r'conv_tc_kernelI(\w+?)Li1ELi(\d+)ELi3ELi3ELb([01])EE')


def _cuobjdump():
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    cands = [os.path.join(os.path.dirname(nvcc), 'cuobjdump'), shutil.which('cuobjdump')]
    return next((c for c in cands if c and os.path.isfile(c)), None)


@pytest.fixture(scope='module')
def dump():
    tool = _cuobjdump()
    if not os.path.isfile(LIB):
        pytest.skip('library not built')
    if tool is None:
        pytest.skip('cuobjdump not found')
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
    return funcs, stack


def _fixed(funcs):
    return {name: m for name in funcs if (m := FIXED.search(name))}


def test_fixed_tap_loop_is_instantiated_for_bf16_and_f16(dump):
    funcs, _ = dump
    fixed = _fixed(funcs)
    types = {m.group(1) for m in fixed.values()}
    assert any('bfloat16' in t for t in types) and any(t.startswith('6__half') for t in types), sorted(fixed)
    assert {int(m.group(2)) for m in fixed.values()} >= {16, 48, 96}, sorted(fixed)


def test_each_stage_is_one_arrive_and_one_scoreboard(dump):
    funcs, _ = dump
    fixed = _fixed(funcs)
    assert fixed
    for name in fixed:
        stages, cur = [], None
        for line in funcs[name]:
            if 'WARPGROUP.ARRIVE' in line:
                cur = []
                stages.append(cur)
            elif 'HGMMA' in line:
                assert cur is not None, f'{name}: HGMMA before any WARPGROUP.ARRIVE'
                cur.append('gsb0' in line)
        assert stages, name
        for st in stages:
            assert len(st) == MMAS_PER_STAGE, (name, len(st))
            assert st[-1] and not any(st[:-1]), f'{name}: gsb0 on HGMMAs {[i for i, g in enumerate(st) if g]}'


def test_fixed_tap_loop_does_not_spill(dump):
    funcs, stack = dump
    local = re.compile(r'\b(LDL|STL)\b')
    fixed = _fixed(funcs)
    assert fixed
    for name in fixed:
        sibling = re.sub(r'ELi3ELi3ELb[01]EE', 'ELi0ELi0ELb0EE', name)
        assert sibling in funcs and name in stack and sibling in stack, name
        assert stack[name] == stack[sibling], (name, stack[name], stack[sibling])
        n_fixed = sum(1 for line in funcs[name] if local.search(line))
        n_loop = sum(1 for line in funcs[sibling] if local.search(line))
        assert n_fixed == n_loop, (name, n_fixed, n_loop)


def test_pixel_shuffle_twin_stores_16_byte_rows(dump):
    funcs, _ = dump
    psv = [name for name, m in _fixed(funcs).items() if m.group(3) == '1']
    assert any('bfloat16' in n for n in psv) and any('6__half' in n for n in psv), psv
    for name in psv:
        stores = [line for line in funcs[name] if re.search(r'\bSTG\.', line)]
        assert stores and all('STG.E.128' in line for line in stores), (name, [s.split(';')[0].strip() for s in stores[:4]])
