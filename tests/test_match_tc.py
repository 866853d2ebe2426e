"""The wgmma matching GEMM (match.cu, rv_match_argmax impl=1): 256-row CTAs, K streamed as 64-column chunks plus a tail of
16-column slices, consumers taking turns on the tensor cores.  conf / idx must not depend on the zero padding of K (the
dropped k-steps only added zeros), ragged P and R around the tiles must be handled, and equal scores resolve to the lowest
reference index.  The GPU tests are marked; the machine-code and engine-buffer checks run without a GPU."""
import os
import re
import shutil
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'refvsr_b200', 'librefvsr_b200.so')


def _rand(shape, seed):
    return torch.rand(shape, generator=torch.Generator().manual_seed(seed)) * 2 - 1


def _packed(ops, feat, kpad, mode):
    out = torch.empty((feat.shape[0] * feat.shape[1], kpad), dtype=torch.float16, device='cuda')
    ops.patch_pack(feat.cuda(), out, mode)
    return out


def _match(ops, A, B):
    conf = torch.empty(A.shape[0], device='cuda')
    idx = torch.empty(A.shape[0], dtype=torch.int32, device='cuda')
    ops.match_argmax(A, B, conf, idx, impl=1)
    torch.cuda.synchronize()
    return conf.cpu(), idx.cpu()


def _check_against_fp32(A, B, conf, idx, chunk=4096):
    """conf against the fp32 GEMM's column max, idx where it differs only on near-ties (tolerances of test_match_argmax)"""
    a, b = A.float(), B.float()
    mism, worst, worst_gap = 0, 0.0, 0.0
    for s in range(0, a.shape[0], chunk):
        S = (a[s:s + chunk] @ b.t()) / 4096.0
        v, i = S.max(dim=1)
        c, k = conf[s:s + chunk].to(S.device), idx[s:s + chunk].to(S.device).long()
        assert int(k.min()) >= 0 and int(k.max()) < b.shape[0]
        worst = max(worst, float((c - v).abs().max()))
        worst_gap = max(worst_gap, float((v - S.gather(1, k[:, None])[:, 0]).max()))
        mism += int((k != i).sum())
    assert worst <= 1e-4, f'conf max err {worst:.3e}'
    assert worst_gap <= 1e-4 + 1e-5, f'score at the returned index is {worst_gap:.3e} below the maximum'
    assert mism / a.shape[0] <= 2e-3, f'index mismatch rate {mism / a.shape[0]:.4f}'


@pytest.mark.gpu
@pytest.mark.parametrize('split', [False, True])
def test_zero_k_padding_does_not_change_results(cuda_ops, split):
    """the same patches packed with and without zero columns give bitwise-equal conf / idx"""
    lr_f, ref_f = _rand((61, 83, 16), 1), _rand((37, 45, 16), 2)
    mode_a, mode_b = (1, 2) if split else (0, 0)
    res = []
    for kpad in ((432, 448) if split else (144, 192, 256, 320)):
        res.append(_match(cuda_ops, _packed(cuda_ops, lr_f, kpad, mode_a), _packed(cuda_ops, ref_f, kpad, mode_b)))
    for conf, idx in res[1:]:
        assert torch.equal(conf, res[0][0]) and torch.equal(idx, res[0][1])


@pytest.mark.gpu
@pytest.mark.parametrize('P', [1, 255, 256, 257, 1000])
@pytest.mark.parametrize('R', [1, 127, 128, 129, 700])
def test_ragged_sizes(cuda_ops, P, R):
    A = (_rand((P, 144), 10 + P) * 8).half().cuda()
    B = (_rand((R, 144), 20 + R) * 8).half().cuda()
    conf, idx = _match(cuda_ops, A, B)
    _check_against_fp32(A.cpu(), B.cpu(), conf, idx)


@pytest.mark.gpu
@pytest.mark.parametrize('kpad', [144, 192, 432])
def test_duplicate_reference_rows_return_the_lowest_index(cuda_ops, kpad):
    """copies of a reference row in the same thread's columns, in other threads', in later tiles and in the ragged last tile:
    every LR row equal to that row must get the first copy, in both consumers' rows and both m64 blocks of each"""
    R, P = 700, 1000
    B = (_rand((R, kpad), 3) * 8).half()
    groups = [[3, 4, 11, 131, R - 1], [200, 201, 328, 456], [129, 130, 138, 699 - 128]]
    for g in groups:
        for r in g[1:]:
            B[r] = B[g[0]]
    A = torch.stack([B[groups[i % len(groups)][0]] for i in range(P)])
    conf, idx = _match(cuda_ops, A.cuda(), B.cuda())
    exp = torch.tensor([min(groups[i % len(groups)]) for i in range(P)], dtype=torch.int32)
    assert torch.equal(idx, exp), (idx != exp).nonzero()[:8].flatten().tolist()
    # the duplicates differ from every other row, so their score is the strict maximum of each LR row
    S = (A.float() @ B.float().t()) / 4096.0
    assert torch.equal(S.argmax(dim=1).int(), exp)


@pytest.mark.gpu
def test_full_size_against_fp32_gemm(cuda_ops):
    """the bench shape: 270 x 480 LR patches against 135 x 240 reference patches, K = 144"""
    lr_f, ref_f = _rand((270, 480, 16), 5).cuda(), _rand((135, 240, 16), 6).cuda()
    A, B = _packed(cuda_ops, lr_f, 144, 0), _packed(cuda_ops, ref_f, 144, 0)
    assert (A.shape[0], B.shape[0]) == (129600, 32400)
    conf, idx = _match(cuda_ops, A, B)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        _check_against_fp32(A, B, conf, idx)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.mark.gpu
def test_bad_kpad_and_misaligned_operands_raise(cuda_ops):
    conf = torch.empty(64, device='cuda')
    idx = torch.empty(64, dtype=torch.int32, device='cuda')
    for kpad in (152, 464):
        A = torch.zeros((64, kpad), dtype=torch.float16, device='cuda')
        with pytest.raises(ValueError, match='kpad'):
            cuda_ops.match_argmax(A, A, conf, idx, impl=1)
    flat = torch.zeros(64 * 144 + 4, dtype=torch.float16, device='cuda')
    A = flat[4:].view(64, 144)                   # 8-byte aligned rows
    with pytest.raises(ValueError, match='aligned'):
        cuda_ops.match_argmax(A, A, conf, idx, impl=1)
    torch.cuda.synchronize()


def _cuobjdump():
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    cands = [os.path.join(os.path.dirname(nvcc), 'cuobjdump'), shutil.which('cuobjdump')]
    return next((c for c in cands if c and os.path.isfile(c)), None)


def test_match_kernel_uses_no_local_memory():
    tool = _cuobjdump()
    if not os.path.isfile(LIB):
        pytest.skip('library not built')
    if tool is None:
        pytest.skip('cuobjdump not found')
    sass = subprocess.run([tool, '-sass', LIB], capture_output=True, text=True, check=True).stdout
    res = subprocess.run([tool, '-res-usage', LIB], capture_output=True, text=True, check=True).stdout
    stack = {m.group(1): int(m.group(2)) for m in re.finditer(r'Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)', res)}
    names = [n for n in stack if 'match_tc_kernel' in n]
    assert {re.search(r'match_tc_kernelILi(\d)E', n).group(1) for n in names} == {'1', '2'}, names
    for n in names:
        assert stack[n] == 0, (n, stack[n])
    cur, local = None, []
    for line in sass.splitlines():
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            cur = m.group(1)
        elif cur and 'match_tc_kernel' in cur and re.search(r'\b(LDL|STL)\b', line):
            local.append((cur, line.strip()))
    assert not local, local[:4]


@pytest.mark.parametrize('mode,width', [('single', 144), ('split', 432)])
def test_engine_match_operands_have_no_zero_columns(oracle_ops, mode, width):
    """single mode packs the 144 patch values per row, split mode 3 x 144"""
    from refvsr_b200.synth import sliding_windows
    from util import build_case
    with torch.random.fork_rng():            # module construction draws from the global generator: leave it as it was
        spec, cfg, net, lrs, refs, golden = build_case('small_t7_24x32', 'cpu', ops=oracle_ops, b200_precision='fp32',
                                                       b200_match=mode)
        assert net.Network.match_mode == mode
        k, wl, wr, first = next(iter(sliding_windows(lrs, refs, spec['T'])))
        net(wl, wr, first, False, False)
    widths = {key[0]: key[1][1] for key in net.Network._bufs if key[0] in ('fm.A', 'fm.B')}
    assert widths == {'fm.A': width, 'fm.B': width}, widths
