"""rv_frames_differ, the reuse guard (pointwise.cu): it decides whether the per-frame products cached for the previous window may
be reused, so a difference it misses puts stale features into the output without any sign.  The contract is exact and bitwise
(network.py, _enqueue_overlap_compare): the flag is non-zero iff some 4-byte word of some pair differs.

Every pair index of 1 to 16 pairs in turn holds the only differing word, at the first word, the last word and a word only a
later iteration of the 64 x 256-thread grid-stride loop reaches - each of the four words of one 16-byte load there, since the
16-byte path compares x, y, z and w separately - on both load paths: 16-byte (uint4) loads when every buffer is 16-byte aligned
and a multiple of 16 bytes long, 4-byte loads otherwise (one pair 4 bytes off, or one size of 4, 8 or 12 mod 16).  Then the bitwise contract on fp32 words (equal NaN payloads are equal, +0 and -0 differ, different NaN payloads
differ), the engine's frame sizes with 12 pairs, and the refused calls."""
import ctypes as C

import pytest
import torch

THREADS = 64 * 256                       # the kernel's grid: 64 blocks of 256 threads per pair
WORDS = 3 * 4 * THREADS + 12             # 3 iterations of 16-byte loads (12 of 4-byte loads), plus a partial one
LATE = 4 * THREADS + 4 * 777             # the words of 16-byte load 16384 + 777 (iteration 1): its x, y, z and w
LATE_WORDS = tuple(LATE + k for k in range(4))
PATHS = {                                 # extra words of one pair, its offset in words
    'uint4': (0, 0),
    'u32-offset-4': (0, 1),
    'u32-size-4-mod-16': (1, 0),
    'u32-size-8-mod-16': (2, 0),
    'u32-size-12-mod-16': (3, 0),
}


def _buf(words, off, g):
    """random int32 words starting `off` words past the start of a fresh (256-byte aligned) allocation"""
    base = torch.randint(-2 ** 31, 2 ** 31 - 1, (words + off,), generator=g, dtype=torch.int32).cuda()
    return base[off:]


def _equal_pairs(n, path, seed):
    """n equal (a, b) pairs in separate allocations, sizes WORDS + 4 i words (multiples of 16 bytes); pair n // 2 takes the
    path's extra words and offset"""
    extra, off = PATHS[path]
    g = torch.Generator().manual_seed(seed)
    pairs = []
    for i in range(n):
        w, o = WORDS + 4 * i + (extra if i == n // 2 else 0), (off if i == n // 2 else 0)
        a = _buf(w, o, g)
        b = torch.empty(w + o, dtype=torch.int32, device='cuda')[o:]
        b.copy_(a)
        pairs.append((a, b))
    return pairs


def _takes_uint4(pairs):
    """rv_frames_differ's choice of load path: 16-byte loads iff every buffer is 16-byte aligned and a multiple of 16 bytes"""
    return all(t.data_ptr() % 16 == 0 and t.numel() * t.element_size() % 16 == 0 for p in pairs for t in p)


def _differ(ops, pairs):
    """the flag after one call; it starts at a sentinel so that a call that does not zero it shows"""
    flag = torch.full((1,), 7, dtype=torch.int32, device='cuda')
    ops.frames_differ(pairs, flag)
    return int(flag.item())


@pytest.mark.gpu
@pytest.mark.parametrize('path', list(PATHS))
def test_one_differing_word_is_found(cuda_ops, path):
    """for n = 1 .. 16 pairs, each pair in turn differs in one word only - the first, the last, or one a later grid-stride
    iteration reaches - and the flag is set; equal pairs, before and after, give 0"""
    assert LATE // 4 >= THREADS and LATE + 3 < WORDS - 1 and {p % 4 for p in LATE_WORDS} == {0, 1, 2, 3}
    for n in range(1, 17):
        pairs = _equal_pairs(n, path, n)
        assert _takes_uint4(pairs) == (path == 'uint4')
        assert _differ(cuda_ops, pairs) == 0, f'{path}: {n} equal pairs flagged'
        for i in range(n):
            b = pairs[i][1]
            for pos in (0, b.numel() - 1) + LATE_WORDS:
                bit = 1 << ((7 * i + pos) % 31)
                b[pos] ^= bit
                assert _differ(cuda_ops, pairs) == 1, f'{path}: n {n}, pair {i}, word {pos} of {b.numel()}: difference missed'
                b[pos] ^= bit
                assert _differ(cuda_ops, pairs) == 0, f'{path}: n {n}, pair {i}, word {pos}: equal pairs flagged after a difference'


@pytest.mark.gpu
@pytest.mark.parametrize('path', ['uint4', 'u32-offset-4', 'u32-size-8-mod-16'])
def test_comparison_is_bitwise(cuda_ops, path):
    """fp32 words compare as bits: identical NaN payloads are equal, +0 and -0 differ, two different NaN payloads differ"""
    pairs = _equal_pairs(3, path, 99)
    a, b = pairs[1]
    for pos in (0, a.numel() - 1) + LATE_WORDS:
        a[pos] = b[pos] = 0x7FC00001                     # a quiet NaN with a payload, in both
        assert _differ(cuda_ops, [(x.view(torch.float32), y.view(torch.float32)) for x, y in pairs]) == 0
        a[pos], b[pos] = 0, -2 ** 31                     # +0.0 and -0.0
        assert _differ(cuda_ops, pairs) == 1, f'{path}: +0 and -0 at word {pos} compared equal'
        a[pos], b[pos] = 0x7FC00001, 0x7FC00002          # two NaN payloads
        assert _differ(cuda_ops, pairs) == 1, f'{path}: different NaN payloads at word {pos} compared equal'
        a[pos] = b[pos] = 0


@pytest.mark.gpu
@pytest.mark.parametrize('sizes', [((3, 270, 480),) * 12, ((3, 270, 480), (3, 540, 960)) * 6],
                         ids=['x4-ref1x-12-pairs', 'x4-ref2x-12-pairs'])
def test_engine_frame_sizes(cuda_ops, sizes):
    """the guard's own calls: 12 pairs of fp32 frames (6 LR and 6 reference frames of a 7-frame window); each pair in turn
    differs at its first word, its last word and each word of a 16-byte load in a later grid-stride iteration"""
    g = torch.Generator().manual_seed(3)
    pairs = [(lambda a: (a, a.clone()))(torch.rand(s, generator=g).cuda()) for s in sizes]
    assert _differ(cuda_ops, pairs) == 0
    for i, (_, b) in enumerate(pairs):
        w = b.view(-1).view(torch.int32)
        for pos in (0, w.numel() - 1) + tuple(2 * 4 * THREADS + 4 * 5 + k for k in range(4)):
            w[pos] ^= 1
            assert _differ(cuda_ops, pairs) == 1, f'pair {i} {tuple(b.shape)}: word {pos} missed'
            w[pos] ^= 1
    assert _differ(cuda_ops, pairs) == 0


@pytest.mark.gpu
def test_bad_calls_are_refused(cuda_ops):
    """no pair, more than 16 pairs and a size that is not a multiple of 4 bytes are refused by the library"""
    from refvsr_b200.lib import _check
    lib = cuda_ops.lib
    flag = torch.zeros(1, dtype=torch.int32, device='cuda')
    bufs = [torch.zeros(64, dtype=torch.int32, device='cuda') for _ in range(17)]
    for n in (0, 17):
        pa = (C.c_void_p * 17)(*[t.data_ptr() for t in bufs])
        nb = (C.c_uint64 * 17)(*([256] * 17))
        with pytest.raises(ValueError, match='1..16 buffer pairs'):
            _check(lib, lib.rv_frames_differ(pa, pa, nb, n, C.c_void_p(flag.data_ptr()), None), 'rv_frames_differ')
    a = torch.zeros(4 * 1000 + 2, dtype=torch.uint8, device='cuda')
    with pytest.raises(ValueError, match='multiple of 4'):
        cuda_ops.frames_differ([(a, a.clone())], flag)
    torch.cuda.synchronize()
