"""The matching GEMM (match.cu, rv_match_argmax) checked row by row against a float64 reference, at every shape the engine
launches it and at shapes that force each branch of its launch plan.

The bound.  The operands are fp16 rows a_m (LR patches) and b_r (reference patches) of K = kpad columns.  fp16 x fp16 products
are exact, so S[m, r] = sum_k a_mk b_rk in float64 is exact up to about K 2^-53 relative.  Both kernels multiply exactly and
accumulate in fp32 - the tensor-core kernel in an order and with a rounding it does not specify, the CUDA-core kernel in k
order with fused multiply-adds - so, as in test_conv_fp64's derivation (K - 1 fp32 additions, each within 2u of the magnitude
it works on) and with Cauchy-Schwarz applied to sum_k |a_mk| |b_rk|, the kernel's fp32 score satisfies

    |S^[m, r] - S[m, r]| <= E_m = C_ACC K u |a_m| max_r |b_r|,        u = 2^-24,

and conf = S^ / 4096 (out_scale = 1 / 4096 is exact).  With S*_m = max_r S[m, r], every row m must satisfy
  1. 0 <= idx[m] < R;
  2. |4096 conf[m] - S*_m| <= E_m;
  3. S[m, idx[m]] >= S*_m - 2 E_m: the returned row lies in the window of rows the bound cannot tell apart, so wherever that
     window holds a single row the index is exact - there is no mismatch allowance;
  4. |4096 conf[m] - S[m, idx[m]]| <= E_m: conf is the score of the returned row, not of another lane's or row's;
  5. where every row of the window is a bitwise copy of one B row, idx[m] is the lowest copy (equal operands give equal fp32
     scores, and equal scores resolve to the lowest index); an all-zero A row scores exactly 0 everywhere and gets index 0;
  6. the guard elements around conf and idx keep their sentinels.

The reference is a float64 GEMM of the operands, in chunks of 1024 rows (129 600 x 129 600 scores do not fit as one matrix):
up to 1.1 GB of float64 scores and 0.5 GB of int32 temporaries for the copy rule at a time.  It is exact for every row, not
only for the candidates an fp32 pre-filter would keep.  NVIDIA's H100 SXM data sheet gives the fp64 tensor cores the rate of
non-TF32 fp32 (67 TFLOP/s each), so a filter would not make it cheaper; the GPU half of this file, every full-size case
included, runs in well under a minute.

Operand families (given straight to rv_match_argmax):
  * engine: rv_patch_pack of smooth 16-channel maps (box-filtered noise) in the engine's pairing - mode 0 / 0 at kpad 144 for
    16-bit features, modes 1 / 2 at kpad 432 for fp32 features - with zero blocks and constant blocks, which give zero A rows,
    exact ties between bitwise-equal B rows and near-ties;
  * planted: B random unit rows x 64, A[m] = B[w(m)] with w(m) = (s m + c) mod R, gcd(s, R) = 1, so every reference row is the
    winner of some LR row and idx must equal w(m).  S* = sum |a| |b| here, so the bound is relatively tight (about 3 K u:
    2.6e-5 at K = 144) and a second rounding of the accumulator to bf16 or fp16 fails it;
  * duplicates: copies of a few B rows at every column residue mod 128 (every lane & 3, j and e of the wgmma accumulator) in
    the first tile, a middle tile and the ragged last tile; every A row is one of the copied rows, spread over both consumers,
    both m64 blocks, every warp quarter and the ragged last CTA;
  * negative: B entries positive and every third A row negative, so each real score of those rows is below the 0 that an
    out-of-range (zero-filled) B row would score;
  * generic: fp16 values of comparable magnitude in every column (+-[0.5, 2)), so dropping or repeating any k-slice or chunk
    moves S far outside the bound.

Composition (one test per match mode at the x4 geometry): patch_pack + GEMM against the float64 cosine similarity (x 4096) of
the fp64-normalised, reflect-padded 3 x 3 patches.  The window widens by the packing error of test_pointwise_fp64's
patch_pack bound (|hi - v| <= ulp_fp16(v); split: |hi + lo - v| <= ulp_fp16(v - hi) + (K + C_AR) u |v|) and, in split mode, by
the dropped lo x lo term: the "split mode is fp32-grade" claim of match.cu as a checked inequality.

Without a GPU: the list of the engine's match_argmax calls, the launch-plan coverage of the branch cases, and the bound's
self-tests on a CPU model of the kernel's tile scan (correct variants pass, planted defects fail with a report naming the
tile, lane and row).  With a GPU: every listed call with the engine, planted, duplicate and negative families, the branch cases
and the composition."""
import collections
import math

import pytest
import torch
import torch.nn.functional as F

from test_conv_fp64 import C_ACC, ulp
from test_pointwise_fp64 import C_AR, _run_engine, _seed, ref_patches

U = 2.0 ** -24
GUARD = 4096
IDX_SENTINEL = -7
H100_SMEM_OPTIN = 232448            # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100: 227 KB

# ------------------------------------------------------------------------------------------------------------------
# the list: every match_argmax call of the engine
# ------------------------------------------------------------------------------------------------------------------
# (impl, kpad, LR matching grid (h, w), reference matching grid (hr, wr)): P = h w LR rows, R = hr wr reference rows.
# kpad 144: the 16-bit engines (single mode), 432: the fp32 engine (split mode); impl 1: wgmma kernel, impl 0: the CUDA-core
# kernel of b200_tensor_cores=False.  test_engine_match_calls_are_all_listed keeps this complete.
Match = collections.namedtuple('Match', 'impl kpad lr ref')
X4_GRID, REF1_GRID, HD_GRID, HD_REF_GRID = (270, 480), (135, 240), (68, 120), (34, 60)
ENGINE_MATCH = [Match(impl, kpad, lr, ref) for impl in (1, 0) for kpad in (144, 432) for lr, ref in (
    (X4_GRID, REF1_GRID),           # x4 (LR 270x480, Ref 1x) and x2 (LR 540x960: the VGG max-pool halves it)
    (X4_GRID, X4_GRID),             # x4 with Ref 2x: the bench's small_mfid workload, 1013 N tiles
    (HD_GRID, HD_REF_GRID))]        # flag_HD_in at LR 272x480


def _pr(e):
    return e.lr[0] * e.lr[1], e.ref[0] * e.ref[1]


# ------------------------------------------------------------------------------------------------------------------
# CPU: the list above is what the engine launches
# ------------------------------------------------------------------------------------------------------------------
def _recording_ops():
    """the CPU operator set with every operator a no-op, recording (impl, kpad, P, R) of every match_argmax call"""
    from u8_ops import U8OracleOps

    class Recording(U8OracleOps):
        def __init__(self):
            self.seen = collections.Counter()

        def __getattribute__(self, name):
            attr = object.__getattribute__(self, name)
            if name.startswith('_') or name == 'seen' or not callable(attr):
                return attr
            if name == 'match_argmax':
                def rec(A, B, conf, idx, impl=1):
                    self.seen[(impl, A.shape[1], A.shape[0], B.shape[0])] += 1
                return rec
            return attr if name == 'pack_conv' else (lambda *a, **k: 0)
    return Recording()


def test_engine_match_calls_are_all_listed():
    """the full-size x4 (Ref 1x and 2x), x2 and flag_HD_in schedules at bf16 and fp32, with tensor cores on and off, shapes
    only: every match_argmax call they make is listed, and every listed entry is launched"""
    seen = set()
    for prec in ('bf16', 'fp32'):
        for tc in (True, False):
            runs = [_run_engine(_recording_ops(), 270, 480, prec, b200_tensor_cores=tc),
                    _run_engine(_recording_ops(), 270, 480, prec, ref_scale=2, b200_tensor_cores=tc),
                    _run_engine(_recording_ops(), 540, 960, prec, b200_tensor_cores=tc, scale=2, matching_ksize=4),
                    _run_engine(_recording_ops(), 272, 480, prec, cfg_name='config_RefVSR_MFID_8K', b200_tensor_cores=tc)]
            for ops in runs:
                assert ops.seen, 'no match_argmax call recorded'
                seen |= set(ops.seen)
    listed = {(e.impl, e.kpad) + _pr(e) for e in ENGINE_MATCH}
    assert not seen - listed, f'match_argmax calls the engine makes and ENGINE_MATCH does not list: {sorted(seen - listed)}'
    assert not listed - seen, f'listed calls the engine does not make: {sorted(listed - seen)}'


# ------------------------------------------------------------------------------------------------------------------
# the launch plan (match.cu, match_tc's host arithmetic)
# ------------------------------------------------------------------------------------------------------------------
Plan = collections.namedtuple('Plan', 'impl nfull ntail nch mb slots')
MT_BN, MT_SLOT, MT_SLOTS_MAX = 128, 128 * 128, 8


def match_plan(kpad, smem_optin, impl=1):
    """the plan match_tc derives for kpad on a device with `smem_optin` bytes of opt-in shared memory per block: 64-column
    chunks, 16-column tail slices, MB = 2 when a 256-row A block leaves room for two tiles' chunks in the ring, and the ring's
    slot count.  impl 0 (the CUDA-core kernel) has no plan: 64-row CTAs over 64-column tiles."""
    if impl == 0:
        return Plan(0, 0, 0, 0, 0, 0)
    nfull, ntail = kpad // 64, (kpad % 64) // 16
    nch = nfull + (ntail > 0)
    budget = smem_optin - 1024 - 2048
    a2, a1 = 256 * kpad * 2, 128 * kpad * 2
    mb = 2 if budget >= a2 + 2 * nch * MT_SLOT else 1
    slots = min(MT_SLOTS_MAX, (budget - (a2 if mb == 2 else a1)) // MT_SLOT)
    assert slots >= nch, f'kpad {kpad}: the kernel refuses it (not enough shared memory)'
    return Plan(1, nfull, ntail, nch, mb, slots)


# the branch cases: kpad (nfull 0 and > 0, ntail 0 to 3, MB 2 and 1, a ring of exactly nch slots) crossed with ragged P and
# R around the CTA (128 MB rows) and N-tile (128 rows) sizes
BRANCH_KPAD = [16, 48, 64, 80, 96, 144, 192, 208, 416, 432, 448]
BRANCH_P = [1, 63, 64, 65, 255, 256, 257, 1000]
BRANCH_R = [1, 7, 8, 127, 128, 129, 700]
BRANCH_SIMT_KPAD = [16, 144, 432]


def test_branch_cases_reach_every_plan():
    """at an H100's 227 KB the branch cases reach MB 1 and 2, nfull 0 and > 0, every ntail 0..3 and a ring of exactly nch
    slots; MB = 2 exactly for kpad <= 192 (derived from match_tc's arithmetic, not measured).  The engine's kpad 144 runs with
    MB = 2, its kpad 432 with MB = 1 and 7 = nch slots."""
    plans = {k: match_plan(k, H100_SMEM_OPTIN) for k in BRANCH_KPAD}
    assert {p.mb for p in plans.values()} == {1, 2}
    assert any(p.nfull == 0 for p in plans.values()) and any(p.nfull > 0 for p in plans.values())
    assert {p.ntail for p in plans.values()} == {0, 1, 2, 3}
    assert any(p.slots == p.nch for p in plans.values())
    for k, p in plans.items():
        assert p.mb == (2 if k <= 192 else 1), (k, p)
    assert plans[144].mb == 2 and plans[432] == Plan(1, 6, 3, 7, 1, 7)
    assert any(P % 256 and P > 256 for P in BRANCH_P) and any(R % 128 and R > 128 for R in BRANCH_R)


# ------------------------------------------------------------------------------------------------------------------
# operands
# ------------------------------------------------------------------------------------------------------------------
def _gen(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


def _unit_rows(g, n, K, dev):
    """n random rows of K columns, L2-normalised x 64 (the scale of packed patches), in fp16"""
    x = torch.randn(n, K, generator=g, device=dev, dtype=torch.float64)
    return (x / x.norm(dim=1, keepdim=True) * 64).half()


def make_feat(g, H, W, dt, dev):
    """(H, W, 16) box-filtered noise with zero blocks and constant blocks: zero patches (all-zero rows), bitwise-equal patches
    (exact ties) and near-ties.  The constant blocks take one of two vectors c0 and 2 c0, the same in every map of a seed
    family, so LR rows of one map have exact copies among the reference rows of another."""
    x = torch.randn(1, 16, H + 4, W + 4, generator=g, device=dev)
    x = F.avg_pool2d(x, 5, stride=1)[0].permute(1, 2, 0).contiguous()
    c0 = torch.linspace(-1.0, 1.0, 16, device=dev) + 0.25
    bs = max(4, min(16, min(H, W) // 4))
    by = (torch.arange(H, device=dev) // bs).view(H, 1)
    bx = (torch.arange(W, device=dev) // bs).view(1, W)
    kind = (by * 7 + bx * 3) % 11
    x = torch.where((kind == 0)[..., None], torch.zeros_like(x), x)
    x = torch.where((kind == 1)[..., None], c0.expand_as(x), x)
    x = torch.where((kind == 2)[..., None], (2 * c0).expand_as(x), x)
    return x.to(dt)


def _coprime_step(R):
    s = max(1, int(R * 0.618))
    while math.gcd(s, R) != 1:
        s += 1
    return s


def planted(g, P, R, K, dev):
    """B random unit rows; A[m] = B[w(m)], w(m) = (s m + c) mod R with gcd(s, R) = 1.  Returns A, B, w."""
    B = _unit_rows(g, R, K, dev)
    s, c = _coprime_step(R), int(torch.randint(0, R, (1,), generator=g, device=dev))
    w = (torch.arange(P, device=dev, dtype=torch.int64) * s + c) % R
    return B[w].contiguous(), B, w


def duplicates(g, P, R, K, dev):
    """B random unit rows with copies of 20 value rows: groups 0-15 spread over every column residue of the first tile and of a
    middle tile and over the ragged last tile, groups 16-19 only in the last tile.  A[m] is the value row of group (7 m + m // 64)
    mod the groups placed.  Returns A, B and the expected index (each group's lowest copy)."""
    nt = (R + MT_BN - 1) // MT_BN
    last, nlast = nt - 1, R - (nt - 1) * MT_BN
    pos = collections.defaultdict(list)
    for t in sorted({0, nt // 2} - {last}):
        perm = torch.randperm(MT_BN, generator=g, device=dev).tolist()
        for i, q in enumerate(perm):
            pos[i % 16].append(t * MT_BN + q)
    perm = torch.randperm(nlast, generator=g, device=dev).tolist()
    only_last = min(8, nlast // 2)
    for i, q in enumerate(perm):
        pos[16 + i // 2 if i < only_last else i % 16].append(last * MT_BN + q)
    V = _unit_rows(g, 20, K, dev)
    B = _unit_rows(g, R, K, dev)
    groups = sorted(pos)
    for gi in groups:
        B[torch.tensor(pos[gi], device=dev)] = V[gi]
    m = torch.arange(P, device=dev)
    sel = torch.tensor(groups, device=dev)[(7 * m + m // 64) % len(groups)]
    low = torch.tensor([min(pos[gi]) if gi in pos else -1 for gi in range(20)], device=dev)
    return V[sel].contiguous(), B, low[sel]


def negative(g, P, R, K, dev):
    """B entries positive; every third A row negative, the others of mixed sign"""
    A = _unit_rows(g, P, K, dev)
    A[::3] = -A[::3].abs()
    return A, _unit_rows(g, R, K, dev).abs(), None


def generic(g, P, R, K, dev):
    """fp16 values +-[0.5, 2) in every column"""
    def m(n):
        v = 0.5 + 1.5 * torch.rand(n, K, generator=g, device=dev)
        return torch.where(torch.rand(n, K, generator=g, device=dev) < 0.5, -v, v).half()
    return m(P), m(R), None


def engine(g, lr, ref, kpad, dev, ops):
    """rv_patch_pack (through `ops`) of smooth 16-channel maps at the LR and reference matching grids, in the engine's pairing"""
    split = kpad == 432
    dt = torch.float32 if split else torch.bfloat16
    fa, fb = make_feat(g, *lr, dt, dev), make_feat(g, *ref, dt, dev)
    A = torch.empty(lr[0] * lr[1], kpad, dtype=torch.float16, device=dev)
    B = torch.empty(ref[0] * ref[1], kpad, dtype=torch.float16, device=dev)
    ops.patch_pack(fa, A, 1 if split else 0)
    ops.patch_pack(fb, B, 2 if split else 0)
    return A, B, None


FAMILIES = {'planted': planted, 'duplicates': duplicates, 'negative': negative, 'generic': generic}


def make_operands(family, P, R, kpad, dev, seed, ops=None, lr=None, ref=None):
    g = _gen(dev, seed)
    if family == 'engine':
        return engine(g, lr, ref, kpad, dev, ops)
    return FAMILIES[family](g, P, R, kpad, dev)


# ------------------------------------------------------------------------------------------------------------------
# the check
# ------------------------------------------------------------------------------------------------------------------
def _row_where(m, plan):
    """where LR row m sits in the kernel: CTA, consumer, m64 block, warp quarter and the four lanes of its row"""
    if plan.impl == 0:
        return f'CTA {m // 64}, thread row {(m % 64) // 4}, lanes {16 * ((m % 64) // 4)}..{16 * ((m % 64) // 4) + 15} of the block'
    bm = 128 * plan.mb
    w = m % bm
    rr = w % 16
    return (f'CTA {m // bm}, consumer {w // (64 * plan.mb)}, m64 block {(w // 64) % plan.mb}, warp quarter {(w % 64) // 16}, '
            f'lanes {4 * (rr % 8)}..{4 * (rr % 8) + 3}, r2 {rr // 8}')


def _col_where(r, plan):
    """where reference row r sits in the scan: N tile and the accumulator column 8 j + 2 (lane & 3) + e"""
    if plan.impl == 0:
        return f'N tile {r // 64} (64 wide), lane&3 -, thread column {(r % 64) // 4}, j {r % 4}'
    c = r % MT_BN
    return f'N tile {r // MT_BN}, lane&3 {(c % 8) // 2}, j {c // 8}, e {c % 2}'


def _group_ids(B):
    """id of each B row's bit pattern: equal ids <=> bitwise-equal rows"""
    return torch.unique(B.view(torch.int16), dim=0, return_inverse=True)[1].to(torch.int32)


def check_rows(A, B, conf, idx, what, plan, score=None, widen=None, chunk=1024, expect=None):
    """conditions 1-5 of the module docstring for every row.  score(s, e) -> float64 S of rows s..e (default: the float64 GEMM
    of the operands); widen: float64 per-row term added to E_m (the composition's packing error; no copy rule then).  expect:
    per-row indices the family fixes (planted winners, lowest duplicates): each row's window must be that row alone or its
    copies.  Prints rows, rows resolved by a window of more than one and the largest |4096 conf - S*| / E; a failure report names
    the tile, lane and row of the first failing rows.  Returns (largest ratio, multi-row windows)."""
    P, K = A.shape
    R = B.shape[0]
    a64, b64 = A.double(), B.double()
    na = a64.norm(dim=1)
    E = C_ACC * K * U * na * float(b64.norm(dim=1).max())
    if widen is not None:
        E = E + widen
    if score is None:
        score = lambda s, e: a64[s:e] @ b64.t()                                      # noqa: E731
    gid = _group_ids(B) if widen is None else None
    c4 = conf.double() * 4096
    k = idx.long()
    bad = torch.zeros(P, 6, dtype=torch.bool, device=A.device)
    first_all = torch.zeros(P, dtype=torch.int64, device=A.device)
    sstar_all = torch.zeros(P, dtype=torch.float64, device=A.device)
    multi, worst = 0, 0.0
    for s in range(0, P, chunk):
        e = min(P, s + chunk)
        S = score(s, e)
        Sstar = S.max(dim=1).values
        Em = E[s:e]
        win = S >= (Sstar - 2 * Em)[:, None]
        first = win.to(torch.uint8).argmax(dim=1)                                  # lowest row of the window
        nwin = win.sum(dim=1)
        multi += int((nwin > 1).sum())
        kk = k[s:e]
        inr = (kk >= 0) & (kk < R)
        Sk = S.gather(1, kk.clamp(0, R - 1)[:, None])[:, 0]
        cc = c4[s:e]
        bad[s:e, 0] = ~inr
        bad[s:e, 1] = ~((cc - Sstar).abs() <= Em)
        bad[s:e, 2] = inr & ~(Sk >= Sstar - 2 * Em)
        bad[s:e, 3] = inr & ~((cc - Sk).abs() <= Em)
        if gid is not None:
            gmin = torch.where(win, gid[None, :], R).min(dim=1).values
            gmax = torch.where(win, gid[None, :], -1).max(dim=1).values
            copies = (gmin == gmax) | (na[s:e] == 0)
            bad[s:e, 4] = copies & (kk != first)
            if expect is not None:
                ex = expect[s:e]
                bad[s:e, 5] = ~copies | (first != ex) | (kk != ex)
        del S, win
        ratio = torch.where(Em > 0, (cc - Sstar).abs() / Em, torch.where(cc == Sstar, 0.0, math.inf))
        worst = max(worst, float(ratio.max()))
        first_all[s:e], sstar_all[s:e] = first, Sstar
    print(f'[match_fp64] {what}: {P} rows, {multi} resolved by a window of more than one row, '
          f'max |4096 conf - S*| / E = {worst:.4f}')
    if bool(bad.any()):
        pytest.fail(_explain(bad, k, c4, sstar_all, first_all, what, plan))
    return worst, multi


_COND = ['1: idx outside [0, R)', '2: conf is not S*', '3: idx outside the window', '4: conf is not the score of idx',
         '5: not the lowest of bitwise-equal rows', 'the family\'s expected index']


def _explain(bad, k, c4, sstar, first, what, plan):
    rows = bad.any(dim=1).nonzero()[:, 0]
    msg = [f'{what}: {rows.numel()} of {bad.shape[0]} rows fail; by condition: '
           + ', '.join(f'{_COND[i]}: {int(bad[:, i].sum())}' for i in range(6) if bool(bad[:, i].any()))]
    for m in rows[:6].tolist():
        conds = [str(i + 1) if i < 5 else 'expected' for i in range(6) if bool(bad[m, i])]
        msg.append(f'  row {m} ({_row_where(m, plan)}) returned idx {int(k[m])} ({_col_where(int(k[m]), plan)}), '
                   f'4096 conf = {float(c4[m])!r}; S* = {float(sstar[m])!r}, window starts at {int(first[m])} '
                   f'({_col_where(int(first[m]), plan)}); conditions {",".join(conds)}')
    if plan.impl == 1:
        bm = 128 * plan.mb
        kk = k[rows]
        for label, v in (('warp quarter', (rows % 64) // 16), ('lane & 3 of the returned column', (kk % 8) // 2),
                         ('N tile of the returned column', kk // MT_BN), ('CTA', rows // bm)):
            u, cnt = torch.unique(v, return_counts=True)
            top = cnt.argsort(descending=True)[:8]
            msg.append(f'  failing rows by {label}: ' + ', '.join(f'{int(u[j])}: {int(cnt[j])}' for j in top.tolist()))
    return '\n'.join(msg)


def run_guarded(fn, A, B, dev):
    """fn(A, B, conf, idx) with conf / idx GUARD elements into buffers of NaN / IDX_SENTINEL: the guards must be intact"""
    P = A.shape[0]
    cbuf = torch.full((P + 2 * GUARD,), float('nan'), device=dev)
    ibuf = torch.full((P + 2 * GUARD,), IDX_SENTINEL, dtype=torch.int32, device=dev)
    conf, idx = cbuf[GUARD:GUARD + P], ibuf[GUARD:GUARD + P]
    fn(A, B, conf, idx)
    if dev != 'cpu':
        torch.cuda.synchronize()
    for t in (cbuf[:GUARD], cbuf[GUARD + P:]):
        assert bool(torch.isnan(t).all()), 'conf written outside its P elements'
    for t in (ibuf[:GUARD], ibuf[GUARD + P:]):
        assert bool((t == IDX_SENTINEL).all()), 'idx written outside its P elements'
    return conf, idx


# ------------------------------------------------------------------------------------------------------------------
# CPU: the bound separates a correct kernel from subtly wrong ones
# ------------------------------------------------------------------------------------------------------------------
def fake_match(A, B, conf, idx, accum='k', mutant=None):
    """a CPU model of match_tc_kernel: fp32 accumulation of the exact products (accum 'k': in k order, 'reversed', 'k16': each
    16-column k-step summed on its own, then added), B zero-filled to whole 128-row N tiles, and the scan - thread lane & 3 = q
    of a row holds the columns 8 j + 2 q + e of each tile, keeps a running max with a strict > over its columns in increasing
    order (the last tile masked to the columns < R), and the four threads combine theirs, equal values to the lowest index.
    mutant: one planted defect (MUTANTS)."""
    P, K = A.shape
    R = B.shape[0]
    nt = (R + MT_BN - 1) // MT_BN
    a = A.float()
    b = torch.zeros(nt * MT_BN, K)
    b[:R] = B.float()
    cols = list(range(K))
    if mutant == 'tail-slice-dropped':
        t0 = (K // 64) * 64 + ((K % 64) // 16 - 1) * 16
        cols = [c for c in cols if not t0 <= c < t0 + 16]
    acc = torch.zeros(P, nt * MT_BN)
    if accum == 'k16':
        for s in range(0, K, 16):
            part = torch.zeros_like(acc)
            for c in [c for c in cols if s <= c < s + 16]:
                part = part + a[:, c, None] * b[None, :, c]
            acc = acc + part
    else:
        for c in (cols[::-1] if accum == 'reversed' else cols):
            acc = acc + a[:, c, None] * b[None, :, c]
    if mutant == 'bf16-accumulator':
        acc = acc.bfloat16().float()
    col = torch.arange(nt * MT_BN)
    valid = col <= R if mutant == 'ragged-mask-off-by-one' else col < R
    if mutant == 'last-tile-dropped':
        valid &= col < (nt - 1) * MT_BN
    q = (col % 8) // 2
    best, bidx = [], []
    for lq in range(4):
        v = torch.where((valid & (q == lq))[None, :], acc, torch.full_like(acc, -math.inf))
        mx = v.max(dim=1).values
        hit = (v == mx[:, None]) & (mx[:, None] > -math.inf)
        if mutant == 'scan-ge':                    # >= keeps the last maximum of the thread's columns
            j = torch.where(hit, col[None, :], -1).max(dim=1).values
        else:
            j = torch.where(hit, col[None, :], nt * MT_BN).min(dim=1).values
        j = torch.where(mx > -math.inf, j, torch.zeros_like(j))
        if mutant == 'lane-offset':                # rbase = tile + (lane & 3) instead of + 2 (lane & 3)
            j = j - lq
        best.append(mx)
        bidx.append(j)
    bv, bi = best[0], bidx[0]
    for lq in range(1, 4):
        ov, oi = best[lq], bidx[lq]
        tie_wins = oi > bi if mutant == 'combine-higher-index' else oi < bi
        take = (ov > bv) | ((ov == bv) & tie_wins)
        bv, bi = torch.where(take, ov, bv), torch.where(take, oi, bi)
    if mutant == 'conf-other-row':                 # r2 swapped: the row 8 apart within the 16-row group
        other = torch.arange(P) ^ 8
        bv = torch.where(other < P, bv[other.clamp(max=P - 1)], bv)
    conf.copy_(bv * (1.0 / 4096.0))
    idx.copy_(bi.to(torch.int32))


# CPU sizes: P = 300 rows (two 256-row CTAs, the second ragged), R = 700 (five full N tiles and a ragged one of 60 rows)
FAKE_LR, FAKE_REF, FAKE_K = (15, 20), (25, 28), 144


def _fake_case(family, seed, accum='k', mutant=None, kpad=FAKE_K):
    from u8_ops import U8OracleOps
    P, R = FAKE_LR[0] * FAKE_LR[1], FAKE_REF[0] * FAKE_REF[1]
    A, B, ex = make_operands(family, P, R, kpad, 'cpu', seed, ops=U8OracleOps(), lr=FAKE_LR, ref=FAKE_REF)
    conf, idx = run_guarded(lambda a, b, c, i: fake_match(a, b, c, i, accum, mutant), A, B, 'cpu')
    return A, B, conf, idx, ex


@pytest.mark.parametrize('accum', ['k', 'reversed', 'k16'])
@pytest.mark.parametrize('family', ['engine', 'planted', 'duplicates', 'negative', 'generic'])
def test_bound_passes_a_correct_kernel(family, accum):
    """the model with a correct scan passes on every family, whatever the fp32 accumulation order; the planted winners and
    the duplicates' lowest copies are returned exactly"""
    for kpad in ((FAKE_K, 432) if family == 'engine' else (FAKE_K,)):
        A, B, conf, idx, ex = _fake_case(family, _seed(family, kpad), accum, kpad=kpad)
        plan = match_plan(kpad, H100_SMEM_OPTIN)
        check_rows(A, B, conf, idx, f'fake {family} k{kpad} {accum}', plan, expect=ex, chunk=128)
        if family == 'engine':
            assert bool((A.double().norm(dim=1) == 0).any()), 'no all-zero A row'
            gid = _group_ids(B)
            assert int(gid.unique().numel()) < B.shape[0], 'no bitwise-equal B rows'


# (mutant, the family that exposes it)
MUTANTS = [
    ('last-tile-dropped', 'planted'),
    ('ragged-mask-off-by-one', 'negative'),
    ('lane-offset', 'planted'),
    ('scan-ge', 'duplicates'),
    ('combine-higher-index', 'duplicates'),
    ('tail-slice-dropped', 'generic'),
    ('conf-other-row', 'generic'),
    ('bf16-accumulator', 'planted'),
]


@pytest.mark.parametrize('mutant,family', MUTANTS, ids=[m[0] for m in MUTANTS])
def test_bound_fails_a_subtly_wrong_kernel(mutant, family):
    """each planted defect fails, with a report naming the tile, lane and row of the failing rows"""
    A, B, conf, idx, ex = _fake_case(family, _seed(family, FAKE_K), mutant=mutant)
    with pytest.raises(pytest.fail.Exception, match=r'rows fail(.|\n)*row \d+ \(CTA \d+, consumer \d, m64 block \d, '
                                                    r'warp quarter \d, lanes \d+\.\.\d+.*N tile \d+, lane&3 \d'):
        check_rows(A, B, conf, idx, f'fake {family} {mutant}', match_plan(FAKE_K, H100_SMEM_OPTIN), expect=ex, chunk=128)


def test_families_reach_their_targets():
    """the duplicates sit at every column residue of the first and a middle tile and in the ragged last tile, with groups
    found only there; their A rows cover both consumers, both m64 blocks, every warp quarter and the ragged last CTA; planted
    winners cover every reference row"""
    P, R, K = 1000, 700, 144
    A, B, low = duplicates(_gen('cpu', 1), P, R, K, 'cpu')
    gid = _group_ids(B)
    _, inv, cnt = torch.unique(gid, return_inverse=True, return_counts=True)
    dup = cnt[inv] > 1
    cols = torch.arange(R)[dup]
    for t in (0, (R + 127) // 128 // 2):
        assert set((cols[cols // 128 == t] % 128).tolist()) == set(range(128))
    last = cols[cols // 128 == R // 128]
    assert last.numel() == R % 128
    assert bool((low // 128 == R // 128).any()), 'no group found only in the ragged last tile'
    assert bool((A == B[low]).all()), 'every A row is a copied row'
    _, _, wp = planted(_gen('cpu', 2), 1000, 700, K, 'cpu')
    assert set(wp.tolist()) == set(range(700))
    An, Bn, _ = negative(_gen('cpu', 3), 30, 20, K, 'cpu')
    assert bool((An[::3].double() @ Bn.double().t() < 0).all())


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _device_plan(kpad, impl=1):
    return match_plan(kpad, torch.cuda.get_device_properties(0).shared_memory_per_block_optin, impl)


def _gpu_match(ops, impl):
    return lambda A, B, conf, idx: ops.match_argmax(A, B, conf, idx, impl=impl)


_ENGINE_CASES = [(e, f) for e in ENGINE_MATCH for f in ('engine', 'planted', 'duplicates', 'negative')]


@pytest.mark.gpu
@pytest.mark.parametrize('case', _ENGINE_CASES, ids=[f'impl{e.impl}-k{e.kpad}-{_pr(e)[0]}x{_pr(e)[1]}-{f}' for e, f in _ENGINE_CASES])
def test_engine_match(cuda_ops, case):
    e, family = case
    P, R = _pr(e)
    plan = _device_plan(e.kpad, e.impl)
    A, B, ex = make_operands(family, P, R, e.kpad, 'cuda', _seed(e, family), ops=cuda_ops, lr=e.lr, ref=e.ref)
    conf, idx = run_guarded(_gpu_match(cuda_ops, e.impl), A, B, 'cuda')
    _, multi = check_rows(A, B, conf, idx, f'impl{e.impl} k{e.kpad} {P}x{R} {family} (MB {plan.mb})', plan, expect=ex)
    if family == 'planted':
        assert multi == 0, 'planted winners must be alone in their windows'


_BRANCH = [(k, 1) for k in BRANCH_KPAD] + [(k, 0) for k in BRANCH_SIMT_KPAD]


@pytest.mark.gpu
@pytest.mark.parametrize('kpad,impl', _BRANCH, ids=[f'k{k}-impl{i}' for k, i in _BRANCH])
def test_match_branch(cuda_ops, kpad, impl):
    """one kpad (one launch plan) against every ragged P x R of the branch sets, with the generic, negative, duplicates and
    planted families"""
    plan = _device_plan(kpad, impl)
    print(f'[match_fp64] kpad {kpad} impl {impl}: {plan}')
    assert plan == match_plan(kpad, H100_SMEM_OPTIN, impl), \
        'this device\'s opt-in shared memory gives another launch plan than the H100 plans test_branch_cases_reach_every_plan covers'

    for P in BRANCH_P:
        for R in BRANCH_R:
            for family in ('generic', 'negative', 'duplicates', 'planted'):
                A, B, ex = make_operands(family, P, R, kpad, 'cuda', _seed(kpad, P, R, family))
                conf, idx = run_guarded(_gpu_match(cuda_ops, impl), A, B, 'cuda')
                check_rows(A, B, conf, idx, f'k{kpad} impl{impl} P{P} R{R} {family}', plan, expect=ex)


@pytest.mark.gpu
@pytest.mark.parametrize('kpad', [144, 432], ids=['single-k144', 'split-k432'])
def test_patch_pack_and_match_against_cosine_similarity(cuda_ops, kpad):
    """patch_pack + the GEMM at the x4 geometry against 4096 x the float64 cosine similarity of the fp64-normalised patches:
    the window widens by the packing error (and, in split mode, the dropped lo x lo term) - how far split mode's scores are
    from the exact ones, as a checked inequality"""
    e = Match(1, kpad, X4_GRID, REF1_GRID)
    split = kpad == 432
    g = _gen('cuda', _seed('composition', kpad))
    dt = torch.float32 if split else torch.bfloat16
    fa, fb = make_feat(g, *e.lr, dt, 'cuda'), make_feat(g, *e.ref, dt, 'cuda')
    P, R = _pr(e)
    A = torch.empty(P, kpad, dtype=torch.float16, device='cuda')
    B = torch.empty(R, kpad, dtype=torch.float16, device='cuda')
    cuda_ops.patch_pack(fa, A, 1 if split else 0)
    cuda_ops.patch_pack(fb, B, 2 if split else 0)
    conf, idx = run_guarded(_gpu_match(cuda_ops, 1), A, B, 'cuda')
    va, vb = ref_patches(fa), ref_patches(fb)                       # (P, 144), (R, 144) float64: 64 x unit patches
    K = va.shape[1]

    def err(v, packed, lo_col):
        hi = packed[:, :K].double()
        if lo_col is None:
            return ulp(v, torch.float16).norm(dim=1), None
        lo = packed[:, lo_col:lo_col + K].double()
        return (ulp(v - hi, torch.float16) + (K + C_AR) * U * v.abs()).norm(dim=1), lo.norm(dim=1)
    ea, la = err(va, A, K if split else None)
    eb, lb = err(vb, B, 2 * K if split else None)
    nva, nvb, ebm = va.norm(dim=1), float(vb.norm(dim=1).max()), float(eb.max())
    D = ea * nvb + nva * ebm + ea * ebm
    if split:
        D = D + la * float(lb.max())
    check_rows(A, B, conf, idx, f'composition k{kpad}', _device_plan(kpad), score=lambda s, t: va[s:t] @ vb.t(), widen=D)
    E = C_ACC * kpad * U * A.double().norm(dim=1) * float(B.double().norm(dim=1).max())
    rel = ((E + D) / 4096)[nva > 0]
    print(f'[match_fp64] composition k{kpad}: window half-width (E + packing) / 4096: median {float(rel.median()):.3g}, '
          f'max {float(rel.max()):.3g} of the cosine similarity')
