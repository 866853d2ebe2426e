"""-m gpu: Network.forward / push_frames with n > 1 windows per call (one batched window schedule) against n independent engines
with the same weights, each fed one clip: the results must be the same bits, window by window, across first windows, steady
windows, forced resets (reset_branch) and the windows after them."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _engine(name, prec, seed, **over):
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    net = SRNet(get_config(name, device='cuda', b200_precision=prec, **over)).eval()
    seeded_test_weights(net, seed=seed)
    return net.cuda()


def _clips(n, frames, h, w, T, seed):
    from refvsr_b200.synth import make_clip, sliding_windows
    return [list(sliding_windows(*make_clip(frames, h, w, 1, seed=seed + 17 * i), T)) for i in range(n)]


def _check_batch(name, prec, n, h, w, frames=12, T=7, seed=5, **over):
    wins = _clips(n, frames, h, w, T, seed)
    batched = _engine(name, prec, seed, **over)
    singles = [_engine(name, prec, seed, **over) for _ in range(n)]
    for k in range(frames):
        first = wins[0][k][3]
        wl = torch.cat([wins[i][k][1] for i in range(n)]).cuda()
        wr = torch.cat([wins[i][k][2] for i in range(n)]).cuda()
        out = batched(wl, wr, first, False, False)['result']
        assert out.shape[0] == n
        for i in range(n):
            exp = singles[i](wins[i][k][1].cuda(), wins[i][k][2].cuda(), first, False, False)['result'][0]
            assert torch.equal(out[i], exp), f'window {k}, element {i}: the batched window differs from its own engine'
    net = batched.Network
    assert net.batch_fallbacks == 0 and net.reuse_fallbacks == 0
    if net.use_graphs:
        assert any(key[0] == 'batch' for key in net._graphs), 'the steady windows must run as one batched graph'


CASES = [
    ('small-bf16-n2', 'RefVSR_small_MFID', 'bf16', 2, 24, 32, dict(num_blocks=2)),
    ('small-fp16-n3-eager', 'RefVSR_small_MFID', 'fp16', 3, 24, 32, dict(num_blocks=2, b200_cuda_graphs=False)),
    ('small-fp32-n2', 'RefVSR_small_MFID', 'fp32', 2, 24, 32, dict(num_blocks=2)),
    ('mfid-bf16-n3-no-overlap', 'RefVSR_MFID', 'bf16', 3, 40, 56, dict(num_blocks=3, b200_overlap_branches=False)),
    ('mfid-bf16-n2-eager-overlap', 'RefVSR_MFID', 'bf16', 2, 40, 56, dict(num_blocks=3, b200_cuda_graphs=False)),
    ('small8k-bf16-n2', 'RefVSR_small_MFID_8K', 'bf16', 2, 48, 64, dict(num_blocks=2)),
    ('x2-small-bf16-n2', 'RefVSR_small_MFID', 'bf16', 2, 40, 56, dict(num_blocks=2, scale=2, matching_ksize=4)),
    ('x2-small-fp16-n3', 'RefVSR_small_MFID', 'fp16', 3, 40, 56, dict(num_blocks=2, scale=2, matching_ksize=4)),
]


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_batched_forward_equals_independent_engines(case):
    _, name, prec, n, h, w, over = case
    _check_batch(name, prec, n, h, w, **over)


def test_batched_forward_full_size_mfid():
    """MFID, 30 blocks, 270 x 480, two clips: first window, steady windows, the forced reset at window 9 and after it"""
    _check_batch('RefVSR_MFID', 'bf16', 2, 270, 480, frames=11)


def test_batched_reuse_guard_one_element_does_not_slide():
    """element 1 jumps within its clip while element 0 slides: the call runs element by element, element 1 is recomputed from
    scratch, and every output still equals its independent engine; later calls batch again"""
    n, T, frames = 2, 7, 12
    wins = _clips(n, frames, 24, 32, T, 3)
    over = dict(num_blocks=2)
    batched = _engine('RefVSR_small_MFID', 'bf16', 3, **over)
    singles = [_engine('RefVSR_small_MFID', 'bf16', 3, **over) for _ in range(n)]
    order = [[0, 1, 2, 3, 4, 5, 6, 7, 8], [0, 1, 2, 6, 7, 8, 9, 10, 11]]
    for step in range(len(order[0])):
        picks = [wins[i][order[i][step]] for i in range(n)]
        first = step == 0
        wl = torch.cat([p[1] for p in picks]).cuda()
        wr = torch.cat([p[2] for p in picks]).cuda()
        out = batched(wl, wr, first, False, False)['result']
        for i in range(n):
            exp = singles[i](picks[i][1].cuda(), picks[i][2].cuda(), first, False, False)['result'][0]
            assert torch.equal(out[i], exp), f'step {step}, element {i}'
    net = batched.Network
    assert net.reuse_fallbacks == 1 and singles[1].Network.reuse_fallbacks == 1
    assert net.batch_fallbacks >= 1
    assert any(key[0] == 'batch' for key in net._graphs)


def test_batched_push_frames_equals_batched_forward():
    n, T, frames = 3, 7, 12
    wins = _clips(n, frames, 40, 56, T, 11)
    outs = {}
    for mode in ('forward', 'push'):
        net = _engine('RefVSR_MFID', 'bf16', 11, num_blocks=2)
        res = []
        for k in range(frames):
            wl = torch.cat([wins[i][k][1] for i in range(n)]).cuda()
            wr = torch.cat([wins[i][k][2] for i in range(n)]).cuda()
            if mode == 'forward' or k == 0:
                res.append(net(wl, wr, k == 0, False, False)['result'].cpu())
            else:
                res.append(net.push_frames(wl[:, -1].contiguous(), wr[:, -1].contiguous()).cpu())
        outs[mode] = res
        assert net.Network.batch_fallbacks == 0
    for k, (a, b) in enumerate(zip(outs['push'], outs['forward'])):
        assert torch.equal(a, b), f'window {k}: push_frames differs from the batched forward()'
