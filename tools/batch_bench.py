"""Throughput of n clips per forward() call on one GPU: config_RefVSR_MFID, bf16, LR 270x480 -> 1080x1920, Ref 270x480, T = 7,
at each batch size of --batch (default 1, 2, 4).

    python tools/batch_bench.py [--batch 1 2 4] [--steps 27] [--warmup 9] [--reps 3] [--json OUT]

Timed as tools/x2_bench.py times one stream: seeded synthetic clips (one per batch element, different scenes) resident on the
device, the CUDA graphs of every window kind captured in an untimed pass, then `steps` consecutive windows between CUDA events
(forced resets every reset_branch windows included).  Reported per batch size: frames/s per card (n frames per window) and per
clip (one stream's rate), and the median device time of a steady window.  The card's name, power limit and SM clocks are read
in the same run and printed with the numbers."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from x2_bench import card  # noqa: E402

H, W, T = 270, 480, 7


def window_indices(k, n):
    return [min(max(k - T // 2 + j, 0), n - 1) for j in range(T)]      # data_loader/datasets.py:233-234


def run(nb, args):
    import torch
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip_range
    dev = torch.device('cuda', 0)
    cfg = get_config('config_RefVSR_MFID', device='cuda', b200_precision=args.precision)
    net = SRNet(cfg).eval()
    seeded_test_weights(net, seed=1234)
    net = net.to(dev)
    Wm, K = args.warmup, args.steps
    n = Wm + K
    clips = [make_clip_range(0, n, H, W, 1, seed=1234 + i) for i in range(nb)]
    lrs = torch.stack([c[0] for c in clips]).to(dev)          # (nb, frames, 3, H, W)
    refs = torch.stack([c[1] for c in clips]).to(dev)

    def step(k):
        idx = torch.tensor(window_indices(k, n), device=dev)
        return net(lrs.index_select(1, idx), refs.index_select(1, idx), k == 0, False, False)['result']

    with torch.no_grad():
        net.Network.reset_state()
        for k in range(n):                                                 # untimed: graph capture of every window kind
            out = step(k)
        assert out.shape == (nb, 3, 4 * H, 4 * W)
        torch.cuda.synchronize()
        fps = []
        for rep in range(args.reps):
            net.Network.reset_state()
            for k in range(Wm):
                step(k)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for k in range(Wm, n):
                step(k)
            e1.record()
            torch.cuda.synchronize()
            fps.append(nb * K / (e0.elapsed_time(e1) / 1e3))
        net.Network.reset_state()
        rb, steady = cfg.reset_branch, []
        for k in range(n):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(k)
            b.record()
            torch.cuda.synchronize()
            if k >= Wm and k % rb:
                steady.append(a.elapsed_time(b))
    assert net.Network.batch_fallbacks == 0
    med = statistics.median(fps)
    return dict(n=nb, frames_per_s_card=[round(v, 2) for v in fps], frames_per_s_card_median=round(med, 2),
                frames_per_s_per_clip_median=round(med / nb, 2), steady_window_ms_median=round(statistics.median(steady), 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, nargs='+', default=[1, 2, 4])
    ap.add_argument('--steps', type=int, default=27)
    ap.add_argument('--warmup', type=int, default=9)
    ap.add_argument('--reps', type=int, default=3, help='timed passes over the same windows')
    ap.add_argument('--precision', default='bf16', choices=['bf16', 'fp16', 'fp32'])
    ap.add_argument('--json', default=None, help='also write the result here')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('batch_bench: needs a CUDA device')
    rows = []
    for nb in args.batch:
        rows.append(run(nb, args))
        print(json.dumps(rows[-1]), flush=True)
        torch.cuda.empty_cache()
    res = dict(workload='config_RefVSR_MFID', precision=args.precision, lr=f'{H}x{W}', ref=f'{H}x{W}', out=f'{4 * H}x{4 * W}',
               T=T, steps=args.steps, warmup=args.warmup, reps=args.reps, batches=rows, **card())
    line = json.dumps(res)
    print(line, flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
