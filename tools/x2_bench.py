"""Throughput of a x2 model on one GPU: config_RefVSR_MFID with scale=2, matching_ksize=4, bf16, LR 540x960 -> 1080x1920 with the
Ref at 540x960 (the eval size of the x2 models: LR and Ref both come from LRx2).

    python tools/x2_bench.py [--steps 27] [--warmup 9] [--reps 3] [--json OUT]

Frames are seeded synthetic clips (refvsr_b200.synth.make_clip_range), weights seeded_test_weights(1234).  Like bench.py's resident
leg, the frames are on the device before timing starts, and the CUDA graphs of every window kind are captured in an untimed pass
over the same windows.  Reported (CUDA events, device time):
  * frames/s over `steps` consecutive windows of one stream (forced resets every reset_branch windows included, as in bench.py);
  * the median device time of a steady window (each window timed on its own) and of a first / forced-reset window.
The card's name, power limit and SM clocks are read in the same run and printed with the numbers."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W, T = 540, 960, 7


def window_indices(k, n):
    return [min(max(k - T // 2 + j, 0), n - 1) for j in range(T)]      # data_loader/datasets.py:233-234


def card():
    import torch
    q = 'name,power.limit,clocks.max.sm,clocks.sm'
    try:
        row = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), f'--query-gpu={q}', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as ex:                                                 # noqa: BLE001
        row = f'nvidia-smi unavailable ({ex})'
    return {'device': torch.cuda.get_device_name(), 'nvidia_smi': row}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=27)
    ap.add_argument('--warmup', type=int, default=9)
    ap.add_argument('--reps', type=int, default=3, help='timed passes over the same windows')
    ap.add_argument('--precision', default='bf16', choices=['bf16', 'fp16', 'fp32'])
    ap.add_argument('--json', default=None, help='also write the result here')
    args = ap.parse_args()
    import torch
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip_range
    if not torch.cuda.is_available():
        raise SystemExit('x2_bench: needs a CUDA device')
    dev = torch.device('cuda', 0)
    cfg = get_config('config_RefVSR_MFID', device='cuda', scale=2, matching_ksize=4, b200_precision=args.precision)
    net = SRNet(cfg).eval()
    seeded_test_weights(net, seed=1234)
    net = net.to(dev)
    Wm, K = args.warmup, args.steps
    n = Wm + K
    lrs, refs = make_clip_range(0, n, H, W, 1, seed=1234)
    lrs, refs = lrs.to(dev), refs.to(dev)
    assert tuple(refs.shape[2:]) == (H, W)

    def step(k):
        idx = torch.tensor(window_indices(k, n), device=dev)
        return net(lrs.index_select(0, idx).unsqueeze(0), refs.index_select(0, idx).unsqueeze(0), k == 0, False, False)['result']

    with torch.no_grad():
        net.Network.reset_state()
        for k in range(n):                                                 # untimed: graph capture of every window kind
            out = step(k)
        assert out.shape == (1, 3, 2 * H, 2 * W)
        torch.cuda.synchronize()
        fps, steady, first = [], [], []
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
            fps.append(K / (e0.elapsed_time(e1) / 1e3))
        # per-window device time (each window bracketed by its own events)
        net.Network.reset_state()
        rb = cfg.reset_branch
        for k in range(n):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(k)
            b.record()
            torch.cuda.synchronize()
            if k >= Wm or k % rb == 0:
                (first if k % rb == 0 else steady).append(a.elapsed_time(b))
    res = dict(workload='config_RefVSR_MFID x2', precision=args.precision, lr=f'{H}x{W}', ref=f'{H}x{W}', out=f'{2 * H}x{2 * W}',
               T=T, steps=K, warmup=Wm, reps=args.reps, frames_per_s=[round(v, 2) for v in fps],
               frames_per_s_median=round(statistics.median(fps), 2),
               steady_window_ms_median=round(statistics.median(steady), 2), steady_windows=len(steady),
               first_window_ms_median=round(statistics.median(first), 2) if first else None, **card())
    line = json.dumps(res)
    print(line, flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
