"""Device time of the matching GEMM (rv_match_argmax, impl=1) at the bench workload's shape: P = 270 x 480 LR patches against
R = 135 x 240 reference patches of 16 channels x 3 x 3 = 144 values.

    python tools/match_bench.py [--kpad 144 192 432 448] [--iters 10] [--reps 5] [--json OUT]

Operands are patches of seeded random features packed by rv_patch_pack: single mode (one fp16 pass) at kpad 144 / 192, split
mode (fp16 hi / lo, three passes) at kpad 432 / 448; columns past 144 (3 x 144) are zero.  Like bench.py's timeit, `iters`
launches are captured into one CUDA graph and each replay is timed with CUDA events; the median over `reps` replays is
reported per launch.  TFLOP/s is algorithmic: 2 P R 144 = 1.209 TFLOP per call, x3 in split mode, whatever kpad is issued.
The card's name, power limit and SM clocks are read in the same run and printed with the numbers.  A kpad the library rejects
is reported with its error."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W, C = 270, 480, 16


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
    ap.add_argument('--kpad', type=int, nargs='+', default=[144, 192, 432, 448])
    ap.add_argument('--iters', type=int, default=10, help='launches per CUDA graph')
    ap.add_argument('--reps', type=int, default=5, help='timed graph replays')
    ap.add_argument('--json', default=None, help='also write the result lines here')
    args = ap.parse_args()
    import torch
    from refvsr_b200.lib import CudaOps
    if not torch.cuda.is_available():
        raise SystemExit('match_bench: needs a CUDA device')
    ops = CudaOps()
    g = torch.Generator().manual_seed(1234)
    lr_f = (torch.rand((H, W, C), generator=g) * 2 - 1).cuda()
    ref_f = (torch.rand((H // 2, W // 2, C), generator=g) * 2 - 1).cuda()
    P, R = H * W, (H // 2) * (W // 2)
    info = card()
    lines = []
    for kpad in args.kpad:
        split = kpad >= 3 * 144
        A = torch.empty((P, kpad), dtype=torch.float16, device='cuda')
        B = torch.empty((R, kpad), dtype=torch.float16, device='cuda')
        ops.patch_pack(lr_f, A, 1 if split else 0)
        ops.patch_pack(ref_f, B, 2 if split else 0)
        conf = torch.empty(P, device='cuda')
        idx = torch.empty(P, dtype=torch.int32, device='cuda')
        flop = 2.0 * P * R * 144 * (3 if split else 1)
        res = dict(kernel='rv_match_argmax', P=P, R=R, kpad=kpad, mode='split' if split else 'single', algorithmic_tflop=round(flop / 1e12, 3))
        try:
            for _ in range(2):
                ops.match_argmax(A, B, conf, idx, impl=1)
            torch.cuda.synchronize()
        except (ValueError, RuntimeError) as ex:
            res['error'] = str(ex)
            lines.append(res)
            print(json.dumps(res), flush=True)
            continue
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(args.iters):
                ops.match_argmax(A, B, conf, idx, impl=1)
        graph.replay()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            graph.replay()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1) / args.iters)
        med = statistics.median(ms)
        res.update(ms_median=round(med, 4), ms_min=round(min(ms), 4), ms_max=round(max(ms), 4),
                   tflops_algorithmic=round(flop / (med * 1e-3) / 1e12, 1), **info)
        lines.append(res)
        print(json.dumps(res), flush=True)
        del graph
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            f.write(''.join(json.dumps(r) + '\n' for r in lines))


if __name__ == '__main__':
    main()
