"""Cost of the 8-bit streaming path against the fp32 one; prints JSON lines, the first naming the card and its power limit.

  tail    device time of the window's tail as a caller who wants 8-bit frames runs it: rv_reconstruct + rv_eval_images (fp32
          result, then its BGR bytes) against one rv_reconstruct_u8 (bgr), at 270x480 -> 1080x1920 and 1080x1920 -> 4320x7680.
          CUDA events over replays of a graph of --calls launches of each, median of --reps, with the bytes each must move
          (fp32: 16 read + 12 written + 12 read + 3 written per output pixel; u8: 16 read + 3 written, the LR frame's reads
          aside) and the share of the data sheet's 3.35 TB/s floor.
  stream  a streaming loop from pinned host buffers, RefVSR_MFID at 270x480 -> 1080x1920 in bf16 (one engine per arm, the clip's
          first window through forward, then one push per step):
            u8    uint8 RGB frames uploaded, push_frame_u8, the uint8 RGB result downloaded
            fp32  the same uint8 frames converted on the host (np / 255 into fp32 CHW), uploaded, push_frame, the fp32 result
                  downloaded and converted on the host to uint8 BGR (cv2.cvtColor(x * 255, RGB2BGR).astype(uint8) after the
                  CHW -> HWC transpose), one thread
          --steps steps per arm, the arms alternated --rounds times; frames/s per round, median and spread."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cv2                                                            # noqa: E402
import numpy as np                                                    # noqa: E402
import torch                                                          # noqa: E402

HBM_BPS = 3.35e12


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    name, power = [v.strip() for v in q.stdout.strip().splitlines()[0].split(',')]
    return {'card': name, 'power_limit': power, 'torch_device': torch.cuda.get_device_name()}


def graph_time(fn, calls, reps):
    """median seconds of one fn() from CUDA events around replays of a graph of `calls` fn() launches"""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(calls):
            fn()
    for _ in range(3):
        g.replay()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / 1e3 / calls)
    return statistics.median(ts), min(ts), max(ts)


def tail(ops, h, w, calls, reps):
    H, W = 4 * h, 4 * w
    g = torch.Generator(device='cuda').manual_seed(h)
    x = torch.rand(H, W, 4, device='cuda', generator=g) * 0.2 - 0.1
    lr = torch.rand(3, h, w, device='cuda', generator=g)
    out32 = torch.empty(1, 3, H, W, device='cuda')
    out8 = torch.empty(H, W, 3, dtype=torch.uint8, device='cuda')

    def fp32():
        ops.reconstruct(x, lr, 4, True, out32[0])
        ops.eval_images([out32])

    def u8():
        ops.reconstruct_u8(x, lr, 4, True, out8, True)

    fp32()
    u8()
    torch.cuda.synchronize()
    assert torch.equal(ops.eval_images([out32]).view(H, W, 3), out8), 'rv_reconstruct_u8 bytes differ from the fp32 path'
    res = []
    for arm, fn, bpp in (('fp32+eval_images', fp32, 16 + 12 + 12 + 3), ('u8', u8, 16 + 3)):
        med, lo, hi = graph_time(fn, calls, reps)
        nbytes = bpp * H * W
        res.append({'leg': 'tail', 'arm': arm, 'out': f'{H}x{W}', 'us': round(med * 1e6, 1), 'us_min': round(lo * 1e6, 1),
                    'us_max': round(hi * 1e6, 1), 'bytes': nbytes, 'hbm_floor_share': round(nbytes / HBM_BPS / med, 3)})
    return res


def stream(steps, rounds, warm):
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip_range
    h, w, t = 270, 480, 7
    nclip = 24
    lrs, refs = make_clip_range(0, nclip, h, w)
    lr8 = [np.ascontiguousarray((lrs[i].permute(1, 2, 0).numpy() * 255).round().astype(np.uint8)) for i in range(nclip)]
    rf8 = [np.ascontiguousarray((refs[i].permute(1, 2, 0).numpy() * 255).round().astype(np.uint8)) for i in range(nclip)]
    nets = {}
    for arm in ('u8', 'fp32'):
        net = SRNet(get_config('RefVSR_MFID', device='cuda', b200_precision='bf16')).eval()
        seeded_test_weights(net, seed=3)
        nets[arm] = net.cuda()
    pin = dict(lr8=torch.empty(h, w, 3, dtype=torch.uint8).pin_memory(), rf8=torch.empty(h, w, 3, dtype=torch.uint8).pin_memory(),
               out8=torch.empty(4 * h, 4 * w, 3, dtype=torch.uint8).pin_memory(),
               lr32=torch.empty(3, h, w).pin_memory(), rf32=torch.empty(3, h, w).pin_memory(),
               out32=torch.empty(3, 4 * h, 4 * w).pin_memory())
    first = [min(max(j - t // 2, 0), nclip - 1) for j in range(t)]
    with torch.no_grad():
        nets['u8'].forward_u8(torch.from_numpy(np.stack([lr8[i] for i in first]))[None].cuda(),
                              torch.from_numpy(np.stack([rf8[i] for i in first]))[None].cuda(), True)
        nets['fp32'](lrs[first][None].cuda(), refs[first][None].cuda(), True)
    pos = {'u8': t // 2 + 1, 'fp32': t // 2 + 1}

    def step_u8(i):
        pin['lr8'].numpy()[...] = lr8[i]
        pin['rf8'].numpy()[...] = rf8[i]
        o = nets['u8'].push_frame_u8(pin['lr8'].cuda(non_blocking=True), pin['rf8'].cuda(non_blocking=True))
        pin['out8'].copy_(o, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return pin['out8'].numpy()

    def step_fp32(i):
        pin['lr32'].numpy()[...] = lr8[i].transpose(2, 0, 1) / np.float32(255)
        pin['rf32'].numpy()[...] = rf8[i].transpose(2, 0, 1) / np.float32(255)
        o = nets['fp32'].push_frame(pin['lr32'].cuda(non_blocking=True), pin['rf32'].cuda(non_blocking=True))
        pin['out32'].copy_(o, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return cv2.cvtColor(pin['out32'].numpy().transpose(1, 2, 0) * 255, cv2.COLOR_RGB2BGR).astype(np.uint8)

    fns = {'u8': step_u8, 'fp32': step_fp32}

    def run(arm, n):
        t0 = time.perf_counter()
        for _ in range(n):
            fns[arm](pos[arm] % nclip)
            pos[arm] += 1
        return n / (time.perf_counter() - t0)

    with torch.no_grad():
        for arm in fns:
            run(arm, warm)
        fps = {'u8': [], 'fp32': []}
        for _ in range(rounds):
            for arm in ('u8', 'fp32'):
                fps[arm].append(run(arm, steps))
    return [{'leg': 'stream', 'arm': arm, 'shape': '270x480->1080x1920', 'precision': 'bf16', 'steps': steps,
             'fps': [round(v, 2) for v in v_], 'fps_median': round(statistics.median(v_), 2),
             'fps_spread': round(max(v_) - min(v_), 2)} for arm, v_ in fps.items()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--calls', type=int, default=20)
    ap.add_argument('--reps', type=int, default=15)
    ap.add_argument('--steps', type=int, default=24)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--warm', type=int, default=8)
    ap.add_argument('--out', default=None, help='also write the JSON lines to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('u8_stream_bench needs a CUDA device')
    from refvsr_b200.lib import CudaOps
    ops = CudaOps()
    lines = [card()]
    for h, w in ((270, 480), (1080, 1920)):
        lines += tail(ops, h, w, args.calls, args.reps)
    lines += stream(args.steps, args.rounds, args.warm)
    lines.append(card())
    for ln in lines:
        print(json.dumps(ln), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(''.join(json.dumps(ln) + '\n' for ln in lines))


if __name__ == '__main__':
    main()
