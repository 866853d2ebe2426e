"""Cost of 4:2:0 (I420) frames through the engine against 8-bit RGB frames; prints JSON lines, the first naming the card, its power
limit and SM clock.

  tail    device time of one rv_reconstruct_u8 writing RGB against I420, at 270x480 -> 1080x1920 and 1080x1920 -> 4320x7680.
          CUDA events over replays of a graph of --calls launches, median of --reps, with the bytes each must move (16 read per
          output pixel for conv_last's output, then 3 or 1.5 written; the LR frame's reads aside) and the share of the data
          sheet's 3.35 TB/s floor.
  input   device time of one rv_frames_from_u8 launch converting an LR + Ref pair into fp32 planes, RGB against I420, for 270x480
          and 1080x1920 frames (3 or 1.5 bytes read and 12 written per pixel).
  stream  a streaming loop from pinned host buffers, one engine per arm, the clip's first window through forward, then one push
          per step; a yuv420p caller (I420 frames in, I420 frames out):
            rgb+cv2  cv2.cvtColor I420 -> RGB of the LR and Ref frames on the host, uploaded, push_frame_u8, the RGB result
                     downloaded and converted RGB -> I420 on the host, one thread
            i420     the I420 frames uploaded, push_frame_yuv420, the I420 result downloaded
          RefVSR_MFID 270x480 -> 1080x1920 in bf16 (--steps steps per arm, the arms alternated --rounds times), then with --hd-steps
          > 0 the flag_HD_in RefVSR_MFID_8K at 1080x1920 -> 4320x7680 the same way.  Frames/s per round, median and spread."""
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
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    name, power, sm, sm_max = [v.strip() for v in q.stdout.strip().splitlines()[0].split(',')]
    return {'card': name, 'power_limit': power, 'sm_clock': sm, 'sm_clock_max': sm_max, 'torch_device': torch.cuda.get_device_name()}


def graph_time(fn, calls, reps):
    """median, min and max seconds of one fn() from CUDA events around replays of a graph of `calls` fn() launches"""
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


def _row(leg, arm, shape, t, nbytes):
    med, lo, hi = t
    return {'leg': leg, 'arm': arm, 'shape': shape, 'us': round(med * 1e6, 1), 'us_min': round(lo * 1e6, 1),
            'us_max': round(hi * 1e6, 1), 'bytes': nbytes, 'hbm_floor_share': round(nbytes / HBM_BPS / med, 3)}


def tail(ops, h, w, calls, reps):
    from refvsr_b200.lib import FRAME_I420, FRAME_RGB
    H, W = 4 * h, 4 * w
    g = torch.Generator(device='cuda').manual_seed(h)
    x = torch.rand(H, W, 4, device='cuda', generator=g) * 0.2 - 0.1
    lr = torch.rand(3, h, w, device='cuda', generator=g)
    rgb = torch.empty(H, W, 3, dtype=torch.uint8, device='cuda')
    yuv = torch.empty(3 * H // 2, W, dtype=torch.uint8, device='cuda')
    res = []
    for arm, out, fmt, bpp in (('rgb', rgb, FRAME_RGB, 16 + 3), ('i420', yuv, FRAME_I420, 16 + 1.5)):
        t = graph_time(lambda: ops.reconstruct_u8(x, lr, 4, True, out, fmt), calls, reps)
        res.append(_row('tail', arm, f'{H}x{W}', t, int(bpp * H * W)))
    return res


def inputs(ops, h, w, calls, reps):
    from refvsr_b200.lib import FRAME_I420, FRAME_RGB, frame_shape
    res = []
    dst = [torch.empty(3, h, w, device='cuda') for _ in range(2)]
    for arm, fmt, bpp in (('rgb', FRAME_RGB, 3 + 12), ('i420', FRAME_I420, 1.5 + 12)):
        src = [torch.randint(0, 256, frame_shape(h, w, fmt), dtype=torch.uint8, device='cuda') for _ in range(2)]
        t = graph_time(lambda: ops.frames_from_u8(src, dst, fmt), calls, reps)
        res.append(_row('input', arm, f'2x{h}x{w}', t, int(bpp * 2 * h * w)))
    return res


def stream(config, h, w, steps, rounds, warm):
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip_range
    nets = {}
    for arm in ('rgb+cv2', 'i420'):
        cfg = get_config(config, device='cuda', b200_precision='bf16')
        net = SRNet(cfg).eval()
        seeded_test_weights(net, seed=3)
        nets[arm] = net.cuda()
    t, s = cfg.frame_num, nets['i420'].Network.scale
    nclip = 12
    lrs, refs = make_clip_range(0, nclip, h, w)
    hr, wr = refs.shape[-2:]

    def i420(x):
        return cv2.cvtColor(np.ascontiguousarray((x.permute(1, 2, 0).numpy() * 255).round().astype(np.uint8)), cv2.COLOR_RGB2YUV_I420)
    lr8, rf8 = [i420(lrs[i]) for i in range(nclip)], [i420(refs[i]) for i in range(nclip)]
    H, W = s * h, s * w
    pin = dict(lry=torch.empty(3 * h // 2, w, dtype=torch.uint8).pin_memory(), rfy=torch.empty(3 * hr // 2, wr, dtype=torch.uint8).pin_memory(),
               outy=torch.empty(3 * H // 2, W, dtype=torch.uint8).pin_memory(),
               lr8=torch.empty(h, w, 3, dtype=torch.uint8).pin_memory(), rf8=torch.empty(hr, wr, 3, dtype=torch.uint8).pin_memory(),
               out8=torch.empty(H, W, 3, dtype=torch.uint8).pin_memory())
    first = [min(max(j - t // 2, 0), nclip - 1) for j in range(t)]
    with torch.no_grad():
        nets['i420'].forward_yuv420(torch.from_numpy(np.stack([lr8[i] for i in first]))[None].cuda(),
                                    torch.from_numpy(np.stack([rf8[i] for i in first]))[None].cuda(), True)
        nets['rgb+cv2'].forward_u8(torch.from_numpy(np.stack([cv2.cvtColor(lr8[i], cv2.COLOR_YUV2RGB_I420) for i in first]))[None].cuda(),
                                   torch.from_numpy(np.stack([cv2.cvtColor(rf8[i], cv2.COLOR_YUV2RGB_I420) for i in first]))[None].cuda(), True)
    pos = {'rgb+cv2': t // 2 + 1, 'i420': t // 2 + 1}

    def step_yuv(i):
        pin['lry'].numpy()[...] = lr8[i]
        pin['rfy'].numpy()[...] = rf8[i]
        o = nets['i420'].push_frame_yuv420(pin['lry'].cuda(non_blocking=True), pin['rfy'].cuda(non_blocking=True))
        pin['outy'].copy_(o, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return pin['outy'].numpy()

    def step_rgb(i):
        pin['lr8'].numpy()[...] = cv2.cvtColor(lr8[i], cv2.COLOR_YUV2RGB_I420)
        pin['rf8'].numpy()[...] = cv2.cvtColor(rf8[i], cv2.COLOR_YUV2RGB_I420)
        o = nets['rgb+cv2'].push_frame_u8(pin['lr8'].cuda(non_blocking=True), pin['rf8'].cuda(non_blocking=True))
        pin['out8'].copy_(o, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return cv2.cvtColor(pin['out8'].numpy(), cv2.COLOR_RGB2YUV_I420)

    fns = {'rgb+cv2': step_rgb, 'i420': step_yuv}

    def run(arm, n):
        t0 = time.perf_counter()
        for _ in range(n):
            fns[arm](pos[arm] % nclip)
            pos[arm] += 1
        return n / (time.perf_counter() - t0)

    with torch.no_grad():
        a, b = step_rgb(pos['rgb+cv2'] % nclip), step_yuv(pos['i420'] % nclip)    # the two arms agree byte for byte
        assert np.array_equal(a, b), 'push_frame_yuv420 differs from cvtColor(push_frame_u8(cvtColor(frame)))'
        pos = {k: v + 1 for k, v in pos.items()}
        for arm in fns:
            run(arm, warm)
        fps = {arm: [] for arm in fns}
        for _ in range(rounds):
            for arm in fns:
                fps[arm].append(run(arm, steps))
    out = [{'leg': 'stream', 'arm': arm, 'config': config, 'shape': f'{h}x{w}->{H}x{W}', 'precision': 'bf16', 'steps': steps,
            'fps': [round(v, 2) for v in v_], 'fps_median': round(statistics.median(v_), 2),
            'fps_spread': round(max(v_) - min(v_), 2)} for arm, v_ in fps.items()]
    del nets
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--calls', type=int, default=20)
    ap.add_argument('--reps', type=int, default=15)
    ap.add_argument('--steps', type=int, default=24)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--warm', type=int, default=8)
    ap.add_argument('--hd-steps', type=int, default=0, help='steps per round of the flag_HD_in stream (0: not run)')
    ap.add_argument('--out', default=None, help='also write the JSON lines to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('yuv_stream_bench needs a CUDA device')
    from refvsr_b200.lib import CudaOps
    ops = CudaOps()
    lines = []

    def emit(rows):
        for ln in rows:
            print(json.dumps(ln), flush=True)
            lines.append(ln)
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, 'w') as f:
                f.write(''.join(json.dumps(ln) + '\n' for ln in lines))

    emit([card()])
    for h, w in ((270, 480), (1080, 1920)):
        emit(tail(ops, h, w, args.calls, args.reps))
    for h, w in ((270, 480), (1080, 1920)):
        emit(inputs(ops, h, w, args.calls, args.reps))
    emit(stream('RefVSR_MFID', 270, 480, args.steps, args.rounds, args.warm))
    if args.hd_steps > 0:
        emit(stream('RefVSR_MFID_8K', 1080, 1920, args.hd_steps, args.rounds, 2))
    emit([card()])


if __name__ == '__main__':
    main()
