"""Cost of the default evaluation mode's image work (`run.py --eval_mode qual_quan`, evaluation/eval_qual_quan.py) per frame;
prints JSON lines.

  kernel  one CudaOps.eval_images call (rv_eval_images, CUDA events, median of --calls) on a 1080x1920 and on a 4320x7680
          output frame, with the bytes it must move (12 read + 3 written per pixel) over the data sheet's 3.35 TB/s as the floor.
  host    the drop-in's per-frame image work before and after rv_eval_images, as seconds per frame over --frames frames on a
          pool of REFVSR_EVAL_WRITERS threads (so one frame's encoding overlaps the next), for input, output and ground truth
          written as png and jpg (6 writes):
            before  three float32 copies into pinned memory, then cv2.cvtColor(x * 255, RGB2BGR) and cv2.imwrite per write
            after   one eval_images call, one copy of its uint8 bytes into pinned memory, cv2.imwrite of the uint8 images
          at 270x480 -> 1080x1920 (x4) and 1080x1920 -> 4320x7680 (HD -> 8K, ground truth 1080x1920).
  loop    run.py --eval_mode qual_quan on synthetic trees with the reference's loop (REFVSR_DROPIN_EVAL=0) and with the drop-in,
          both on the engine's network, so the difference is the loop: RefVSR_MFID at 270x480 -> 1080x1920 (bf16), and
          RefVSR_small_MFID_8K with --qualitative_only at 1080x1920 -> 4320x7680.  Wall seconds between consecutive per-frame
          lines, median over the frames after each video's first, and whether every png / jpg is byte-identical."""
import argparse
import json
import os
import re
import shutil
import statistics
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import cv2                                                            # noqa: E402
import torch                                                          # noqa: E402

import test_dropin_runpy as R                                         # noqa: E402
from refvsr_b200.lib import CudaOps                                   # noqa: E402

HBM_BPS = 3.35e12


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else 'unknown'


def bench_kernel(ops, h, w, calls):
    out = torch.rand(1, 3, h, w, device='cuda')
    for _ in range(5):
        ops.eval_images([out])
    times = []
    for _ in range(calls):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ops.eval_images([out])
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    t = statistics.median(times)
    nbytes = 15 * h * w
    return dict(kernel_us=round(t * 1e6, 1), calls=calls, bytes_moved=nbytes, hbm_floor_us=round(nbytes / HBM_BPS * 1e6, 1),
                hbm_share=round(nbytes / HBM_BPS / t, 3), achieved_tb_s=round(nbytes / t / 1e12, 2))


def _write(job):
    ev, arrays, paths = job
    ev.synchronize()
    for arr, ps in zip(arrays, paths):
        img = arr if arr.dtype.name == 'uint8' else cv2.cvtColor(arr * 255, cv2.COLOR_RGB2BGR)
        for p in ps:
            cv2.imwrite(p, img)


def bench_host(ops, shapes, frames, tmp):
    """seconds per frame for the before / after image work of frames of `shapes` (input, output, gt), 6 writes each"""
    srcs = [torch.rand(1, 3, h, w, device='cuda') for h, w in shapes]
    paths = [[os.path.join(tmp, f'{name}.{fmt}') for fmt in ('png', 'jpg')] for name in ('input', 'output', 'gt')]
    workers = int(os.environ.get('REFVSR_EVAL_WRITERS', '4'))
    res = {}
    for arm in ('before', 'after'):
        pool = ThreadPoolExecutor(max_workers=workers)
        if arm == 'before':
            ring = [[torch.empty(h, w, 3).pin_memory() for h, w in shapes] for _ in range(3)]
        else:
            ring = [torch.empty(sum(3 * h * w for h, w in shapes), dtype=torch.uint8).pin_memory() for _ in range(3)]
        pending = []
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for k in range(frames):
            if arm == 'before':
                for dst, src in zip(ring[k % 3], srcs):
                    dst.copy_(src[0].permute(1, 2, 0), non_blocking=True)
                arrays = [b.numpy() for b in ring[k % 3]]
            else:
                ring[k % 3].copy_(ops.eval_images(srcs), non_blocking=True)
                buf, off, arrays = ring[k % 3].numpy(), 0, []
                for h, w in shapes:
                    arrays.append(buf[off:off + 3 * h * w].reshape(h, w, 3))
                    off += 3 * h * w
            ev = torch.cuda.Event()
            ev.record()
            pending.append(pool.submit(_write, (ev, arrays, paths)))
            while len(pending) > 2:
                pending.pop(0).result()
        for f in pending:
            f.result()
        res[arm + '_s_per_frame'] = round((time.perf_counter() - t0) / frames, 4)
        pool.shutdown()
    res.update(frames=frames, writers=workers, shapes=shapes)
    return res


def run_loop(ref, tmp, tag, config, env_extra, frame_num, extra=()):
    out = os.path.join(tmp, 'out_' + tag)
    pp = [R.ENV_DIR, os.path.join(ROOT, 'refvsr_b200', 'dropin'), ROOT, R.SHIMS]
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(pp), REFVSR_TEST_ENV='1', PYTHONDONTWRITEBYTECODE='1', PYTHONUNBUFFERED='1',
               **env_extra)
    cmd = [sys.executable, '-B', 'run.py', '--mode', 'qq_' + tag, '--project', os.path.join(tmp, 'logs_' + tag), '--config',
           config, '--data', 'RealMCVSR', '--ckpt_abs_name', os.path.join(tmp, 'ckpt.pytorch'), '--data_offset',
           os.path.join(tmp, 'data'), '--output_offset', out, '--frame_num', str(frame_num)] + list(extra)
    t_start = time.time()
    p = subprocess.Popen(cmd, cwd=ref, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    stamps, log = [], []
    for line in p.stdout:
        log.append(line)
        m = re.match(r'\[EVAL [^\]]*\]\[\d+/\d+\]\[(\d+)/\d+\]', line)
        if m:
            stamps.append((int(m.group(1)), time.time()))
    rc = p.wait()
    assert rc == 0, ''.join(log[-40:])
    gaps = [t - stamps[i - 1][1] for i, (f, t) in enumerate(stamps) if i > 0 and f > 1]
    lines = [re.sub(r'\(\d+\.\d+sec\)', '(#sec)', x).replace('qq_' + tag, 'MODE') for x in log
             if x.startswith(('[EVAL', '[MEAN', '[TOTAL'))]
    return dict(frames=len(stamps), wall_s=round(time.time() - t_start, 1), frame_s=round(statistics.median(gaps), 4)), out, lines


def same_images(a, b, tags):
    def files(root, tag):
        return {re.sub(r'/\d{4}_\d{2}_\d{2}_\d{4}/', '/DATE/', os.path.relpath(os.path.join(d, f), root)).replace('qq_' + tag, 'MODE'):
                os.path.join(d, f) for d, _, fs in os.walk(root) for f in fs if f.endswith(('.png', '.jpg'))}
    fa, fb = files(a, tags[0]), files(b, tags[1])
    if set(fa) != set(fb):
        return False, len(fa), len(fb)
    return all(open(fa[k], 'rb').read() == open(fb[k], 'rb').read() for k in fa), len(fa), len(fb)


def bench_loop(ref, name, config, lr_hw, frame_num, videos, frames, extra, env):
    tmp = tempfile.mkdtemp(prefix='qqbench_')
    R.make_tree(os.path.join(tmp, 'data'), *lr_hw, videos=videos, frames=frames)
    R.make_ckpt(os.path.join(tmp, 'ckpt.pytorch'), config)
    res, outs, lines = {}, {}, {}
    for tag, e in (('reference_loop', {'REFVSR_DROPIN_EVAL': '0'}), ('dropin_loop', {})):
        res[tag], outs[tag], lines[tag] = run_loop(ref, tmp, tag, config, dict(env, **e), frame_num, extra)
        print(name, tag, res[tag], flush=True)
    res['lines_identical'] = lines['reference_loop'] == lines['dropin_loop']
    res['images_identical'], res['images_reference'], res['images_dropin'] = same_images(
        outs['reference_loop'], outs['dropin_loop'], ('reference_loop', 'dropin_loop'))
    res['speedup'] = round(res['reference_loop']['frame_s'] / res['dropin_loop']['frame_s'], 2)
    shutil.rmtree(tmp, ignore_errors=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--calls', type=int, default=50, help='eval_images calls timed (median)')
    ap.add_argument('--frames', type=int, default=20, help='frames of the host measurement at 1080p (a quarter of that at 8K)')
    ap.add_argument('--loop-frames', type=int, default=10, help='frames per synthetic video of the x4 loop')
    ap.add_argument('--loop-frames-8k', type=int, default=4, help='frames per synthetic video of the HD -> 8K loop')
    ap.add_argument('--videos', type=int, default=2)
    ap.add_argument('--no-loop', action='store_true', help='skip the run.py loop measurements')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'qual_quan_bench measures on a CUDA device'
    ops = CudaOps()
    res = dict(card=card(), kernel_1080x1920=bench_kernel(ops, 1080, 1920, args.calls),
               kernel_4320x7680=bench_kernel(ops, 4320, 7680, args.calls))
    print(json.dumps(res), flush=True)
    tmp = tempfile.mkdtemp(prefix='qqbench_')
    res['host_x4_270x480_to_1080x1920'] = bench_host(ops, [(270, 480), (1080, 1920), (1080, 1920)], args.frames, tmp)
    res['host_hd_to_8k_1080x1920_to_4320x7680'] = bench_host(ops, [(1080, 1920), (4320, 7680), (1080, 1920)],
                                                             max(args.frames // 4, 3), tmp)
    shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res), flush=True)
    if not args.no_loop:
        ref = R._ref_root()
        assert ref, 'stage the reference first: python oracle/build_ref.py'
        res['loop_x4_mfid_270x480'] = bench_loop(ref, 'x4', 'config_RefVSR_MFID', (270, 480), 7, args.videos, args.loop_frames, (),
                                                 {'REFVSR_TEST_PRECISION': 'bf16'})
        print(json.dumps(res), flush=True)
        # flag_HD_in reads the HR tree (4x the LR size) as its input: 270x480 LR -> 1080x1920 input -> 4320x7680 output
        res['loop_small_mfid_8k_1080x1920'] = bench_loop(ref, '8k', 'config_RefVSR_small_MFID_8K', (270, 480), 3, args.videos,
                                                         args.loop_frames_8k, ('--qualitative_only',), {})
    res['card_after'] = card()
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
