"""Cost of the FOV evaluation mode (`run.py --eval_mode FOV`, evaluation/eval_quan_FOV.py) per 1080p frame; prints one JSON line.

  metrics  the reference's per-frame metric work on the host (eval_quan_FOV.py:146-189: both frames copied to the host, the masks,
           psnr / ssim / psnr_masked / ssim_masked with the tests' skimage stand-in, tests/runpy_env) against one
           CudaOps.region_metrics call (CUDA events, median of --calls) and the drop-in's whole per-frame scoring
           (refvsr_b200.fov.score_frame: the launch, the 112-byte copy back and the host arithmetic; host clock).
  loop     run.py --eval_mode FOV on a synthetic 270x480 -> 1080x1920 tree (RefVSR_MFID, bf16 engine, --videos x --frames), with
           the reference's loop (REFVSR_DROPIN_EVAL=0) and with the drop-in: wall seconds between consecutive per-frame lines,
           median over the frames after each video's first.  Both arms run the engine's network, so the difference is the loop."""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import torch                                                          # noqa: E402

import test_fov_eval as T                                             # noqa: E402
from refvsr_b200.fov import score_frame                               # noqa: E402
from refvsr_b200.lib import CudaOps                                   # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else 'unknown'


def bench_metrics(calls, host_calls):
    ops = CudaOps()
    M = T.load_reference_metrics()
    out, gt = (t.cuda() for t in T.frame_pair(1080, 1920, seed=11))
    host = []
    for _ in range(host_calls):
        t0 = time.perf_counter()
        T.reference_scores(M, out.cpu().numpy()[0].transpose(1, 2, 0), gt.cpu().numpy()[0].transpose(1, 2, 0))
        host.append(time.perf_counter() - t0)
    boxes = T.fov_boxes(1080, 1920)
    for _ in range(5):
        ops.region_metrics(out, gt, boxes)
    # the kernel pair alone: the launches, timed by events, without the binding's synchronising copy
    import ctypes as C
    from refvsr_b200.lib import _ptr
    ws, sums = ops._region_ws
    arr = (C.c_int32 * 28)(*[v for b in boxes for v in b])
    kern = []
    for _ in range(calls):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = ops.lib.rv_region_metrics(_ptr(out), _ptr(gt), 1080, 1920, arr, 7, _ptr(ws), _ptr(sums), ops._stream())
        e1.record()
        assert rc == 0, ops.lib.rv_last_error()
        e1.synchronize()
        kern.append(e0.elapsed_time(e1) / 1e3)
    frame = []
    for _ in range(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        score_frame(ops, out, gt)
        frame.append(time.perf_counter() - t0)
    ours, ref = score_frame(ops, out, gt), T.reference_scores(M, T.hwc(out.cpu()), T.hwc(gt.cpu()))
    worst = max(abs(float(a) - float(b)) for k in ours for a, b in zip(ours[k], ref[k]))
    return dict(host_reference_s=statistics.median(host), host_reference_calls=host_calls,
                region_metrics_kernel_us=round(statistics.median(kern) * 1e6, 2), kernel_calls=calls,
                dropin_score_frame_us=round(statistics.median(frame) * 1e6, 1), max_abs_diff_vs_reference=worst,
                hbm_floor_us=round(2 * 3 * 1080 * 1920 * 4 / 3.35e12 * 1e6, 1))


def run_loop(ref, tmp, tag, env_extra, frame_num=7):
    out = os.path.join(tmp, 'out_' + tag)
    pp = [T.ENV_DIR, os.path.join(ROOT, 'refvsr_b200', 'dropin'), ROOT, T.SHIMS]
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(pp), REFVSR_TEST_ENV='1', PYTHONDONTWRITEBYTECODE='1', PYTHONUNBUFFERED='1',
               REFVSR_TEST_PRECISION='bf16', **env_extra)
    cmd = [sys.executable, '-B', 'run.py', '--mode', 'fov_' + tag, '--project', os.path.join(tmp, 'logs_' + tag), '--config',
           'config_RefVSR_MFID', '--data', 'RealMCVSR', '--ckpt_abs_name', os.path.join(tmp, 'ckpt.pytorch'), '--data_offset',
           os.path.join(tmp, 'data'), '--output_offset', out, '--frame_num', str(frame_num), '--eval_mode', 'FOV']
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
    printed = [float(x) for x in re.findall(r'\[EVAL [^\n]*\(([\d.]+)sec\)', ''.join(log))]
    return dict(frames=len(stamps), wall_s=round(time.time() - t_start, 1), frame_s=statistics.median(gaps),
                printed_evaluation_s=statistics.median(printed)), ''.join(log)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--calls', type=int, default=50, help='region_metrics launches / score_frame calls timed (median)')
    ap.add_argument('--host-calls', type=int, default=3, help='host reference frames timed (median)')
    ap.add_argument('--videos', type=int, default=2)
    ap.add_argument('--frames', type=int, default=10)
    ap.add_argument('--no-loop', action='store_true', help='skip the run.py loop measurement')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'fov_bench measures on a CUDA device'
    res = dict(card=card(), metrics_1080p=bench_metrics(args.calls, args.host_calls))
    print(json.dumps(res), flush=True)
    if not args.no_loop:
        ref = T._ref_root()
        assert ref, 'stage the reference first: python oracle/build_ref.py'
        tmp = tempfile.mkdtemp(prefix='fovbench_')
        T.make_tree(os.path.join(tmp, 'data'), 270, 480, videos=args.videos, frames=args.frames)
        T.make_ckpt(os.path.join(tmp, 'ckpt.pytorch'), 'config_RefVSR_MFID')
        logs = {}
        for tag, env in (('reference_loop', {'REFVSR_DROPIN_EVAL': '0'}), ('dropin_loop', {})):
            res[tag], logs[tag] = run_loop(ref, tmp, tag, env)
            print(tag, res[tag], flush=True)
        a, b = T.printed_numbers(logs['reference_loop']), T.printed_numbers(logs['dropin_loop'])
        res['loop_max_abs_diff'] = max(abs(x - y) for (_, x), (_, y) in zip(a, b)) if len(a) == len(b) else None
        res['loop_speedup'] = res['reference_loop']['frame_s'] / res['dropin_loop']['frame_s']
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
