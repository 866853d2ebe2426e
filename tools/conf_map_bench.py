"""Cost of the confidence-map evaluation mode (`run.py --eval_mode conf`, evaluation/eval_quan_conf_map.py) per frame at
270x480 -> 1080x1920; prints JSON lines.

  frame  the reference's per-frame work after the model (eval_quan_conf_map.py:64-170: the four maps normalised on the device,
         copied back and coloured by `inferno` - matplotlib's, or the tests' stand-in where it is absent - the input and the
         output copied back, 12 cv2.imwrite calls) against the drop-in's: one CudaOps.conf_map_images call (CUDA events), the
         call plus the copy into pinned memory (host clock), and the whole frame with the 12 writes on a pool of
         REFVSR_EVAL_WRITERS threads, as the drop-in queues them (seconds per frame over --frames frames, so the encoding of
         one frame overlaps the next).
  loop   run.py --eval_mode conf on a synthetic 270x480 -> 1080x1920 tree (RefVSR_MFID, bf16 engine, --videos x --frames), with
         the reference's loop (REFVSR_DROPIN_EVAL=0) and with the drop-in: wall seconds between consecutive per-frame lines,
         median over the frames after each video's first.  Both arms run the engine's network, so the difference is the loop."""
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

import conf_map_oracle as CO                                          # noqa: E402
import test_conf_map_eval as T                                        # noqa: E402
from refvsr_b200.colormap import inferno_lut                          # noqa: E402
from refvsr_b200.lib import CudaOps                                   # noqa: E402

NAMES = ('conf_map_norm', 'conf_map_prop_norm', 'conf_map_prop_b_norm', 'conf_map_prop_f_norm', 'input', 'output')


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else 'unknown'


def reference_frame(cmap, maps, inp, out, root):
    """the reference's post-model steps of one frame (eval_quan_conf_map.py:64-170), writing its 12 files under root"""
    arrays = []
    for m in maps:
        m = m - m.min()
        m = m / m.max()
        rgb = cmap(m.cpu().numpy()[0].transpose(1, 2, 0)[:, :, 0])[:, :, :3]
        arrays.append(torch.Tensor(rgb)[None, :].permute(0, 3, 1, 2).cpu().numpy()[0].transpose(1, 2, 0))
    arrays += [inp.cpu().numpy()[0].transpose(1, 2, 0), out.cpu().numpy()[0].transpose(1, 2, 0)]
    for fmt in ('png', 'jpg'):
        for name, a in zip(NAMES, arrays):
            cv2.imwrite(os.path.join(root, f'{name}.{fmt}'), cv2.cvtColor(a * 255, cv2.COLOR_RGB2BGR))


def bench_frame(calls, host_calls, frames):
    ops = CudaOps()
    h, w = 270, 480
    maps = [m.cuda() for m in T.conf_maps(h, w, seed=1)]
    inp, out = T.frame(h, w, 2).clamp(0, 1).cuda(), T.frame(4 * h, 4 * w, 3).clamp(0, 1).cuda()
    lut = inferno_lut('cuda')
    tmp = tempfile.mkdtemp(prefix='confbench_')
    cmap = CO.colormap()
    host = []
    for _ in range(host_calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        reference_frame(cmap, maps, inp, out, tmp)
        host.append(time.perf_counter() - t0)
    for _ in range(5):
        ops.conf_map_images(maps, inp, out, lut, True)
    kern = []
    for _ in range(calls):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        packed = ops.conf_map_images(maps, inp, out, lut, True)
        e1.record()
        e1.synchronize()
        kern.append(e0.elapsed_time(e1) / 1e3)
    pinned = torch.empty(packed.numel(), dtype=torch.uint8).pin_memory()
    copy = []
    for _ in range(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pinned.copy_(ops.conf_map_images(maps, inp, out, lut, True), non_blocking=True)
        torch.cuda.current_stream().synchronize()
        copy.append(time.perf_counter() - t0)
    exact = bool((pinned.numpy() == CO.packed(CO.reference_images(maps, inp, out, True, cmap))).all())
    # whole frames as the drop-in runs them: the call, the copy, then the writes on the pool while the next frame goes on
    def write(ev, buf, paths):
        ev.synchronize()
        off = 0
        for (hh, ww), ps in zip([(h, w)] * 5 + [(4 * h, 4 * w)], paths):
            img = buf[off:off + 3 * hh * ww].reshape(hh, ww, 3)
            off += 3 * hh * ww
            for p in ps:
                cv2.imwrite(p, img)

    pool = ThreadPoolExecutor(max_workers=int(os.environ.get('REFVSR_EVAL_WRITERS', '4')))
    ring = [torch.empty(packed.numel(), dtype=torch.uint8).pin_memory() for _ in range(3)]
    pending = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(frames):
        ring[k % 3].copy_(ops.conf_map_images(maps, inp, out, lut, True), non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        paths = [[os.path.join(tmp, f'dropin_{name}.{fmt}') for fmt in ('png', 'jpg')] for name in NAMES]
        pending.append(pool.submit(write, ev, ring[k % 3].numpy(), paths))
        while len(pending) > 2:
            pending.pop(0).result()
    for f in pending:
        f.result()
    frame_s = (time.perf_counter() - t0) / frames
    pool.shutdown()
    shutil.rmtree(tmp, ignore_errors=True)
    return dict(reference_host_s=round(statistics.median(host), 4), reference_calls=host_calls,
                kernel_us=round(statistics.median(kern) * 1e6, 2), kernel_calls=calls,
                kernel_and_copy_us=round(statistics.median(copy) * 1e6, 1), dropin_frame_with_writes_s=round(frame_s, 4),
                dropin_frames=frames, writers=int(os.environ.get('REFVSR_EVAL_WRITERS', '4')), bytes_per_frame=packed.numel(),
                bytes_equal_reference_steps=exact, hbm_floor_us=round((4 * 4 * h * w + 4 * 3 * 17 * h * w + packed.numel()) / 3.35e12 * 1e6, 1),
                colormap='matplotlib' if CO.have_matplotlib() else 'tests/conf_map_env stand-in')


def run_loop(ref, tmp, tag, env_extra, frame_num=7):
    out = os.path.join(tmp, 'out_' + tag)
    standin = [CO.ENV] if (env_extra.get('REFVSR_DROPIN_EVAL') == '0' and not CO.have_matplotlib()) else []
    pp = [T.ENV_DIR] + standin + [os.path.join(ROOT, 'refvsr_b200', 'dropin'), ROOT, T.SHIMS]
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(pp), REFVSR_TEST_ENV='1', PYTHONDONTWRITEBYTECODE='1', PYTHONUNBUFFERED='1',
               REFVSR_TEST_PRECISION='bf16', **env_extra)
    cmd = [sys.executable, '-B', 'run.py', '--mode', 'conf_' + tag, '--project', os.path.join(tmp, 'logs_' + tag), '--config',
           'config_RefVSR_MFID', '--data', 'RealMCVSR', '--ckpt_abs_name', os.path.join(tmp, 'ckpt.pytorch'), '--data_offset',
           os.path.join(tmp, 'data'), '--output_offset', out, '--frame_num', str(frame_num), '--eval_mode', 'conf']
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
    return dict(frames=len(stamps), wall_s=round(time.time() - t_start, 1), frame_s=round(statistics.median(gaps), 4),
                printed_evaluation_s=round(statistics.median(printed), 4)), out


def same_images(a, b):
    def files(root):
        return {re.sub(r'/\d{4}_\d{2}_\d{2}_\d{4}/', '/DATE/', os.path.relpath(os.path.join(d, f), root)).split('/', 1)[-1]:
                os.path.join(d, f) for d, _, fs in os.walk(root) for f in fs if f.endswith(('.png', '.jpg'))}
    fa, fb = files(a), files(b)
    fa = {re.sub(r'conf_(reference|dropin)_loop', 'MODE', k): v for k, v in fa.items()}
    fb = {re.sub(r'conf_(reference|dropin)_loop', 'MODE', k): v for k, v in fb.items()}
    if set(fa) != set(fb):
        return False, len(fa), len(fb)
    return all(open(fa[k], 'rb').read() == open(fb[k], 'rb').read() for k in fa), len(fa), len(fb)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--calls', type=int, default=50, help='conf_map_images calls timed (median)')
    ap.add_argument('--host-calls', type=int, default=5, help='reference frames timed (median)')
    ap.add_argument('--frames', type=int, default=20, help='drop-in frames with writes, and frames per synthetic video')
    ap.add_argument('--videos', type=int, default=2)
    ap.add_argument('--no-loop', action='store_true', help='skip the run.py loop measurement')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'conf_map_bench measures on a CUDA device'
    res = dict(card=card(), frame_270x480_to_1080x1920=bench_frame(args.calls, args.host_calls, args.frames))
    print(json.dumps(res), flush=True)
    if not args.no_loop:
        ref = T._ref_root()
        assert ref, 'stage the reference first: python oracle/build_ref.py'
        tmp = tempfile.mkdtemp(prefix='confbench_')
        T.make_tree(os.path.join(tmp, 'data'), 270, 480, videos=args.videos, frames=args.frames)
        T.make_ckpt(os.path.join(tmp, 'ckpt.pytorch'), 'config_RefVSR_MFID')
        outs = {}
        for tag, env in (('reference_loop', {'REFVSR_DROPIN_EVAL': '0'}), ('dropin_loop', {})):
            res[tag], outs[tag] = run_loop(ref, tmp, tag, env)
            print(tag, res[tag], flush=True)
        res['loop_images_identical'], res['loop_images_reference'], res['loop_images_dropin'] = same_images(
            outs['reference_loop'], outs['dropin_loop'])
        res['loop_speedup'] = round(res['reference_loop']['frame_s'] / res['dropin_loop']['frame_s'], 2)
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
