"""BASELINE configs[4]: config_RefVSR_MFID_8K at its real size - LR (and Ref) 1080x1920 -> 4320x7680, T = 7, bf16 - on ONE GPU.
Reports ms / window (first, steady, CUDA-graph replays), peak device memory against DESIGN.md's plan, and - at 540x960 LR, where
the fp32 CUDA-core yardstick path is still affordable - PSNR of the bf16 tensor-core path against the fp32 path (which is pinned
to the reference by the flag_HD_in goldens at fixture size).  Writes gpurun_out/r02_8k.json."""
import faulthandler, json, os, signal, sys, time
faulthandler.register(signal.SIGUSR1, all_threads=True)      # `timeout -s USR1`: where is the host when a run is too slow?
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from refvsr_b200 import SRNet, get_config
from refvsr_b200.modules import seeded_test_weights
from refvsr_b200.synth import make_clip, sliding_windows

dev = torch.device('cuda', 0)
out = {}
os.makedirs('gpurun_out', exist_ok=True)


def run(h, w, prec, nwin, frames=None):
    cfg = get_config('config_RefVSR_MFID_8K', device='cuda', b200_precision=prec)
    net = SRNet(cfg).eval()
    seeded_test_weights(net, seed=1234)
    net = net.to(dev)
    T = cfg.frame_num
    lrs, refs = frames
    torch.cuda.reset_peak_memory_stats(dev)
    res, times = [], []
    for k, wl, wr, first in sliding_windows(lrs, refs, T):
        if k >= nwin:
            break
        a, b = wl.to(dev), wr.to(dev)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        o = net(a, b, first, False, False)['result']
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
        print(f'  [{prec} {h}x{w}] window {k}: {times[-1]:.1f} ms, peak {torch.cuda.max_memory_allocated(dev) / 2 ** 30:.1f} GiB', flush=True)
        res.append(o[0].float().cpu())
        del a, b, o
    peak = torch.cuda.max_memory_allocated(dev) / 2 ** 30
    nbuf = sum(t.numel() * t.element_size() for t in net.Network._bufs.values()) / 2 ** 30
    del net
    torch.cuda.empty_cache()
    return res, times, peak, nbuf


t0 = time.time()
H, W = (int(os.environ.get('R8K_H', 1080)), int(os.environ.get('R8K_W', 1920)))
frames = make_clip(10, H, W, 1, seed=1234)
print(f'clip {H}x{W} built in {time.time() - t0:.1f} s', flush=True)
NWIN = int(os.environ.get('R8K_NWIN', 10))
res, times, peak, nbuf = run(H, W, 'bf16', NWIN, frames)
# windows 0 (first), 1-2 (steady, eager capture), 3+ graph replays? every (phase, kind) key is captured on first use: with T = 7
# the ring phase repeats every 7 windows, so within 10 windows only windows 8, 9 replay graphs (phases 1, 2 seen at windows 1, 2)
out['full'] = dict(lr=[H, W], out=[4 * H, 4 * W], precision='bf16', ms_per_window=times, peak_mem_gib=peak, engine_buffers_gib=nbuf,
                   first_window_ms=times[0], steady_eager_ms=(sorted(times[1:8])[len(times[1:8]) // 2] if len(times) > 1 else None), steady_graph_ms=min(times[8:]) if len(times) > 8 else None,
                   out_mean=[float(r.mean()) for r in res[:3]], finite=all(bool(torch.isfinite(r).all()) for r in res))
print(json.dumps(out['full']), flush=True)
del res
json.dump(out, open('gpurun_out/r02_8k.json', 'w'), indent=1)
if os.environ.get('R8K_NO_PARITY'):
    sys.exit(0)
if os.environ.get('R8K_ONLY_PARITY') and os.path.isfile('gpurun_out/r02_8k_full.json'):
    out = json.load(open('gpurun_out/r02_8k_full.json'))
# parity of the 16-bit tensor-core path vs the fp32 yardstick path at half size
h2, w2 = int(os.environ.get('R8K_PH', 544)), int(os.environ.get('R8K_PW', 960))      # (Ref sizes must be multiples of 8)
frames2 = make_clip(4, h2, w2, 1, seed=99)
r16, t16, _, _ = run(h2, w2, 'bf16', 2, frames2)
r32, t32, p32, _ = run(h2, w2, 'fp32', 2, frames2)
ps = []
for a, b in zip(r16, r32):
    mse = float(((a.double() - b.double()) ** 2).mean())
    ps.append(10 * __import__('math').log10(1.0 / max(mse, 1e-20)))
out['half_parity'] = dict(lr=[h2, w2], psnr_bf16_vs_fp32_path_db=ps, max_abs=[float((a - b).abs().max()) for a, b in zip(r16, r32)],
                          ms_bf16=t16, ms_fp32=t32, peak_mem_fp32_gib=p32)
print(json.dumps(out['half_parity']), flush=True)
json.dump(out, open('gpurun_out/r02_8k.json', 'w'), indent=1)
