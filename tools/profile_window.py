"""Kernel-time table of one steady RefVSR_MFID 270x480 window: eager launches (no CUDA graph), 1 first + 3 steady
windows, torch.profiler (CUDA activities) around the last one only.

    python tools/profile_window.py [OUT_DIR] [--batch N]

--batch N: N clips per forward() call (one batched window schedule; a different seeded scene per clip); the totals are also
given per clip.  Prints the table, the window's device time and the share of the 3x3 48-channel tensor-core conv (the
compile-time NB 48 kernels, two or three consumers); with OUT_DIR, also writes them to OUT_DIR/profile_window[_nN].txt."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import profile, ProfilerActivity
import bench
args = sys.argv[1:]
nb = 1
if '--batch' in args:
    i = args.index('--batch')
    nb = int(args[i + 1])
    del args[i:i + 2]
cfg, net = bench.make_model('mfid', None, torch.device('cuda', 0), graphs=False)
from refvsr_b200.synth import make_clip_range
clips = [make_clip_range(0, 8, bench.H, bench.W, 1, seed=1234 + i) for i in range(nb)]
lrs, refs = torch.stack([c[0] for c in clips]).cuda(), torch.stack([c[1] for c in clips]).cuda()
NW = 4
for k in range(NW):
    ids = torch.tensor(bench.window_indices(k, 8), device='cuda')
    a, b = lrs.index_select(1, ids), refs.index_select(1, ids)
    torch.cuda.synchronize()
    if k < NW - 1:
        out = net(a, b, k == 0, False, False)
        torch.cuda.synchronize()
        continue
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = net(a, b, k == 0, False, False)
        torch.cuda.synchronize()
ev = prof.key_averages()
table = ev.table(sort_by='cuda_time_total', row_limit=40, max_name_column_width=90)
tot = sum(e.self_device_time_total for e in ev)
conv3 = [e for e in ev if ('conv_tc_kernel' in e.key and ', 1, 48, 3, 3, false>' in e.key) or 'conv_tc3_kernel' in e.key]
c3 = sum(e.self_device_time_total for e in conv3)
c3n = sum(e.count for e in conv3)
summary = (f'batch {nb}: device time of the window, all kernels: {tot / 1e3:.2f} ms ({tot / 1e3 / nb:.2f} ms per clip); '
           f'3x3 48-channel conv: {c3n} launches, {c3 / 1e3:.2f} ms ({c3 / 1e3 / nb:.2f} ms per clip, {100 * c3 / max(tot, 1):.1f} %)')
print(table)
print(summary)
if args:
    os.makedirs(args[0], exist_ok=True)
    with open(os.path.join(args[0], 'profile_window%s.txt' % ('' if nb == 1 else f'_n{nb}')), 'w') as f:
        f.write(table + '\n' + summary + '\n')
print('done', tuple(out['result'].shape), 'batch fallbacks', net.Network.batch_fallbacks)
