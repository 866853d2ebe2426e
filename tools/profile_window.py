"""Kernel-time table of one steady RefVSR_MFID 270x480 window: eager launches (no CUDA graph), 1 first + 3 steady
windows, torch.profiler (CUDA activities) around the last one only.  Usage: python tools/profile_window.py [OUT_DIR]
prints the table and, with OUT_DIR, also writes it to OUT_DIR/profile_window.txt."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import profile, ProfilerActivity
import bench
cfg, net = bench.make_model('mfid', None, torch.device('cuda', 0), graphs=False)
from refvsr_b200.synth import make_clip_range
lrs, refs = make_clip_range(0, 8, bench.H, bench.W, 1, seed=1234)
lrs, refs = lrs.cuda(), refs.cuda()
NW = 4
for k in range(NW):
    ids = torch.tensor(bench.window_indices(k, 8), device='cuda')
    a, b = lrs.index_select(0, ids).unsqueeze(0), refs.index_select(0, ids).unsqueeze(0)
    torch.cuda.synchronize()
    if k < NW - 1:
        out = net(a, b, k == 0, False, False)
        torch.cuda.synchronize()
        continue
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = net(a, b, k == 0, False, False)
        torch.cuda.synchronize()
table = prof.key_averages().table(sort_by='cuda_time_total', row_limit=40, max_name_column_width=90)
tot = sum(e.self_device_time_total for e in prof.key_averages())
print(table)
print(f'device time of the window, all kernels: {tot / 1e3:.2f} ms')
if len(sys.argv) > 1:
    os.makedirs(sys.argv[1], exist_ok=True)
    with open(os.path.join(sys.argv[1], 'profile_window.txt'), 'w') as f:
        f.write(table + f'\ndevice time of the window, all kernels: {tot / 1e3:.2f} ms\n')
print('done', tuple(out['result'].shape))
