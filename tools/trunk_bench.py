"""Where the time of the trunk convs goes, measured the way the window runs them: a chain of 60 conv launches (30 residual blocks,
ping-pong maps that stay L2-resident) inside one CUDA graph, against the isolated launch with L2-cold / L2-warm buffers, plus an
L2-resident copy for scale.  Usage: python tools/trunk_bench.py"""
import os
import sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch                                    # noqa: E402
import refvsr_b200.lib as L                     # noqa: E402
ops = L.CudaOps()
from refvsr_b200 import packing                 # noqa: E402
from refvsr_b200.lib import ACT_RELU, ACT_NONE  # noqa: E402

H, W, C = 270, 480, 48
dt = torch.bfloat16
dev = 'cuda'


def timeit(fn, iters=20, warm=3, reps=3):
    for i in range(warm):
        fn(i)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(iters):
            fn(i)
    g.replay()
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) / iters * 1e3)
    return best


gen = torch.Generator().manual_seed(0)
w = (torch.rand((C, C, 3, 3), generator=gen) - 0.5) * 0.1
layer = packing.pack_conv('t', w, torch.zeros(C), [(C, C)], 1, 1, dt, dev, True)
nrot = int(160e6 // (H * W * C * 2)) + 1
xs = [torch.randn((H, W, C), device=dev).to(dt) for _ in range(nrot)]
ys = [torch.empty((H, W, C), device=dev, dtype=dt) for _ in range(nrot)]
a, t, b = xs[0], xs[1], xs[2]


def trunk(_):
    x, y = a, b
    for _i in range(30):
        ops.conv2d(layer, x, None, t, act_pre=ACT_RELU)
        ops.conv2d(layer, t, None, y, res=x)
        x, y = y, x


def report(tag):
    cold = timeit(lambda i: ops.conv2d(layer, xs[i % nrot], None, ys[i % nrot], res=xs[(i + 1) % nrot], act_pre=ACT_RELU), iters=30)
    warm = timeit(lambda i: ops.conv2d(layer, a, None, b, res=t, act_pre=ACT_RELU), iters=30)
    ch = timeit(trunk, iters=2, warm=1) / 60
    print(f'{tag:34s} cold {cold:6.2f} us   warm {warm:6.2f} us   trunk chain {ch:6.2f} us / conv', flush=True)


report('baseline')
# L2-resident copy for scale (12.4 MB maps): read + write bytes per second through L2
for n in (1, 2, 4):
    src = [torch.randn((n * H, W, C), device=dev).to(dt) for _ in range(2)]
    dst = [torch.empty_like(s) for s in src]
    tc = timeit(lambda i: dst[i % 2].copy_(src[i % 2]), iters=30)
    by = 2.0 * src[0].numel() * 2
    print(f'L2-resident copy {by / 2e6:6.1f} MB maps: {tc:6.2f} us  {by / tc / 1e6:6.2f} TB/s (read + write)')
