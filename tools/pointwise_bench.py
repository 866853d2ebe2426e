"""Graph-timed launches of the HBM-bound kernels at the BASELINE shapes (same method as bench.kernel_rooflines: buffers
rotated through > L2)."""
import os
import sys
import torch
sys.path.insert(0, os.path.join(os.path.dirname(__file__), '..'))
from refvsr_b200.lib import CudaOps   # noqa: E402

H, W, C = 270, 480, int(os.environ.get('PW_C', 48))
dt = torch.bfloat16
e = 2
PEAK = 3350.0                     # H100 SXM data-sheet HBM3 bandwidth, GB/s


def timeit(fn, iters=30, warm=5):
    for i in range(warm):
        fn(i)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for i in range(iters):
            fn(i)
    graph.replay()
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) / iters * 1e-3)
    return best


def main():
    ops = CudaOps()
    dev = 'cuda'
    n2 = max(2, int(160e6 // (4 * H * W * C * e)) + 1)
    flow = torch.randn((H, W, 2), device=dev)
    fs = [torch.randn((2 * H, 2 * W, C), device=dev).to(dt) for _ in range(n2)]
    fo = [torch.empty((2 * H, 2 * W, C), device=dev, dtype=dt) for _ in range(n2)]
    lf = [torch.randn((H, W, C), device=dev).to(dt) for _ in range(n2)]
    lo = [torch.empty((H, W, C), device=dev, dtype=dt) for _ in range(n2)]
    cf, co = torch.rand((H, W), device=dev), torch.empty((H, W), device=dev)
    t = timeit(lambda i: ops.warp3(lf[i % n2], fs[i % n2], cf, flow, lo[i % n2], fo[i % n2], co))
    b = 2.0 * 5 * H * W * C * e + 2.0 * 4 * H * W + 8.0 * H * W
    print(f'warp3          {t * 1e6:7.2f} us  {b / t / 1e9:7.0f} GB/s  frac {b / t / 1e9 / PEAK:.3f}')
    aff = torch.rand((H, W, 3), device=dev) * 0.4 + 0.8
    t = timeit(lambda i: ops.aligned_sample(fs[i % n2], aff, 2, fo[(i + 1) % n2]))
    b = 12.0 * H * W + 2.0 * 4 * C * H * W * e
    print(f'aligned_sample {t * 1e6:7.2f} us  {b / t / 1e9:7.0f} GB/s  frac {b / t / 1e9 / PEAK:.3f}')
    t = timeit(lambda i: ops.warp(fs[i % n2], flow, fo[i % n2], flow_up2=True))
    b = 2.0 * 4 * H * W * C * e + 8.0 * H * W
    print(f'warp_up        {t * 1e6:7.2f} us  {b / t / 1e9:7.0f} GB/s  frac {b / t / 1e9 / PEAK:.3f}')


if __name__ == '__main__':
    main()
