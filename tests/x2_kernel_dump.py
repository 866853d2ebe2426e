"""Helper of tests/test_gpu_x2.py, run in a subprocess: REFVSR_NO_FAST_POINTWISE is read once per process, so the fast and the
generic pointwise kernels can only be compared across two processes.

    python tests/x2_kernel_dump.py OUT.npz

Runs the three x2 hot-path operators (rv_gather_blocks with 4x4 blocks, rv_aligned_sample with ks 4, rv_reconstruct at scale 2) on
seeded inputs at x2 and 8K shapes and saves every output together with the names of the kernels that ran (torch.profiler).  Whole
model windows are not compared this way: the switch also turns off older fast paths that are close to, not bit-identical with,
their generic kernels."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]

# (name, cells (hq, wq), value (Hv, Wv)): aa2 of the x2 models at LR 136x240, aa1 of the 8K models at LR 1080x1920
SHAPES = [('x2', (68, 120), (136, 240)), ('8k', (270, 480), (540, 960))]
DTYPES = {'bf16': torch.bfloat16, 'fp16': torch.float16, 'fp32': torch.float32}


def inputs(cells, value_hw, C, dt, seed):
    g = torch.Generator().manual_seed(seed)
    hq, wq = cells
    Hv, Wv = value_hw
    value = torch.rand(Hv, Wv, C, generator=g).to(dt)
    idx = torch.randint(0, (Hv // 4) * (Wv // 4), (hq * wq,), generator=g, dtype=torch.int32)
    aff = torch.stack([1 + 0.6 * (torch.rand(hq, wq, generator=g) - 0.5), 1 + 0.6 * (torch.rand(hq, wq, generator=g) - 0.5),
                       1 + 0.8 * (torch.rand(hq, wq, generator=g) - 0.5)], -1).contiguous()
    x = torch.rand(4 * hq, 4 * wq, C, generator=g).to(dt)
    return value, idx, aff, x


def run_ops(ops, out):
    dev = 'cuda'
    for sname, cells, value_hw in SHAPES:
        hq, wq = cells
        for C, dname in ((48, 'bf16'), (8, 'bf16'), (24, 'bf16'), (48, 'fp16'), (48, 'fp32'), (8, 'fp32'), (24, 'fp32')):
            if sname == '8k' and dname == 'fp32' and C != 48:
                continue
            value, idx, aff, x = (t.to(dev) for t in inputs(cells, value_hw, C, DTYPES[dname], seed=C))
            g = torch.empty(4 * hq, 4 * wq, C, dtype=value.dtype, device=dev)
            ops.gather_blocks(value, idx, hq, wq, 4, g)
            out[f'gather/{sname}/{dname}/{C}'] = g
            if C != 8:
                a = torch.empty_like(x)
                ops.aligned_sample(x, aff, 4, a)
                out[f'aligned/{sname}/{dname}/{C}'] = a
    for h, w in ((540, 960), (136, 240), (37, 53)):                 # the eval size, the mid-size case, an odd size
        g = torch.Generator().manual_seed(h)
        last = (0.3 * (torch.rand(2 * h, 2 * w, 4, generator=g) - 0.5)).to(dev)
        lr = torch.rand(3, h, w, generator=g).to(dev)
        for clamp in (True, False):
            o = torch.empty(3, 2 * h, 2 * w, device=dev)
            ops.reconstruct(last, lr, 2, clamp, o)
            out[f'reconstruct/{h}x{w}/{int(clamp)}'] = o


def main(path):
    from refvsr_b200.lib import CudaOps
    ops = CudaOps()
    out = {}
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_ops(ops, out)
        torch.cuda.synchronize()
    names = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
    arrs = {k: (v.view(torch.int16) if v.dtype in (torch.bfloat16, torch.float16) else v).cpu().numpy() for k, v in out.items()}
    np.savez(path, kernels=np.array(names), **arrs)


if __name__ == '__main__':
    main(sys.argv[1])
