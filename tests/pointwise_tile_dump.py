"""Helper of tests/test_pointwise_fp64.py, run in a subprocess: REFVSR_W3_TILE and REFVSR_AS_TILE are read once per process, so each
selectable tile shape of warp3 / aligned_sample runs in its own process.

    REFVSR_W3_TILE=1 python tests/pointwise_tile_dump.py OUT.npz

Runs the cases of test_pointwise_fp64.TILE_CASES on their seeded operands and saves every output together with the names of the
kernels that ran (torch.profiler); the parent checks them against the float64 reference."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]


def main(path):
    from torch.profiler import ProfilerActivity, profile

    from refvsr_b200.lib import CudaOps
    from test_pointwise_fp64 import TILE_CASES, run_guarded, tile_case
    ops = CudaOps()
    out = {}
    with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(len(TILE_CASES)):
            for j, t in enumerate(run_guarded(ops, tile_case(i), 'cuda')):
                out[f'{i}/{j}'] = t
        torch.cuda.synchronize()
    names = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
    arrs = {k: (v.view(torch.int16) if v.dtype in (torch.bfloat16, torch.float16) else v).cpu().numpy() for k, v in out.items()}
    np.savez(path, kernels=np.array(names), **arrs)


if __name__ == '__main__':
    main(sys.argv[1])
