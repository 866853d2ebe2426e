"""GPU experiment: graph-timed conv_tc launches over channel counts / kernel sizes / epilogue options, plus the
other conv shapes one steady RefVSR_MFID window runs (gate + residual, two sources, pixel shuffle, the HR tail).
Buffers rotate over six sets, so the larger maps are L2-cold."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from refvsr_b200 import packing
from refvsr_b200.lib import CudaOps, ACT_RELU
ops = CudaOps()
H, W = 270, 480
dt = torch.bfloat16

def timeit(fn, iters=20, warm=3):
    for i in range(warm): fn(i)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(iters): fn(i)
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3

def case(cin, cout, k, res=True, calloc=None, hw=(H, W), gate=False, cin1=0, shuffle=False, out_dtype=dt, cout_alloc=None):
    h, w = hw
    calloc = calloc or cin
    cout_alloc = cout_alloc or cout
    wgt = torch.randn(cout, cin + cin1, k, k) * 0.05
    srcs = [(cin, calloc)] + ([(cin1, cin1)] if cin1 else [])
    layer = packing.pack_conv('x', wgt, torch.zeros(cout), srcs, 1, k // 2, dt, 'cuda', True, ps_rows=shuffle)
    nrot = 6
    oshape = (2 * h, 2 * w, cout // 4) if shuffle else (h, w, cout_alloc)
    xs = [torch.randn((h, w, calloc), device='cuda').to(dt) for _ in range(nrot)]
    x1 = [torch.randn((h, w, cin1), device='cuda').to(dt) for _ in range(nrot)] if cin1 else None
    rs = [torch.randn((h, w, cout), device='cuda').to(dt) for _ in range(nrot)] if res else None
    gs = [torch.rand((h, w, cout), device='cuda').to(dt) for _ in range(nrot)] if gate else None
    ys = [torch.empty(oshape, device='cuda', dtype=out_dtype) for _ in range(nrot)]
    t = timeit(lambda i: ops.conv2d(layer, xs[i % nrot], x1[i % nrot] if cin1 else None, ys[i % nrot],
                                    gate=gs[i % nrot] if gate else None, res=rs[i % nrot] if res else None,
                                    act_pre=ACT_RELU, pixel_shuffle=shuffle))
    fl = 2.0 * k * k * (cin + cin1) * cout * h * w
    tag = (f'cin {cin:3d}{"+" + str(cin1) if cin1 else "":3s} (alloc {calloc:3d}) cout {cout:3d} k{k} res={int(res)} gate={int(gate)}'
           f' ps={int(shuffle)} {str(out_dtype)[6:]:8s} {h}x{w}')
    print(f'{tag}: {t:7.1f} us  {fl / t / 1e6:7.1f} TFLOP/s', flush=True)

case(48, 48, 3)
case(48, 48, 3, res=False)
case(64, 64, 3)
case(64, 64, 3, res=False)
case(48, 48, 3, calloc=64)
case(32, 32, 3)
case(16, 16, 3)
case(48, 48, 1)
case(64, 64, 1)
case(48, 48, 5)
case(64, 64, 7)
case(32, 64, 7)
case(48, 48, 3, hw=(540, 960))
case(64, 64, 3, hw=(540, 960))
case(48, 192, 3)
case(96, 48, 3)
# the window's other conv shapes
case(48, 48, 3, gate=True)                                     # feat_fusion.1.0
case(48, 48, 3, gate=True, hw=(540, 960))                      # feat_fusion2.1.0 / feat_fusion_BWFW.1.0
case(48, 48, 3, res=False, cin1=48)                            # feat_fusion.0.0 (two sources)
case(48, 48, 3, res=False, cin1=48, hw=(540, 960))             # feat_fusion2.0.0 / feat_fusion_BWFW.0.0
case(48, 192, 3, res=False, shuffle=True)                      # upsample1
case(48, 192, 3, res=False, shuffle=True, hw=(540, 960))       # upsample2
case(48, 48, 3, res=False, hw=(1080, 1920))                    # conv_hr
case(48, 3, 3, res=False, hw=(1080, 1920), out_dtype=torch.float32, cout_alloc=4)   # conv_last
