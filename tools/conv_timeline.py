"""Per-tile cycle timeline of the tensor-core convolution (conv_tc.cu) on the GPU.

Builds conv_tc.cu with -DRV_CONV_TIMELINE into a separate library (linked with the product's other objects from
build(), which must have run), loads it in place of librefvsr_b200.so and runs the 3x3 convs that dominate a window.
The instrumented kernel writes clock64 stamps per CTA, per role and per local tile (see RV_TL in conv_tc.cu); this prints,
per phase, the median and p90 cycles per tile, the time per tile per CTA, and the share of each CTA's span in which at
least one consumer has wgmmas in flight.  Besides the product kernel (`full`) it runs four diagnostic variants that split
the cost: `mma` (the consumers re-issue the 54-wgmma batch on a resident slot: no slot waits, no epilogue), `mma_aligned`
(the same count with every A view on a 1024-byte swizzle atom), `epi` (epilogue only) and `nosmem_epi` (the full
pipeline with an epilogue that neither reads nor writes shared memory; TMA-store kernels only).  The variants need convs with
one pipeline stage per tile (one channel chunk), which all shapes here are.

    python tools/conv_timeline.py [--csrc DIR] [--tag NAME] [--json FILE] [--out DIR] [--build-only | --prebuilt]
                                  [--shapes SUBSTR,...] [--max-slots N] [--consumers 2]

--csrc builds the conv_tc.cu of another tree (e.g. the parent commit's, whose build() has run) for a before/after
comparison; the stamp layout of either version is read from the library.  --consumers 2 runs the two-consumer kernel for
every conv (rv_set_conv_consumers) where the plan would take three.
The library goes to --out, by default a new temporary directory; --build-only stops there and --prebuilt runs what an
earlier --build-only left in --out."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VARIANTS = {'full': 0, 'mma': 1, 'mma_aligned': 2, 'epi': 3, 'nosmem_epi': 4}


def build_lib(csrc, out_dir):
    from __graft_entry__ import SOURCES
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    # the other objects come from build() of the tree that holds `csrc`, so that an older conv_tc.cu links against the
    # host code of its own version
    objs = [os.path.join(csrc, 'build', s[:-3] + '.o') for s in SOURCES if s != 'conv_tc.cu']
    missing = [o for o in objs if not os.path.isfile(o)]
    if missing:
        raise SystemExit(f'product objects missing (run build() first): {missing}')
    obj = os.path.join(out_dir, 'conv_tc_timeline.o')
    lib = os.path.join(out_dir, 'librefvsr_b200_timeline.so')
    arch = ['-gencode', 'arch=compute_90a,code=sm_90a']
    cmd = [nvcc] + arch + ['-O3', '-std=c++17', '-Xcompiler', '-fPIC', '-DRV_CONV_TIMELINE',
                           '-I', csrc, '-c', os.path.join(csrc, 'conv_tc.cu'), '-o', obj]
    print('[timeline]', ' '.join(cmd), flush=True)
    subprocess.run(cmd, check=True)
    subprocess.run([nvcc] + arch + ['-shared', '-o', lib, obj] + objs, check=True)
    return lib


def shapes():
    # (name, cin, cout, H, W, residual, pixel shuffle, gate)
    return [('48->48 res 270x480', 48, 48, 270, 480, True, False, False),
            ('48->48 nores 270x480', 48, 48, 270, 480, False, False, False),
            ('48->48 res 540x960', 48, 48, 540, 960, True, False, False),
            ('48->48 gate+res 270x480', 48, 48, 270, 480, True, False, True),
            ('conv_hr 1080x1920', 48, 48, 1080, 1920, False, False, False),
            ('upsample1 270x480', 48, 192, 270, 480, False, True, False),
            ('upsample2 540x960', 48, 192, 540, 960, False, True, False)]


def pct(v, q):
    import numpy as np
    return float(np.percentile(v, q)) if len(v) else float('nan')


def stamp_layout(roles):
    """What the stamps of a library with `roles` roles mean (see RV_TL in conv_tc.cu): producer roles, consumer roles (the
    i-th producer role serves the i-th consumer role), phases (name, 'p' | 'c', event a, event b), the consumer events that
    bracket its wgmmas, and box latencies (name, producer issue event, consumer event that has the box)."""
    if roles == 3:
        # conv_tc.cu before the per-consumer producer warps: one producer for both consumers, the turn wait inside the
        # full-slot wait, the store-drain wait inside the epilogue
        return dict(prod=[], cons=[1, 2], mma=(2, 3), lat=[], phases=[
            ('producer empty-slot wait', 'p0', 0, 1), ('producer TMA issue', 'p0', 1, 2),
            ('consumer full-slot + turn wait', 'c', 0, 1), ('consumer fence to first wgmma', 'c', 1, 2),
            ('consumer wgmma issue -> wait_group 0', 'c', 2, 3), ('consumer epilogue-buffer wait (+ copy)', 'c', 3, 4),
            ('consumer epilogue', 'c', 4, 5), ('consumer tile (full wait start -> epilogue end)', 'c', 0, 5)])
    # roles // 2 consumer roles, consumer c at roles // 2 + c; a kernel with fewer consumers leaves the last ones empty
    n = roles // 2
    return dict(prod=list(range(n)), cons=list(range(n, roles)), mma=(3, 4),
                lat=[('A box issue -> consumer has it', 2, 1), ('gate/res box issue -> consumer has it', 5, 5)], phases=[
                    ('producer A empty-slot wait', 'p', 0, 1), ('producer A issue', 'p', 1, 2),
                    ('producer gate/res empty-buffer wait', 'p', 3, 4),
                    ('consumer full-slot wait', 'c', 0, 1), ('consumer turn wait', 'c', 1, 2),
                    ('consumer fence to first wgmma', 'c', 2, 3), ('consumer wgmma issue -> wait_group 0', 'c', 3, 4),
                    ('consumer epilogue-buffer wait', 'c', 4, 5), ('consumer store-drain wait', 'c', 6, 7),
                    ('consumer epilogue (from operands ready)', 'c', 5, 8),
                    ('consumer tile (full wait start -> epilogue end)', 'c', 0, 8)])


def analyse(tl):
    """tl: int64 [ctas, roles, tiles, ev] (0 = not stamped).  Returns phase -> (median, p90, count) cycles, the cycles per
    tile of each CTA (its span over its consumers' tiles) and each CTA's share of its span with wgmmas in flight.  A box
    latency runs from its issue to the end of the consumer's wait for it, or to the start of a consumer that did not wait."""
    lay = stamp_layout(tl.shape[1])
    ctas = [c for c in range(tl.shape[0]) if tl[c].any()]
    phases = {}

    def put(name, vals):
        if vals:
            phases[name] = (pct(vals, 50), pct(vals, 90), len(vals))

    def add(name, a, b, role_sel):
        vals = []
        for c in ctas:
            for r in role_sel:
                x = tl[c, r]
                ok = (x[:, a] != 0) & (x[:, b] != 0)
                vals.extend((x[ok, b] - x[ok, a]).tolist())
        put(name, vals)

    cons = lay['cons']
    for name, kind, a, b in lay['phases']:
        add(name, a, b, [0] if kind == 'p0' else lay['prod'] if kind == 'p' else cons)
    for name, pe, ce in lay['lat']:
        vals = []
        for c in ctas:
            for pr, cr in zip(lay['prod'], cons):
                x, y = tl[c, pr, :, pe], tl[c, cr, :, ce]
                ok = (x != 0) & (y != 0)
                vals.extend((y[ok] - x[ok]).tolist())
        put(name, vals)
    m0, m1 = lay['mma']
    per_tile, busy = [], []
    for c in ctas:
        st = tl[c][tl[c] != 0]
        span = int(st.max() - st.min())
        n = sum(int(((tl[c, r, :, m1] != 0)).sum()) for r in cons)
        if n:
            per_tile.append(span / n)
        iv = sorted((int(x[m0]), int(x[m1])) for r in cons for x in tl[c, r] if x[m0] and x[m1])
        cover, end = 0, None
        for a, b in iv:
            if end is None or a > end:
                cover += b - a
                end = b
            elif b > end:
                cover += b - end
                end = b
        if span and iv:
            busy.append(cover / span)
    return phases, per_tile, busy


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--csrc', default=os.path.join(ROOT, 'refvsr_b200', 'csrc'), help='directory holding conv_tc.cu')
    ap.add_argument('--tag', default='')
    ap.add_argument('--json', default=None, help='write the results here')
    ap.add_argument('--build-only', action='store_true')
    ap.add_argument('--out', default=None, help='build directory (default: a new temporary directory)')
    ap.add_argument('--prebuilt', action='store_true', help='run the library an earlier --build-only left in --out')
    ap.add_argument('--variants', default='full,mma,mma_aligned,epi')
    ap.add_argument('--shapes', default='', help='comma-separated substrings of the shape names to run (default: all)')
    ap.add_argument('--max-slots', type=int, default=0, help='cap the A ring at this many slots per consumer (0: the plan)')
    ap.add_argument('--consumers', type=int, default=0, help='2: the two-consumer kernel for every conv (0: the plan)')
    args = ap.parse_args()
    out_dir = args.out or tempfile.mkdtemp(prefix='conv_timeline_')
    os.makedirs(out_dir, exist_ok=True)
    if args.prebuilt:
        path = os.path.join(out_dir, 'librefvsr_b200_timeline.so')
    else:
        path = build_lib(os.path.abspath(args.csrc), out_dir)
        print('[timeline] built', path, flush=True)
    if args.build_only:
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('conv_timeline: no CUDA device')
    from refvsr_b200 import lib as L, packing
    L._lib = None
    # an older library (--csrc) may lack host-only queries added since; the timeline calls none of them
    have = C.CDLL(path)
    for name in [n for n in L.SIGNATURES if not hasattr(have, n)]:
        del L.SIGNATURES[name]
    lib = L.load_library(path)
    lib.rv_conv_timeline_set.restype = C.c_int
    lib.rv_conv_timeline_set.argtypes = [C.c_void_p, C.c_int]
    dims = (C.c_int * 3)()
    lib.rv_conv_timeline_dims(dims)
    roles, ntl, nev = dims[0], dims[1], dims[2]
    ops = L.CudaOps()
    props = torch.cuda.get_device_properties(0)
    nsm = props.multi_processor_count
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        print('[timeline] gpu:', q, flush=True)
    except Exception as ex:                                     # noqa: BLE001
        print('[timeline] nvidia-smi unavailable:', ex, flush=True)
    dt = torch.bfloat16
    buf = torch.zeros(2 * nsm * roles * ntl * nev, dtype=torch.int64, device='cuda')
    results = {}
    if args.max_slots:
        lib.rv_conv_timeline_max_slots(args.max_slots)
    if args.consumers:
        lib.rv_set_conv_consumers(args.consumers)
    only = [s for s in args.shapes.split(',') if s]
    for name, cin, cout, h, w, res, ps, gate in shapes():
        if only and not any(s in name for s in only):
            continue
        torch.manual_seed(0)
        wgt = torch.randn(cout, cin, 3, 3) * 0.05
        layer = packing.pack_conv('x', wgt, torch.zeros(cout), [(cin, cin)], 1, 1, dt, 'cuda', True, ps_rows=ps)
        nrot = 3
        xs = [torch.randn((h, w, cin), device='cuda').to(dt) for _ in range(nrot)]
        rs = [torch.randn((h, w, cout), device='cuda').to(dt) for _ in range(nrot)] if res else None
        gs = [torch.rand((h, w, cout), device='cuda').to(dt) for _ in range(nrot)] if gate else None
        oshape = (2 * h, 2 * w, cout // 4) if ps else (h, w, cout)
        ys = [torch.empty(oshape, device='cuda', dtype=dt) for _ in range(nrot)]

        def run(i):
            ops.conv2d(layer, xs[i % nrot], None, ys[i % nrot], gate=gs[i % nrot] if gate else None,
                       res=rs[i % nrot] if res else None, act_pre=L.ACT_RELU, pixel_shuffle=ps)
        results[name] = {}
        for vname in args.variants.split(','):
            diag = VARIANTS[vname]
            assert lib.rv_conv_timeline_set(None, diag) == 0
            for i in range(3):
                run(i)
            torch.cuda.synchronize()
            iters = 20
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(iters):
                run(i)
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) / iters * 1e3
            buf.zero_()
            assert lib.rv_conv_timeline_set(C.c_void_p(buf.data_ptr()), diag) == 0
            run(0)
            torch.cuda.synchronize()
            assert lib.rv_conv_timeline_set(None, 0) == 0
            tl = buf.view(-1, roles, ntl, nev).cpu().numpy()
            phases, per_tile, busy = analyse(tl)
            nct = len([c for c in range(tl.shape[0]) if tl[c].any()])
            r = {'us': us, 'ctas': nct, 'phases': phases,
                 'per_tile_per_cta_cycles': (pct(per_tile, 50), pct(per_tile, 90)),
                 'mma_busy_share': (pct(busy, 50), pct(busy, 10))}
            results[name][vname] = r
            print(f'\n== {args.tag} {name} [{vname}]: {us:.1f} us per launch, {nct} CTAs; per tile per CTA '
                  f'{r["per_tile_per_cta_cycles"][0]:.0f} cycles (p90 {r["per_tile_per_cta_cycles"][1]:.0f}); '
                  f'wgmmas in flight {100 * r["mma_busy_share"][0]:.0f} % of the CTA span (p10 {100 * r["mma_busy_share"][1]:.0f} %)',
                  flush=True)
            for ph, (med, p90, n) in phases.items():
                print(f'   {ph:48s} median {med:8.0f}  p90 {p90:8.0f}  cycles  (n={n})', flush=True)
        del xs, rs, gs, ys
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump({'tag': args.tag, 'results': results}, f, indent=1)


if __name__ == '__main__':
    main()
