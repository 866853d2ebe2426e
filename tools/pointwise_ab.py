"""A/B check of two builds of the kernels library: byte identity and graph-timed launches of the pointwise kernels.

    python tools/pointwise_ab.py OLD.so NEW.so [--repeats 3] [--out DIR]

Every case of tests/test_pointwise_fp64.py (each (signature, geometry, dtype) of ENGINE_POINTWISE and every BRANCH_CASES input)
runs on its seeded operands against each library, in a subprocess per library, with and without REFVSR_NO_FAST_POINTWISE=1
(read once per process).  Each output's SHA-256 must match between the libraries.  Then the gather / reconstruction kernels are
timed at LR 270x480 (x4) and 540x960 (x2) with tools/pointwise_bench.py's method, alternating the libraries, `--repeats` times;
the report gives the card's name and power limit beside the times."""
import argparse
import hashlib
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), HERE]


def _ops(lib_path):
    from refvsr_b200 import lib
    lib.load_library(lib_path)
    return lib.CudaOps()


def hash_cases(lib_path):
    import torch
    import test_pointwise_fp64 as t
    ops = _ops(lib_path)
    res = {}
    for e, geom, dt in t._ENGINE_CASES:
        cid = f'{e.sig.op}-{e.sig.real}of{e.sig.alloc}[{t._flag_id(e)}]-{t.DTN[dt]}-{"x".join(map(str, geom))}'
        c = t.build_case(t._cpu_sig(e, dt), geom, dt, 'cuda', t._seed(e.sig, geom, t.DTN[dt]))
        res[cid] = [hashlib.sha256(o.contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()
                    for o in t.run_guarded(ops, c, 'cuda')]
    for cid, e, geom, dt, opt in t.BRANCH_CASES:
        c = t.build_case(t._cpu_sig(e, dt), geom, dt, 'cuda', t._seed(cid), n=opt.get('n', 0), C=opt.get('C'))
        res[cid] = [hashlib.sha256(o.contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()
                    for o in t.run_guarded(ops, c, 'cuda', off=opt.get('off', 0))]
    return res


def time_kernels(lib_path):
    import torch
    from pointwise_bench import timeit
    ops = _ops(lib_path)
    dev, bf = 'cuda', torch.bfloat16
    g = torch.Generator(device=dev).manual_seed(0)

    def ring(shape, dt=bf, per=None):             # enough buffers that a rotation moves > 160 MB (more than the 50 MB L2)
        nb = per or torch.Size(shape).numel() * torch.tensor([], dtype=dt).element_size()
        k = max(2, int(160e6 // nb) + 1)
        return [(torch.rand(shape, device=dev, generator=g) * 2 - 1).to(dt) for _ in range(k)]

    res = {}
    h, w, C = 270, 480, 48
    flow = torch.randn((h, w, 2), device=dev, generator=g) * 3
    conf = torch.rand((h, w), device=dev, generator=g)
    lf, up = ring((h, w, C)), ring((2 * h, 2 * w, C), per=5 * h * w * C * 2)
    lo, uo, co = [torch.empty_like(lf[0]) for _ in lf], [torch.empty_like(up[0]) for _ in up], torch.empty_like(conf)
    n = min(len(lf), len(up))
    res['warp3 270x480x48 bf16'] = timeit(lambda i: ops.warp3(lf[i % n], up[i % n], conf, flow, lo[i % n], uo[i % n], co))
    res['warp 270x480x48 bf16'] = timeit(lambda i: ops.warp(lf[i % n], flow, lo[i % n]))
    res['warp_up 270x480 -> 540x960x48 bf16'] = timeit(lambda i: ops.warp(up[i % n], flow, uo[i % n], flow_up2=True))
    aff2 = torch.rand((h, w, 3), device=dev, generator=g) * 0.4 + 0.8
    res['aligned_sample ks2 270x480 cells x48 bf16'] = timeit(lambda i: ops.aligned_sample(up[i % n], aff2, 2, uo[(i + 1) % n]))
    upf = ring((2 * h, 2 * w, C), dt=torch.float32)
    uof = [torch.empty_like(upf[0]) for _ in upf]
    nf = len(upf)
    res['aligned_sample ks2 270x480 cells x48 fp32'] = timeit(lambda i: ops.aligned_sample(upf[i % nf], aff2, 2, uof[(i + 1) % nf]))
    aff4 = torch.rand((h // 2, w // 2, 3), device=dev, generator=g) * 0.4 + 0.8
    res['aligned_sample ks4 135x240 cells x48 bf16'] = timeit(lambda i: ops.aligned_sample(up[i % n], aff4, 4, uo[(i + 1) % n]))
    for s, (lh, lw) in ((4, (270, 480)), (2, (540, 960))):
        xs = ring((s * lh, s * lw, 4), dt=torch.float32)
        lrs = [torch.rand((3, lh, lw), device=dev, generator=g) for _ in xs]
        outs = [torch.empty((3, s * lh, s * lw), device=dev) for _ in xs]
        o8 = [torch.empty((s * lh, s * lw, 3), device=dev, dtype=torch.uint8) for _ in xs]
        k = len(xs)
        res[f'reconstruct x{s} LR {lh}x{lw}'] = timeit(lambda i: ops.reconstruct(xs[i % k], lrs[i % k], s, True, outs[i % k]))
        res[f'reconstruct_u8 x{s} LR {lh}x{lw}'] = timeit(lambda i: ops.reconstruct_u8(xs[i % k], lrs[i % k], s, True, o8[i % k], False))
        res[f'reconstruct_u8 bgr x{s} LR {lh}x{lw}'] = timeit(lambda i: ops.reconstruct_u8(xs[i % k], lrs[i % k], s, True, o8[i % k], True))
    return {k: v * 1e6 for k, v in res.items()}


def _child(mode, lib_path, env=None):
    out = subprocess.run([sys.executable, __file__, '--child', mode, os.path.abspath(lib_path)], capture_output=True, text=True,
                         env={**os.environ, **(env or {})})
    if out.returncode != 0:
        raise RuntimeError(f'{mode} with {lib_path} failed:\n{out.stderr[-3000:]}')
    return json.loads(out.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('old')
    ap.add_argument('new')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip()
    report = {'gpu': gpu, 'hash_mismatches': [], 'cases': 0}
    for env in ({}, {'REFVSR_NO_FAST_POINTWISE': '1'}):
        ho, hn = _child('hash', a.old, env), _child('hash', a.new, env)
        assert sorted(ho) == sorted(hn)
        report['cases'] += len(ho)
        report['hash_mismatches'] += [(k, env) for k in ho if ho[k] != hn[k]]
    times = {'old': [], 'new': []}
    for _ in range(a.repeats):
        for which in ('old', 'new'):
            times[which].append(_child('time', getattr(a, which)))
    report['times_us'] = {k: {w: [round(t[k], 2) for t in times[w]] for w in times} for k in times['old'][0]}
    print(f'GPU: {gpu}')
    print(f'cases hashed: {report["cases"]}, mismatches: {len(report["hash_mismatches"])} {report["hash_mismatches"]}')
    print(f'{"kernel":48s} {"old us (min / max)":>22s} {"new us (min / max)":>22s}')
    for k, v in report['times_us'].items():
        print(f'{k:48s} {min(v["old"]):9.2f} / {max(v["old"]):9.2f} {min(v["new"]):9.2f} / {max(v["new"]):9.2f}')
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'pointwise_ab.json'), 'w') as f:
            json.dump(report, f, indent=1)
    return 1 if report['hash_mismatches'] else 0


if __name__ == '__main__':
    if len(sys.argv) > 1 and sys.argv[1] == '--child':
        mode, lib_path = sys.argv[2], sys.argv[3]
        print(json.dumps(hash_cases(lib_path) if mode == 'hash' else time_kernels(lib_path)))
    else:
        sys.exit(main())
