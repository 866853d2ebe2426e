"""The C-ABI library loads and exports every symbol include/refvsr_b200.h declares (no compute calls)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, 'include', 'refvsr_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(rv_[a-z0-9_]+)\s*\(', src)))


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as ge
    ge.build()
    from refvsr_b200.lib import LIB_PATH, SIGNATURES
    lib = ctypes.CDLL(LIB_PATH)
    names = header_functions()
    assert len(names) >= 18
    for n in names:
        assert hasattr(lib, n), f'{n} declared in the header but not exported'
    assert sorted(SIGNATURES) == names, 'python prototypes and header are out of sync'
    lib.rv_version.restype = ctypes.c_int
    assert lib.rv_version() == 100


def test_descriptor_struct_matches_header():
    """field order of rv_conv_desc in the ctypes mirror == the header's struct"""
    from refvsr_b200.lib import rv_conv_desc
    src = open(os.path.join(ROOT, 'include', 'refvsr_b200.h')).read()
    body = src[src.index('typedef struct rv_conv_desc {'):src.index('} rv_conv_desc;')]
    body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
    fields = []
    for decl in body.split('{', 1)[1].split(';'):
        decl = decl.strip()
        if not decl:
            continue
        names = decl.split(None, 1)[1] if not decl.startswith('const') else decl.split(None, 2)[2]
        for nm in names.split(','):
            fields.append(nm.replace('*', '').strip())
    assert fields == [f[0] for f in rv_conv_desc._fields_]


def test_invalid_arguments_return_error_codes_without_a_gpu():
    from refvsr_b200.lib import load_library
    lib = load_library()
    rc = lib.rv_conv2d(None, None)
    assert rc == -1 and b'null descriptor' in lib.rv_last_error()
    rc = lib.rv_conf_max(None, None, None, 0, None)
    assert rc == -1


def test_tensor_core_conv_plans_fit_and_keep_rings_per_consumer():
    """rv_conv2d_tc_plan is host-only, so every conv shape of the path is planned here without a GPU, for the H100's limits
    (232 448 B opt-in shared memory, 132 SMs) and for smaller hypothetical budgets: each of the two consumer warpgroups gets a
    ring of >= 1 slot of its own, the plan fits the budget, and layout 1 (all taps as views of one box) only with resident
    weights."""
    import ctypes as C
    from refvsr_b200.lib import load_library, rv_conv_desc
    lib = load_library()
    buf = (C.c_char * 4096)()
    ptr = (C.addressof(buf) + 255) & ~255
    shapes = []      # (c0, c1, cout, nb, k, layout, pixel_shuffle, res)
    for C_ in (24, 48):
        nb = (C_ + 15) // 16 * 16
        shapes += [(C_, 0, C_, nb, 3, 1, 0, 1), (C_, C_, C_, nb, 3, 1, 0, 0), (8, C_, C_, nb, 3, 1, 0, 0), (C_, 0, 4 * C_, min(96, 4 * C_), 3, 1, 1, 0),
                   (C_, C_, C_, nb, 1, 1, 0, 0), (C_, 0, C_, nb, 3, 0, 0, 1), (C_, 0, C_, nb, 3, 2, 0, 1), (C_, 0, C_, nb, 3, 3, 0, 1)]
    shapes += [(8, 0, 32, 32, 7, 1, 0, 0), (32, 0, 64, 64, 7, 1, 0, 0), (64, 0, 32, 32, 7, 1, 0, 0), (32, 0, 16, 16, 7, 1, 0, 0), (16, 0, 2, 16, 7, 1, 0, 0),
               (8, 0, 64, 64, 3, 1, 0, 0), (64, 0, 64, 64, 3, 1, 0, 0), (64, 0, 128, 64, 3, 1, 0, 0), (128, 0, 16, 16, 1, 1, 0, 0),
               (8, 0, 32, 32, 5, 1, 0, 0), (32, 0, 32, 32, 3, 1, 0, 1), (128, 128, 32, 32, 3, 1, 0, 0), (192, 0, 48, 48, 3, 1, 0, 0), (48, 0, 3, 16, 3, 1, 0, 0)]
    seen = set()
    for max_smem, sms in ((232448, 132), (166912, 132), (101376, 84)):
        for (c0, c1, cout, nb, k, layout, ps, res) in shapes:
            for (H, W) in ((270, 480), (1080, 1920), (37, 53)):
                d = rv_conv_desc()
                d.src0, d.src1 = ptr, (ptr if c1 else None)
                d.c0, d.c1, d.in_dtype, d.H, d.W = c0, c1, 2, H, W
                d.wpack, d.bias, d.cout, d.kh, d.kw, d.stride, d.pad = ptr, ptr, cout, k, k, 1, k // 2
                d.res, d.res_cs, d.res_dtype = (ptr if res else None), (cout if res else 0), 2
                d.out, d.out_cs, d.out_dtype = ptr, (cout // 4 if ps else cout), 2
                d.pixel_shuffle, d.impl, d.nb, d.k_real, d.layout = ps, 1, nb, k * k * (c0 + c1), layout
                out = (C.c_int32 * 8)()
                rc = lib.rv_conv2d_tc_plan(C.byref(d), max_smem, sms, out)
                if rc != 0:      # a shape this budget cannot hold is refused with a message, never mis-planned
                    assert lib.rv_last_error()
                    continue
                mode, slots, resident, S, ncons, nacc, nb_, smem = list(out)
                seen.add((mode, resident))
                assert mode == (1 if layout in (1, 3) else layout) and nb_ == nb, (c0, c1, cout, k, layout, list(out))
                assert ncons == nacc == 2 and slots >= 1 and smem <= max_smem, (c0, c1, cout, k, layout, list(out))
                assert resident or mode != 1, (c0, c1, cout, k, layout, list(out))
    assert {m for m, _ in seen} >= {0, 1, 2}      # the sweep reaches every mode
