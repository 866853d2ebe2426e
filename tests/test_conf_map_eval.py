"""The confidence-map evaluation mode (`run.py --eval_mode conf`, evaluation/eval_quan_conf_map.py) on rv_conf_map_images: the
colour table and matplotlib's index rule, the kernel's bytes against the reference's steps (tests/conf_map_oracle.py), and the
image tree, printed lines and score file of run.py with and without the drop-in."""
import os
import re
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, 'tests')
sys.path.insert(0, ROOT)
sys.path.insert(0, TESTS)

import conf_map_oracle as CO                                                  # noqa: E402
from refvsr_b200.colormap import inferno_lut, matplotlib_inferno_rgb8, opencv_inferno_rgb8, rgb8_of   # noqa: E402
from test_dropin_runpy import ENV_DIR, SHIMS, _ref_root, make_ckpt, make_tree   # noqa: E402

ONE_MINUS_ULP = float(np.nextafter(np.float32(1), np.float32(0)))


def colormap_index(y):
    """the kernel's rule (include/refvsr_b200.h, rv_conf_map_images) for float32 y: table index, or None for the bad colour"""
    t = np.float32(y) * np.float32(256)
    if np.isnan(t):
        return None
    return 255 if t >= 256 else (0 if t < 0 else int(t))


# ---------------------------------------------------------------- CPU

def test_lut_from_opencv_equals_matplotlib():
    if not CO.have_matplotlib():
        pytest.skip('matplotlib is not installed: the OpenCV table is the only source here')
    assert np.array_equal(opencv_inferno_rgb8(), matplotlib_inferno_rgb8())


def test_standin_reproduces_the_opencv_table():
    """the stand-in's float table (OpenCV's bytes / 255) goes through the reference's float32 * 255 rounding to the same bytes"""
    cmap = CO.colormap()
    lut = rgb8_of(cmap(np.arange(256))[:, :3])
    assert np.array_equal(lut, opencv_inferno_rgb8())
    assert lut.shape == (256, 3) and tuple(lut[0]) == (0, 0, 4) and tuple(lut[255]) == (252, 255, 164)


@pytest.mark.parametrize('y,idx', [(0.0, 0), (1.0, 255), (255 / 256, 255), (ONE_MINUS_ULP, 255), (float('nan'), None),
                                   (0.5, 128), (np.float32(1 / 256) - 1e-9, 0), (-0.0, 0), (-0.25, 0), (7.0, 255),
                                   (float('inf'), 255), (float('-inf'), 0)])
def test_colormap_index_rule(y, idx):
    """matplotlib's Colormap.__call__ on a float32 array (the real one when installed) picks the entry the kernel's rule picks"""
    assert colormap_index(y) == idx
    cmap = CO.colormap()
    got = cmap(np.array([[y]], np.float32))[0, 0]
    want = np.zeros(4) if idx is None else cmap(np.array([idx]))[0]
    assert np.array_equal(got, want), (y, got, want)


def test_dropin_resolves_under_run_py():
    """eval.py's `from evaluation.eval_quan_conf_map import eval_quan_conf_map` takes the drop-in, with the reference's
    `init` next to it"""
    ref = _ref_root()
    if ref is None:
        pytest.skip('no reference checkout')
    code = ('import eval as E, evaluation, evaluation.eval_quan_conf_map as m, evaluation.init as i\n'
            'assert E.eval_quan_conf_map is m.eval_quan_conf_map, E.eval_quan_conf_map\n'
            'assert m.__file__.startswith(%r), m.__file__\n'
            'assert i.__file__.startswith(%r), i.__file__\n'
            'assert m._reference_impl().__module__ == "evaluation._reference_eval_quan_conf_map"\n'
            'print("ok")\n' % (os.path.join(ROOT, 'refvsr_b200', 'dropin'), ref))
    pp = [ENV_DIR, os.path.join(ROOT, 'refvsr_b200', 'dropin'), ROOT, SHIMS]
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(pp), REFVSR_TEST_ENV='1')
    r = subprocess.run([sys.executable, '-B', '-c', code], cwd=ref, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and 'ok' in r.stdout, r.stdout + r.stderr


LAUNCH_WITH_ORACLE = ('import sys, runpy; sys.path.insert(0, {tests!r}); import conf_map_oracle as m; '
                      'sys.path.remove({tests!r}); m.install(); sys.argv[0] = "run.py"; runpy.run_path("run.py", run_name="__main__")')


def run_conf(ref, tmp, tag, config, dropin_loop, cpu, frame_num=3, extra_env=None, timeout=1500):
    """run.py --eval_mode conf with the engine network (the models drop-in) in both arms: the drop-in loop, or the reference's
    (REFVSR_DROPIN_EVAL=0, with the matplotlib stand-in when matplotlib is absent).  On the CPU the engine's operator set is the
    oracle's test double, with tests/conf_map_oracle.py as its image step.  Returns (stdout, score file, {relative path: file})."""
    out = os.path.join(tmp, 'out_' + tag)
    standin = [] if (dropin_loop or CO.have_matplotlib()) else [CO.ENV]
    pp = [ENV_DIR] + standin + [os.path.join(ROOT, 'refvsr_b200', 'dropin'), ROOT, SHIMS]
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(pp), REFVSR_TEST_ENV='1', PYTHONDONTWRITEBYTECODE='1')
    if not dropin_loop:
        env['REFVSR_DROPIN_EVAL'] = '0'
    env.update(extra_env or {})
    args = ['--mode', 'conf_eval', '--project', os.path.join(tmp, 'logs_' + tag), '--config', config, '--data', 'RealMCVSR',
            '--ckpt_abs_name', os.path.join(tmp, 'ckpt.pytorch'), '--data_offset', os.path.join(tmp, 'data'),
            '--output_offset', out, '--frame_num', str(frame_num), '--eval_mode', 'conf'] + (['-cpu'] if cpu else [])
    launch = ['-c', LAUNCH_WITH_ORACLE.format(tests=TESTS)] if cpu else ['run.py']
    r = subprocess.run([sys.executable, '-B'] + launch + args, cwd=ref, env=env, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, f'run.py ({tag}) failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}'
    assert 'All keys matched successfully' in r.stdout, r.stdout[-2000:]
    files = {re.sub(r'/\d{4}_\d{2}_\d{2}_\d{4}/', '/DATE/', os.path.relpath(os.path.join(d, f), out)): os.path.join(d, f)
             for d, _, fs in os.walk(out) for f in fs}
    scores = [p for k, p in files.items() if k.endswith('score_RealMCVSR_conf.txt')]
    assert len(scores) == 1, sorted(files)
    return r.stdout, open(scores[0]).read(), files


def loop_lines(text):
    """the loop's printed lines from '[EVAL' on, with the seconds masked"""
    text = text[text.index('[EVAL'):]
    return re.sub(r'\(\d+\.\d+sec\)', '(#sec)', text)


def compare_runs(ref_run, dropin_run, frames):
    (base, base_score, base_files), (ours, ours_score, ours_files) = ref_run, dropin_run
    assert loop_lines(base) == loop_lines(ours)
    assert loop_lines(base_score) == loop_lines(ours_score)
    assert len(re.findall(r'^\[EVAL ', base_score, re.M)) == frames and base_score.count('[MEAN EVAL') == 1
    assert '[TOTAL' in base_score
    assert set(base_files) == set(ours_files), sorted(set(base_files) ^ set(ours_files))[:8]
    images = sorted(k for k in base_files if k.endswith(('.png', '.jpg')))
    # input, output and four maps, png and jpg, per frame
    assert len(images) == 12 * frames, len(images)
    for k in images:
        with open(base_files[k], 'rb') as fa, open(ours_files[k], 'rb') as fb:
            assert fa.read() == fb.read(), k
    return images


def test_run_py_conf_reference_loop_vs_dropin_cpu(tmp_path):
    """both arms run the engine network on the oracle's CPU operator set, so only the loop differs: the drop-in's (images from
    the yardstick restatement) and the reference's.  Every png and jpg is byte-identical; the lines match with the seconds masked"""
    ref = _ref_root()
    if ref is None:
        pytest.skip('no reference checkout')
    tmp = str(tmp_path)
    make_tree(os.path.join(tmp, 'data'), 24, 32)
    make_ckpt(os.path.join(tmp, 'ckpt.pytorch'), 'config_RefVSR_small_L1')
    env = {'REFVSR_TEST_ORACLE_OPS': '1'}
    base = run_conf(ref, tmp, 'ref', 'config_RefVSR_small_L1', dropin_loop=False, cpu=True, extra_env=env)
    ours = run_conf(ref, tmp, 'b200', 'config_RefVSR_small_L1', dropin_loop=True, cpu=True, extra_env=env)
    compare_runs(base, ours, frames=6)


# ---------------------------------------------------------------- GPU

def tie_values(n, seed):
    """n float32 values x in (0, 1) with fl32(x * 255) exactly k + 0.5: cv2's round half to even decides them"""
    out = []
    for k in np.random.default_rng(seed).permutation(255):
        x = np.float32((k + 0.5) / 255)
        if np.float32(x * np.float32(255)) == np.float32(k + 0.5):
            out.append(x)
    assert len(out) >= n
    return np.array(out[:n], np.float32)


def frame(h, w, seed):
    """(1, 3, h, w) fp32 with values below 0, above 1, 0 and 1 exactly, and exact x.5 / 255 ties"""
    g = torch.Generator().manual_seed(seed)
    f = torch.rand(1, 3, h, w, generator=g) * 1.4 - 0.2
    flat = f.view(-1)
    ties = torch.from_numpy(tie_values(64, seed))
    idx = torch.randperm(flat.numel(), generator=g)[:min(flat.numel(), 200)]
    flat[idx[:64]] = ties[:len(idx[:64])]
    flat[idx[64:68]] = torch.tensor([0.0, 1.0, -0.0, 255.5 / 255])[:len(idx[64:68])]
    return f


def conf_maps(h, w, seed, constant_forward=False):
    g = torch.Generator().manual_seed(seed)
    bw = torch.rand(1, 1, h, w, generator=g) * 0.8 + 0.1
    fw = torch.full((1, 1, h, w), 0.375) if constant_forward else torch.rand(1, 1, h, w, generator=g)
    conf = torch.rand(1, 1, h, w, generator=g) ** 2
    return [conf, torch.maximum(bw, fw), bw, fw]


def kernel_bytes(ops, maps, inp, out, normalize):
    packed = ops.conf_map_images([m.cuda() for m in maps], inp.cuda(), out.cuda(), inferno_lut('cuda'), normalize)
    torch.cuda.synchronize()
    return packed.cpu().numpy()


def assert_bytes_equal(got, imgs):
    want = CO.packed(imgs)
    assert got.shape == want.shape, (got.shape, want.shape)
    off = 0
    for k, img in enumerate(imgs):                            # name the first image that differs
        n = img.size
        bad = np.flatnonzero(got[off:off + n] != img.reshape(-1))
        assert bad.size == 0, f'image {k}: {bad.size} bytes differ, first at {bad[0]}: {got[off + bad[0]]} vs {img.reshape(-1)[bad[0]]}'
        off += n


@pytest.mark.gpu
@pytest.mark.parametrize('h,w,scale', [(270, 480, 4), (271, 483, 4), (17, 31, 2), (1, 1, 1)])
def test_conf_map_kernel_bytes_match_reference(cuda_ops, h, w, scale):
    maps = conf_maps(h, w, seed=h * w)
    inp, out = frame(h, w, seed=h), frame(scale * h, scale * w, seed=w)
    if h == 1:
        maps = [torch.full((1, 1, 1, 1), v) for v in (0.5, 0.25, 0.125, 1.0)]    # single pixels: 0 / 0 everywhere, all black
    imgs = CO.reference_images(maps, inp, out, normalize=True)
    got = kernel_bytes(cuda_ops, maps, inp, out, True)
    assert_bytes_equal(got, imgs)
    assert np.array_equal(got, kernel_bytes(cuda_ops, maps, inp, out, True)), 'two calls differ'
    if h == 1:
        assert not got[:12].any()


@pytest.mark.gpu
def test_conf_map_kernel_constant_map_is_black(cuda_ops):
    """a constant forward map (a clip's first window) normalises to 0 / 0 = NaN: matplotlib's bad colour, black"""
    h, w = 64, 96
    maps = conf_maps(h, w, seed=3, constant_forward=True)
    inp, out = frame(h, w, 5), frame(4 * h, 4 * w, 6)
    got = kernel_bytes(cuda_ops, maps, inp, out, True)
    assert_bytes_equal(got, CO.reference_images(maps, inp, out, normalize=True))
    fwd = got[3 * 3 * h * w:4 * 3 * h * w]
    assert not fwd.any()
    assert got[:3 * h * w].any()


@pytest.mark.gpu
def test_conf_map_kernel_unnormalised_branch(cuda_ops):
    """a vis without conf_map_prop: conf_map alone, coloured as it is - out-of-range, NaN and the index rule's edge values"""
    h, w = 19, 37
    g = torch.Generator().manual_seed(9)
    conf = torch.rand(1, 1, h, w, generator=g) * 1.6 - 0.3
    edge = torch.tensor([0.0, 1.0, 255 / 256, ONE_MINUS_ULP, float('nan'), -0.0, 2.0, -1.0, float('inf'), float('-inf'), 0.5])
    conf.view(-1)[:edge.numel()] = edge
    inp, out = frame(h, w, 1), frame(2 * h, 2 * w, 2)
    got = kernel_bytes(cuda_ops, [conf], inp, out, False)
    assert_bytes_equal(got, CO.reference_images([conf], inp, out, normalize=False))
    lut = opencv_inferno_rgb8()
    for k, v in enumerate(edge.tolist()):
        idx = colormap_index(v)
        want = (0, 0, 0) if idx is None else tuple(lut[idx][::-1])
        assert tuple(got[3 * k:3 * k + 3]) == want, (v, tuple(got[3 * k:3 * k + 3]), want)


@pytest.mark.gpu
def test_conf_map_kernel_nan_in_a_map(cuda_ops):
    """torch's min() / max() of a map holding NaN are NaN, so the whole normalised map is NaN: black"""
    h, w = 33, 40
    maps = conf_maps(h, w, seed=4)
    maps[2] = maps[2].clone()
    maps[2][0, 0, 5, 7] = float('nan')
    inp, out = frame(h, w, 7), frame(2 * h, 2 * w, 8)
    got = kernel_bytes(cuda_ops, maps, inp, out, True)
    assert_bytes_equal(got, CO.reference_images(maps, inp, out, normalize=True))
    assert not got[2 * 3 * h * w:3 * 3 * h * w].any()


@pytest.mark.gpu
def test_conf_map_kernel_rejects_bad_arguments(cuda_ops):
    h, w = 16, 24
    maps = [m.cuda() for m in conf_maps(h, w, seed=1)]
    inp, out, lut = frame(h, w, 1).cuda(), frame(4 * h, 4 * w, 2).cuda(), inferno_lut('cuda')
    bad = [
        (maps[:3], inp, out, lut, True),                                           # three maps with normalize
        (maps, inp, out, lut, False),                                              # four maps without
        ([maps[0].half()] + maps[1:], inp, out, lut, True),                        # not fp32
        ([maps[0][..., :8].contiguous()] + maps[1:], inp, out, lut, True),         # maps differ in shape
        (maps, inp.transpose(2, 3), out, lut, True),                               # not contiguous
        (maps, inp[:, :2].contiguous(), out, lut, True),                           # two channels
        (maps, inp, out.cpu(), lut, True),                                         # host tensor
        (maps, inp, out, lut[:128].contiguous(), True),                            # short table
        (maps, inp, out, lut.float(), True),                                       # table not uint8
    ]
    for args in bad:
        with pytest.raises(ValueError):
            cuda_ops.conf_map_images(*args)
    from refvsr_b200.lib import _ptr
    lib = cuda_ops.lib
    p = [_ptr(m) for m in maps]
    work = torch.empty(512, dtype=torch.int32, device='cuda')
    buf = torch.empty(1 << 20, dtype=torch.uint8, device='cuda')
    s = cuda_ops._stream()
    assert lib.rv_conf_map_images(*p, h, w, 2, _ptr(inp), h, w, _ptr(out), 4 * h, 4 * w, _ptr(lut), _ptr(work), _ptr(buf), s) == -1
    assert lib.rv_conf_map_images(*p, 0, w, 1, _ptr(inp), h, w, _ptr(out), 4 * h, 4 * w, _ptr(lut), _ptr(work), _ptr(buf), s) == -1
    assert lib.rv_conf_map_images(p[0], None, None, None, h, w, 1, _ptr(inp), h, w, _ptr(out), 4 * h, 4 * w, _ptr(lut),
                                  _ptr(work), _ptr(buf), s) == -1
    assert lib.rv_conf_map_images(*p, h, w, 1, _ptr(inp), h, w, None, 4 * h, 4 * w, _ptr(lut), _ptr(work), _ptr(buf), s) == -1
    got = kernel_bytes(cuda_ops, [m.cpu() for m in maps], inp.cpu(), out.cpu(), True)                # still usable
    assert_bytes_equal(got, CO.reference_images(maps, inp, out, normalize=True))


@pytest.mark.gpu
def test_run_py_conf_reference_loop_vs_dropin_gpu(tmp_path):
    """run.py --eval_mode conf on the H100 engine (RefVSR_MFID, bf16) twice: with the drop-in loop and with the reference's
    (REFVSR_DROPIN_EVAL=0).  Both use the engine network, so every png and jpg must be byte-identical, and the printed and
    score-file lines identical with the seconds masked"""
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    ref = _ref_root()
    if ref is None:
        pytest.skip('no reference checkout staged under oracle/_ref')
    tmp = str(tmp_path)
    make_tree(os.path.join(tmp, 'data'), 64, 96, videos=2, frames=4)
    make_ckpt(os.path.join(tmp, 'ckpt.pytorch'), 'config_RefVSR_MFID')
    env = {'REFVSR_TEST_PRECISION': 'bf16'}
    base = run_conf(ref, tmp, 'ref', 'config_RefVSR_MFID', dropin_loop=False, cpu=False, frame_num=7, extra_env=env)
    ours = run_conf(ref, tmp, 'b200', 'config_RefVSR_MFID', dropin_loop=True, cpu=False, frame_num=7, extra_env=env)
    images = compare_runs(base, ours, frames=8)
    for d in ('conf_map_norm', 'conf_map_prop_norm', 'conf_map_prop_b_norm', 'output'):     # the images are not blank
        assert any(cv2.imread(base[2][k]).any() for k in images if f'/{d}/' in k), d
