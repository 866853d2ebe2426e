"""The default evaluation mode (`run.py --eval_mode qual_quan`, evaluation/eval_qual_quan.py) on the GPU: rv_eval_images' bytes
against OpenCV's own conversion of the reference's float images, the mean SSIM from one rv_region_metrics call against
skimage's, and the image tree, printed lines and score file of run.py with the reference's loop and with the drop-in."""
import importlib.util
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, 'tests')
sys.path.insert(0, ROOT)
sys.path.insert(0, TESTS)

import region_metrics_oracle as RMO                                           # noqa: E402
from conf_map_oracle import imwrite_u8                                        # noqa: E402
from test_conf_map_eval import loop_lines, tie_values                         # noqa: E402
from test_dropin_runpy import ENV_DIR, SHIMS, _ref_root, make_ckpt, make_tree   # noqa: E402


def skimage_ssim(a, b):
    """the tests' stand-in for skimage.metrics.structural_similarity (tests/runpy_env/skimage), loaded by path"""
    spec = importlib.util.spec_from_file_location('_runpy_env_skimage_metrics', os.path.join(ENV_DIR, 'skimage', 'metrics.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.structural_similarity(a, b, data_range=1.0, multichannel=True)


def hwc(t):
    return t.detach().float().cpu().numpy()[0].transpose(1, 2, 0)


def reference_u8(t):
    """the uint8 BGR image cv2.imwrite stores for cv2.cvtColor(x * 255, RGB2BGR) of a (1, 3, H, W) frame, from cv2 itself"""
    import cv2
    return imwrite_u8(cv2.cvtColor(np.ascontiguousarray(hwc(t)) * 255, cv2.COLOR_RGB2BGR))


def frame(h, w, seed):
    """(1, 3, h, w) fp32 with values in [-0.2, 1.2), 0 and 1 exactly, exact x.5 / 255 ties, NaN, +-inf and values beyond int32"""
    g = torch.Generator().manual_seed(seed)
    f = torch.rand(1, 3, h, w, generator=g) * 1.4 - 0.2
    flat = f.view(-1)
    special = torch.cat([torch.from_numpy(tie_values(64, seed)),
                         torch.tensor([0.0, 1.0, -0.0, 255.5 / 255, 0.5 / 255, -0.5 / 255, float('nan'), float('inf'), float('-inf'),
                                       3e7, -3e7, 1e30, -1e30, 2147483520 / 255, 2147483904 / 255])])
    idx = torch.randperm(flat.numel(), generator=g)[:special.numel()]
    flat[idx] = special[:idx.numel()]
    return f


def old_ssim_device(a, b, win=7):
    """the torch float64 SSIM the drop-in used before rv_region_metrics took its place (uniform 7x7 window, valid interior)"""
    a, b = a.double(), b.double()
    cov_norm = win * win / (win * win - 1.0)
    ux, uy = F.avg_pool2d(a, win, 1), F.avg_pool2d(b, win, 1)
    uxx, uyy, uxy = F.avg_pool2d(a * a, win, 1), F.avg_pool2d(b * b, win, 1), F.avg_pool2d(a * b, win, 1)
    vx, vy, vxy = cov_norm * (uxx - ux * ux), cov_norm * (uyy - uy * uy), cov_norm * (uxy - ux * uy)
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    S = ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux ** 2 + uy ** 2 + C1) * (vx + vy + C2))
    return float(S.mean(dim=(2, 3)).mean())


def ssim_pair(h, w, seed):
    """a ground truth in [0, 1] and a noisy, clamped output of it, as a network's output and its target"""
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(1, 3, h, w, generator=g)
    gt = F.avg_pool2d(F.pad(gt, (1, 1, 1, 1), mode='replicate'), 3, 1)        # some spatial structure
    out = (gt + 0.05 * torch.randn(1, 3, h, w, generator=g)).clamp(0, 1)
    return out.contiguous(), gt.contiguous()


# ---------------------------------------------------------------- CPU

@pytest.mark.parametrize('h,w', [(1080, 1920), (271, 483)])
def test_mean_ssim_is_the_interior_box_of_the_full_map(h, w):
    """skimage's mean SSIM = the full-frame SSIM map (rv_region_metrics' map, tests/region_metrics_oracle.py) summed over the
    box (3, H - 3, 3, W - 3) and the 3 channels, over 3 (H - 6)(W - 6)"""
    out, gt = ssim_pair(h, w, seed=h)
    _, s = RMO.region_metrics(out, gt, [(3, h - 3, 3, w - 3)])
    assert abs(s[0] / (3 * (h - 6) * (w - 6)) - skimage_ssim(hwc(out), hwc(gt))) <= 1e-12


# ---------------------------------------------------------------- GPU

def kernel_bytes(ops, frames):
    packed = ops.eval_images([f.cuda() for f in frames])
    torch.cuda.synchronize()
    return packed.cpu().numpy()


def assert_images_equal(got, frames):
    off = 0
    for k, f in enumerate(frames):
        want = reference_u8(f).reshape(-1)
        bad = np.flatnonzero(got[off:off + want.size] != want)
        assert bad.size == 0, f'frame {k}: {bad.size} bytes differ, first at {bad[0]}: {got[off + bad[0]]} vs {want[bad[0]]}'
        off += want.size
    assert off == got.size, (off, got.size)


@pytest.mark.gpu
@pytest.mark.parametrize('sizes', [[(1080, 1920)], [(4320, 7680)], [(271, 483)],
                                   [(270, 480), (1080, 1920), (1080, 1920)],       # input, output, gt of a x4 model
                                   [(271, 483), (1084, 1932), (17, 31)],           # odd sizes: unaligned images in dst
                                   [(1, 1), (2, 2), (1080, 1920)]])
def test_eval_images_bytes_match_opencv(cuda_ops, sizes):
    frames = [frame(h, w, seed=17 * k + h) for k, (h, w) in enumerate(sizes)]
    got = kernel_bytes(cuda_ops, frames)
    assert_images_equal(got, frames)
    assert np.array_equal(got, kernel_bytes(cuda_ops, frames)), 'two calls differ'


@pytest.mark.gpu
def test_eval_images_unaligned_frame(cuda_ops):
    """a frame that starts 4 bytes past a 16-byte boundary converts pixel by pixel to the same bytes"""
    f = frame(64, 96, seed=3).cuda()
    store = torch.empty(f.numel() + 1, device='cuda')
    view = store[1:].view(f.shape)
    view.copy_(f)
    got = cuda_ops.eval_images([view]).cpu().numpy()
    assert np.array_equal(got, kernel_bytes(cuda_ops, [f]))
    assert_images_equal(got, [f])


@pytest.mark.gpu
@pytest.mark.parametrize('h,w', [(270, 480), (271, 483)])
def test_eval_images_equal_conf_map_frames(cuda_ops, h, w):
    """rv_conf_map_images' input and output images come from the same conversion"""
    from refvsr_b200.colormap import inferno_lut
    inp, out = frame(h, w, seed=1).cuda(), frame(4 * h, 4 * w, seed=2).cuda()
    maps = [torch.rand(1, 1, h, w, device='cuda') for _ in range(4)]
    conf = cuda_ops.conf_map_images(maps, inp, out, inferno_lut('cuda'), True).cpu().numpy()
    ours = kernel_bytes(cuda_ops, [inp, out])
    assert np.array_equal(conf[4 * 3 * h * w:], ours)


@pytest.mark.gpu
def test_eval_images_rejects_bad_arguments(cuda_ops):
    import ctypes as C

    from refvsr_b200.lib import _ptr
    f = frame(16, 24, seed=1).cuda()
    bad = [
        [],                                          # no frame
        [f, f, f, f],                                # four frames
        [f.half()],                                  # not fp32
        [f.transpose(2, 3)],                         # not contiguous
        [f[:, :2].contiguous()],                     # two channels
        [f[0]],                                      # (3, H, W)
        [f.cpu()],                                   # host tensor
    ]
    for frames in bad:
        with pytest.raises(ValueError):
            cuda_ops.eval_images(frames)
    lib, s = cuda_ops.lib, cuda_ops._stream()
    buf = torch.empty(1 << 20, dtype=torch.uint8, device='cuda')

    def call(ptrs, hw, n, dst=buf):
        return lib.rv_eval_images((C.c_void_p * max(len(ptrs), 1))(*ptrs), (C.c_int * max(len(hw), 1))(*hw), n, _ptr(dst), s)

    p = f.data_ptr()
    assert call([p], [16, 24], 1) == 0
    assert call([p], [16, 24], 0) == -1                          # no frame
    assert call([p] * 4, [16, 24] * 4, 4) == -1                  # four frames
    assert call([p, None], [16, 24, 16, 24], 2) == -1            # null frame
    assert call([p], [0, 24], 1) == -1                           # empty
    assert call([p], [16, -1], 1) == -1
    assert call([p], [1 << 15, (1 << 13) + 1], 1) == -1          # more than 2^28 pixels
    assert lib.rv_eval_images(None, (C.c_int * 2)(16, 24), 1, _ptr(buf), s) == -1
    assert lib.rv_eval_images((C.c_void_p * 1)(p), None, 1, _ptr(buf), s) == -1
    assert lib.rv_eval_images((C.c_void_p * 1)(p), (C.c_int * 2)(16, 24), 1, None, s) == -1
    assert_images_equal(kernel_bytes(cuda_ops, [f]), [f])        # still usable


@pytest.mark.gpu
@pytest.mark.parametrize('h,w', [(1080, 1920), (271, 483)])
def test_mean_ssim_matches_skimage(cuda_ops, h, w):
    out, gt = ssim_pair(h, w, seed=w)
    got = cuda_ops.mean_ssim(out.cuda(), gt.cuda())
    want = skimage_ssim(hwc(out), hwc(gt))
    assert abs(got - want) <= 1e-12, (got, want)
    old = old_ssim_device(out.cuda(), gt.cuda())
    assert '{:.5f}'.format(got) == '{:.5f}'.format(old), (got, old)
    assert abs(got - old) <= 1e-12, (got, old)
    assert got == cuda_ops.mean_ssim(out.cuda(), gt.cuda()), 'two calls differ'


def run_qual_quan(ref, tmp, tag, config, dropin_loop, frame_num, extra=(), extra_env=None, timeout=1500):
    """run.py --eval_mode qual_quan on the H100 engine (the models drop-in in both arms) with the drop-in loop, or with the
    reference's (REFVSR_DROPIN_EVAL=0).  Returns (stdout, score file, {relative path: file})"""
    out = os.path.join(tmp, 'out_' + tag)
    pp = [ENV_DIR, os.path.join(ROOT, 'refvsr_b200', 'dropin'), ROOT, SHIMS]
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(pp), REFVSR_TEST_ENV='1', PYTHONDONTWRITEBYTECODE='1')
    if not dropin_loop:
        env['REFVSR_DROPIN_EVAL'] = '0'
    env.update(extra_env or {})
    args = ['--mode', 'qq_eval', '--project', os.path.join(tmp, 'logs_' + tag), '--config', config, '--data', 'RealMCVSR',
            '--ckpt_abs_name', os.path.join(tmp, 'ckpt.pytorch'), '--data_offset', os.path.join(tmp, 'data'),
            '--output_offset', out, '--frame_num', str(frame_num)] + list(extra)
    r = subprocess.run([sys.executable, '-B', 'run.py'] + args, cwd=ref, env=env, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, f'run.py ({tag}) failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}'
    assert 'All keys matched successfully' in r.stdout, r.stdout[-2000:]
    files = {re.sub(r'/\d{4}_\d{2}_\d{2}_\d{4}/', '/DATE/', os.path.relpath(os.path.join(d, f), out)): os.path.join(d, f)
             for d, _, fs in os.walk(out) for f in fs}
    scores = [p for k, p in files.items() if k.endswith('score_RealMCVSR_qual_quan.txt')]
    assert len(scores) == 1, sorted(files)
    return r.stdout, open(scores[0]).read(), files


@pytest.mark.gpu
@pytest.mark.parametrize('config,lr_hw,extra,prec', [
    ('config_RefVSR_MFID', (64, 96), (), 'bf16'),                                  # x4: 64x96 -> 256x384
    ('config_RefVSR_small_MFID_8K', (24, 32), ('--qualitative_only',), None),      # HD -> 8K: 96x128 -> 384x512
])
def test_run_py_qual_quan_reference_loop_vs_dropin_gpu(tmp_path, config, lr_hw, extra, prec):
    """run.py --eval_mode qual_quan twice on the H100 engine: with the reference's loop and with the drop-in.  Both run the
    engine's network, so every printed line and the score file are identical with the seconds masked, and every png and jpg
    is byte-identical"""
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    ref = _ref_root()
    if ref is None:
        pytest.skip('no reference checkout staged under oracle/_ref')
    tmp = str(tmp_path)
    make_tree(os.path.join(tmp, 'data'), *lr_hw, videos=2, frames=4)
    make_ckpt(os.path.join(tmp, 'ckpt.pytorch'), config)
    env = {'REFVSR_TEST_PRECISION': prec} if prec else {}
    frame_num = 3 if '8K' in config else 7
    base, base_score, base_files = run_qual_quan(ref, tmp, 'ref', config, False, frame_num, extra, env)
    ours, ours_score, ours_files = run_qual_quan(ref, tmp, 'b200', config, True, frame_num, extra, env)
    assert loop_lines(base) == loop_lines(ours)
    assert loop_lines(base_score) == loop_lines(ours_score)
    assert len(re.findall(r'^\[EVAL ', base_score, re.M)) == 8
    if not extra:
        assert base_score.count('[MEAN EVAL') == 1 and '[TOTAL' in base_score
        assert all(float(v) != 0 for v in re.findall(r'^\[EVAL [^\n]* SSIM: ([-\d.]+)', base_score, re.M)), base_score
    assert set(base_files) == set(ours_files), sorted(set(base_files) ^ set(ours_files))[:8]
    images = sorted(k for k in base_files if k.endswith(('.png', '.jpg')))
    assert len(images) == 2 * 2 * 8, len(images)                  # input and output, png and jpg, per frame
    for k in images:
        with open(base_files[k], 'rb') as fa, open(ours_files[k], 'rb') as fb:
            assert fa.read() == fb.read(), k
    import cv2
    scale = 16 if '8K' in config else 4
    outs = [k for k in images if '/output/' in k and k.endswith('.png')]
    img = cv2.imread(base_files[outs[0]])
    assert img.shape == (scale * lr_hw[0], scale * lr_hw[1], 3) and img.std() > 1, (img.shape, outs[0])
