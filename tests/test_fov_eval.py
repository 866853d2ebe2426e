"""The FOV evaluation mode (`run.py --eval_mode FOV`, evaluation/eval_quan_FOV.py) on rv_region_metrics: the drop-in's boxes
against the reference's masks, its per-frame scores against the reference's metric functions, the kernel against the fp64
yardstick (tests/region_metrics_oracle.py), and run.py's printed numbers with and without the drop-in."""
import importlib.util
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, 'tests')
sys.path.insert(0, ROOT)
sys.path.insert(0, TESTS)

import region_metrics_oracle as RO                                           # noqa: E402
from refvsr_b200.fov import FULL, INTERIOR, KEYS, METRICS, crop_ratio, fov_boxes, fov_regions, score_frame   # noqa: E402
from test_dropin_runpy import ENV_DIR, SHIMS, _ref_root, make_ckpt, make_tree                            # noqa: E402


def reference_masks(h, w, key):
    """mask_fi, mask_fo, mask_fr of one key as evaluation/eval_quan_FOV.py:158-188 builds them (None: not built for the key)"""
    like = np.zeros((h, w, 3), np.float32)
    mask_fo = None
    if key == 1.:
        mask_fi = np.ones_like(like)
    else:
        r = int(1 / ((1 - key) / 2))
        mask_fi = np.zeros_like(like)
        mask_fi[h // r:h - h // r, w // r:w - w // r] = 1.
        mask_fo = np.ones_like(like)
        mask_fo[h // r:h - h // r, w // r:w - w // r] = 0.
    mask_fr = None
    if key > 0.5:
        mask_fr = mask_fi.copy()
        mask_fr[h // 4:h - h // 4, w // 4:w - w // 4] = 0.
    return mask_fi, mask_fo, mask_fr


def indicator(boxes, h, w, plus, minus):
    m = np.zeros((h, w, 3), np.float32)
    y0, y1, x0, x1 = boxes[plus]
    m[y0:y1, x0:x1] = 1.
    if minus is not None:
        y0, y1, x0, x1 = boxes[minus]
        m[y0:y1, x0:x1] = 0.
    return m


def load_reference_metrics():
    """the reference's evaluation/metrics.py, with the tests' skimage stand-in (tests/runpy_env) first on sys.path"""
    ref = _ref_root()
    if ref is None:
        pytest.skip('no reference checkout')
    sys.path.insert(0, ENV_DIR)
    try:
        spec = importlib.util.spec_from_file_location('_reference_eval_metrics', os.path.join(ref, 'evaluation', 'metrics.py'))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        sys.path.remove(ENV_DIR)
    return mod


def reference_scores(M, out, gt):
    """key -> the six metrics (METRICS order) of one frame, (h, w, 3) float32 arrays, as eval_quan_FOV.py:156-195 computes them"""
    h, w, _ = out.shape
    res = {}
    with np.errstate(divide='ignore', invalid='ignore'):
        for key in KEYS:
            fi, fo, fr = reference_masks(h, w, key)
            if key == 1.:
                p_fi, s_fi, p_fo, s_fo = M.psnr(out, gt), M.ssim(out, gt), 0, 0
            else:
                p_fi, s_fi = M.psnr_masked(out, gt, fi), M.ssim_masked(out, gt, fi)
                p_fo, s_fo = M.psnr_masked(out, gt, fo), M.ssim_masked(out, gt, fo)
            p_fr, s_fr = (M.psnr_masked(out, gt, fr), M.ssim_masked(out, gt, fr)) if key > 0.5 else (0, 0)
            res[key] = (p_fi, p_fo, p_fr, s_fi, s_fo, s_fr)
    return res


def assert_scores_close(ours, ref, psnr_tol, ssim_tol):
    for key in KEYS:
        for name, a, b in zip(METRICS, ours[key], ref[key]):
            a, b = float(a), float(b)
            tol = psnr_tol if name.startswith('PSNR') else ssim_tol
            if math.isnan(b) or math.isinf(b):
                assert (math.isnan(a) and math.isnan(b)) or a == b, (key, name, a, b)
            else:
                assert abs(a - b) <= tol, (key, name, a, b)


def frame_pair(h, w, seed, noise=0.05):
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(1, 3, h, w, generator=g)
    gt = torch.nn.functional.avg_pool2d(torch.nn.functional.pad(gt, (1, 1, 1, 1), mode='replicate'), 3, 1)   # some structure
    out = (gt + noise * torch.randn(1, 3, h, w, generator=g)).clamp(0, 1)
    return out.contiguous(), gt.contiguous()


def hwc(t):
    return t[0].permute(1, 2, 0).contiguous().numpy()


class _Oracle:
    region_metrics = staticmethod(RO.region_metrics)


# ---------------------------------------------------------------- CPU

def test_crop_ratios_are_the_references():
    assert [crop_ratio(k) for k in KEYS[1:]] == [20, 10, 6, 5, 4]


@pytest.mark.parametrize('h,w', [(1080, 1920), (271, 483), (96, 128), (12, 19)])
def test_boxes_match_reference_masks(h, w):
    boxes = fov_boxes(h, w)
    assert len(boxes) == 7
    for key in KEYS:
        fi, fo, fr = reference_masks(h, w, key)
        reg = fov_regions(key)
        assert np.array_equal(indicator(boxes, h, w, *reg['PSNR_fi']), fi) and reg['SSIM_fi'] == (reg['PSNR_fi'] if key != 1 else (INTERIOR, None))
        if fo is None:
            assert 'PSNR_fo' not in reg and 'SSIM_fo' not in reg
        else:
            assert np.array_equal(indicator(boxes, h, w, *reg['PSNR_fo']), fo) and reg['SSIM_fo'] == reg['PSNR_fo']
        if fr is None:
            assert 'PSNR_fr' not in reg and 'SSIM_fr' not in reg
        else:
            assert np.array_equal(indicator(boxes, h, w, *reg['PSNR_fr']), fr) and reg['SSIM_fr'] == reg['PSNR_fr']
    # key 1's SSIM inside is skimage's mean over the valid interior of the map (metrics.py:15-16)
    interior = np.zeros((h, w, 3), np.float32)
    interior[3:-3, 3:-3] = 1.
    assert np.array_equal(indicator(boxes, h, w, INTERIOR, None), interior)
    assert boxes[FULL] == (0, h, 0, w)


@pytest.mark.parametrize('h,w,case', [(96, 128, 'random'), (12, 19, 'random'), (24, 32, 'equal')])
def test_frame_scores_match_reference_metrics(h, w, case):
    """per-frame assembly on the fp64 yardstick vs the reference's metric functions: 12x19 has an empty region (key 0.9's
    outside: nan), a frame equal to its ground truth has zero error (inf)"""
    M = load_reference_metrics()
    out, gt = frame_pair(h, w, seed=h * w)
    if case == 'equal':
        out = gt.clone()
    ours = score_frame(_Oracle(), out, gt)
    ref = reference_scores(M, hwc(out), hwc(gt))
    assert_scores_close(ours, ref, psnr_tol=1e-4, ssim_tol=1e-9)
    flat = [float(v) for key in KEYS for v in ours[key]]
    if (h, w) == (12, 19):
        assert math.isnan(ours[0.9][1]) and math.isnan(ours[0.9][4])
    if case == 'equal':
        assert ours[1][0] == float('inf') and ours[1][3] == 1.0
    assert [math.isnan(v) for v in flat] == [math.isnan(float(v)) for key in KEYS for v in ref[key]]


_NUM = r'(-?(?:\d+\.\d+|nan|inf))'


def printed_numbers(log):
    """[(kind, value)] of every number run.py's FOV loop prints: per-frame PSNR / SSIM, then each block row's entries"""
    out = []
    for line in log.splitlines():
        m = re.match(r'\[EVAL [^\]]*\]\[\d+/\d+\]\[\d+/\d+\] \S+ PSNR: ' + _NUM + ' SSIM: ' + _NUM, line)
        if m:
            out += [('PSNR', float(m.group(1))), ('SSIM', float(m.group(2)))]
            continue
        m = re.match(r'\[(PSNR|SSIM)-FOV_(?:in  |out |ring)\] \((.*)\)', line)
        if m:
            out += [(m.group(1), float(v)) for v in re.findall(r'%: ' + _NUM + ',', m.group(2))]
    return out


LAUNCH_WITH_ORACLE = ('import sys, runpy; sys.path.insert(0, {tests!r}); import region_metrics_oracle as m; '
                      'sys.path.remove({tests!r}); m.install(); sys.argv[0] = "run.py"; runpy.run_path("run.py", run_name="__main__")')


def run_fov(ref, tmp, tag, config, dropin, cpu, frame_num=3, extra_env=None, oracle=False, timeout=1500):
    out = os.path.join(tmp, 'out_' + tag)
    pp = [ENV_DIR] + ([os.path.join(ROOT, 'refvsr_b200', 'dropin'), ROOT] if dropin else [ROOT]) + [SHIMS]
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(pp), REFVSR_TEST_ENV='1', PYTHONDONTWRITEBYTECODE='1')
    env.update(extra_env or {})
    args = ['--mode', 'fov_' + tag, '--project', os.path.join(tmp, 'logs_' + tag), '--config', config, '--data', 'RealMCVSR',
            '--ckpt_abs_name', os.path.join(tmp, 'ckpt.pytorch'), '--data_offset', os.path.join(tmp, 'data'),
            '--output_offset', out, '--frame_num', str(frame_num), '--eval_mode', 'FOV'] + (['-cpu'] if cpu else [])
    launch = ['-c', LAUNCH_WITH_ORACLE.format(tests=TESTS)] if oracle else ['run.py']
    r = subprocess.run([sys.executable, '-B'] + launch + args, cwd=ref, env=env, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, f'run.py ({tag}) failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}'
    assert 'All keys matched successfully' in r.stdout, r.stdout[-2000:]
    scores = [os.path.join(d, f) for d, _, fs in os.walk(out) for f in fs if f == 'score_RealMCVSR_FOV.txt']
    assert len(scores) == 1, scores
    return r.stdout, open(scores[0]).read()


def masked(text):
    """a printed block with its numbers and run-specific names blanked: the layout the two loops must share"""
    return re.sub(r'fov_(ref|b200)', 'MODE', re.sub(_NUM, '#', text))


def compare_runs(base, ours, psnr_tol, ssim_tol):
    a, b = printed_numbers(base), printed_numbers(ours)
    assert len(a) == len(b) and [k for k, _ in a] == [k for k, _ in b], (len(a), len(b))
    for (kind, x), (_, y) in zip(a, b):
        if math.isnan(x) or math.isinf(x):
            assert (math.isnan(x) and math.isnan(y)) or x == y, (kind, x, y)
        else:
            assert abs(x - y) <= (psnr_tol if kind == 'PSNR' else ssim_tol), (kind, x, y)
    return a


def test_run_py_fov_unmodified_vs_dropin_cpu(tmp_path):
    ref = _ref_root()
    if ref is None:
        pytest.skip('no reference checkout')
    tmp = str(tmp_path)
    make_tree(os.path.join(tmp, 'data'), 24, 32)
    make_ckpt(os.path.join(tmp, 'ckpt.pytorch'), 'config_RefVSR_small_L1')
    base, base_file = run_fov(ref, tmp, 'ref', 'config_RefVSR_small_L1', dropin=False, cpu=True)
    ours, ours_file = run_fov(ref, tmp, 'b200', 'config_RefVSR_small_L1', dropin=True, cpu=True, oracle=True,
                              extra_env={'REFVSR_TEST_ORACLE_OPS': '1'})
    nums = compare_runs(base, ours, psnr_tol=1e-4, ssim_tol=1e-5)
    # 6 frames x 2, then the first video's MEAN EVAL block (printed when the second starts) and the TOTAL block, 6 rows x 6 keys
    assert len(nums) == 6 * 2 + 2 * 36, len(nums)
    compare_runs(base_file, ours_file, psnr_tol=1e-4, ssim_tol=1e-5)
    assert masked(base_file) == masked(ours_file)


# ---------------------------------------------------------------- GPU

def _kernel_boxes(H, W):
    """overlapping, nested, empty and one-pixel boxes (8 at most)"""
    boxes = [(0, H // 2 + 1, 0, W // 2 + 1), (H // 3, H, W // 3, W), (0, H, 0, W), (3, H - 3, 3, W - 3),
             (2, 2, 0, W), (0, H, 5, 5), (H - 1, H, W - 1, W)]
    if H >= 20 and W >= 20:
        boxes.append(fov_boxes(H, W)[1])
    return boxes


@pytest.mark.gpu
@pytest.mark.parametrize('H,W', [(1080, 1920), (271, 483), (7, 7), (8, 1921)])
def test_region_metrics_kernel_vs_fp64(cuda_ops, H, W):
    out, gt = frame_pair(H, W, seed=H + W)
    for boxes in (_kernel_boxes(H, W), fov_boxes(H, W)):
        sq0, s0 = RO.region_metrics(out, gt, boxes)
        a, b = out.cuda(), gt.cuda()
        sq1, s1 = cuda_ops.region_metrics(a, b, boxes)
        sq2, s2 = cuda_ops.region_metrics(a, b, boxes)
        np.testing.assert_allclose(sq1, sq0, rtol=1e-12, atol=0)
        np.testing.assert_allclose(s1, s0, rtol=1e-12, atol=0)
        assert sq1.tobytes() == sq2.tobytes() and s1.tobytes() == s2.tobytes(), 'two calls differ'


@pytest.mark.gpu
def test_region_metrics_rejects_bad_arguments(cuda_ops):
    a, b = (t.cuda() for t in frame_pair(16, 16, seed=1))
    with pytest.raises(ValueError):
        cuda_ops.region_metrics(a[:, :, :6].contiguous(), b[:, :, :6].contiguous(), [(0, 6, 0, 16)])     # H < 7
    with pytest.raises(ValueError):
        cuda_ops.region_metrics(a, b, [(0, 17, 0, 16)])                                               # box outside the frame
    with pytest.raises(ValueError):
        cuda_ops.region_metrics(a, b, [(0, 16, 0, 16)] * 9)                                           # nbox = 9
    with pytest.raises(ValueError):
        cuda_ops.region_metrics(a.half(), b.half(), [(0, 16, 0, 16)])                                 # not fp32
    with pytest.raises(ValueError):
        cuda_ops.region_metrics(a.transpose(2, 3), b.transpose(2, 3), [(0, 16, 0, 16)])               # not contiguous
    sq, s = cuda_ops.region_metrics(a, b, [(0, 16, 0, 16)])                                            # still usable
    assert sq.shape == s.shape == (1,) and sq[0] > 0


@pytest.mark.gpu
def test_flag_hd_in_frame_path_gpu(cuda_ops):
    """the flag_HD_in branch: a 4x-size output is cv2-resized on the host as the reference does, then scored on the GPU"""
    M = load_reference_metrics()
    import cv2
    out, gt = frame_pair(64, 96, seed=7)
    big = torch.nn.functional.interpolate(out, scale_factor=4, mode='bicubic', align_corners=False).clamp(0, 1).contiguous()
    ours = score_frame(cuda_ops, big.cuda(), gt.cuda(), hd_scale=4)
    big_cpu = big.numpy()[0].transpose(1, 2, 0)
    resized = cv2.resize(big_cpu, dsize=(0, 0), fx=1 / 4, fy=1 / 4, interpolation=cv2.INTER_CUBIC)
    assert_scores_close(ours, reference_scores(M, resized, hwc(gt)), psnr_tol=1e-4, ssim_tol=1e-6)


@pytest.mark.gpu
def test_run_py_fov_on_engine_gpu(tmp_path):
    """run.py --eval_mode FOV with the drop-ins on the H100 engine (RefVSR_MFID, bf16) against the unmodified reference in eager
    PyTorch on the same GPU: every printed PSNR within 0.01 dB"""
    ref = _ref_root()
    if ref is None:
        pytest.skip('no reference checkout staged under oracle/_ref')
    tmp = str(tmp_path)
    make_tree(os.path.join(tmp, 'data'), 64, 96, videos=2, frames=4)
    make_ckpt(os.path.join(tmp, 'ckpt.pytorch'), 'config_RefVSR_MFID')
    base, _ = run_fov(ref, tmp, 'ref', 'config_RefVSR_MFID', dropin=False, cpu=False, frame_num=7)
    ours, _ = run_fov(ref, tmp, 'b200', 'config_RefVSR_MFID', dropin=True, cpu=False, frame_num=7,
                      extra_env={'REFVSR_TEST_PRECISION': 'bf16'})
    a, b = printed_numbers(base), printed_numbers(ours)
    assert len(a) == len(b) == 8 * 2 + 2 * 36 and [k for k, _ in a] == [k for k, _ in b]
    worst = max(abs(x - y) for (k, x), (_, y) in zip(a, b) if k == 'PSNR')
    print(f'FOV: max |dPSNR| vs the unmodified reference on the same GPU = {worst:.5f} dB over {sum(k == "PSNR" for k, _ in a)} numbers')
    assert worst < 0.01, (a, b)
