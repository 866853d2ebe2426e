"""`eval_qual_quan(config)` - drop-in for evaluation/eval_qual_quan.py:17-144 with the same inputs, printed lines, score file and
image tree, re-organised so that the host loop no longer caps a fast network at ~1 frame/s:

  reference (per frame)                                              here
  ------------------------------------------------------------------ ----------------------------------------------------
  gc.collect() + torch.cuda.empty_cache()      (:59-60)              dropped (the engine allocates nothing per call)
  output.cpu().numpy(), gt.cpu().numpy()       (:76-79, sync D2H)    pinned host buffers, non-blocking copies + an event
  SSIM by skimage on the CPU, 1080p, 3 channels (:92, ~1 s)          same formula (uniform 7x7 window, sample covariance, valid
                                                                     interior, mean over channels) in float64 on the device
  6 x cv2.imwrite (png + jpg of input / output / gt) (:103-125)      same files, written by a small thread pool after the
                                                                     frame's D2H event; the loop never waits for the encoder
  errs['PSNR'].item() right after the forward  (:84)                 read together with the SSIM value, one sync per frame

`REFVSR_DROPIN_EVAL=0` restores the reference's own loop (A/B measurements).  flag_HD_in (8K) models keep the reference's CPU SSIM
on the cv2-resized output (:86-89) - that path is rarely evaluated quantitatively and is kept bit-compatible instead."""
import importlib.util
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import cv2
import numpy as np
import torch
import torch.nn.functional as F

from . import REFERENCE_DIR
from .init import init
from .metrics import ssim as ssim_cpu


def _reference_impl():
    spec = importlib.util.spec_from_file_location('evaluation._reference_eval_qual_quan', os.path.join(REFERENCE_DIR, 'eval_qual_quan.py'),
                                                  submodule_search_locations=None)
    mod = importlib.util.module_from_spec(spec)
    mod.__package__ = 'evaluation'
    spec.loader.exec_module(mod)
    return mod.eval_qual_quan


def ssim_device(a, b, data_range=1.0, win=7):
    """skimage.metrics.structural_similarity(a, b, data_range=1.0, multichannel=True) for (1, 3, H, W) tensors in [0, 1]:
    uniform win x win filter, sample covariance (NP / (NP - 1)), mean over the valid interior and the channels; float64."""
    a, b = a.double(), b.double()
    K1, K2 = 0.01, 0.03
    NP = win * win
    cov_norm = NP / (NP - 1.0)
    ux, uy = F.avg_pool2d(a, win, 1), F.avg_pool2d(b, win, 1)             # = the valid interior of the uniform filter
    uxx, uyy, uxy = F.avg_pool2d(a * a, win, 1), F.avg_pool2d(b * b, win, 1), F.avg_pool2d(a * b, win, 1)
    vx, vy, vxy = cov_norm * (uxx - ux * ux), cov_norm * (uyy - uy * uy), cov_norm * (uxy - ux * uy)
    C1, C2 = (K1 * data_range) ** 2, (K2 * data_range) ** 2
    S = ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux ** 2 + uy ** 2 + C1) * (vx + vy + C2))
    return S.mean(dim=(2, 3)).mean()


def _write_images(job):
    ev, arrays, paths = job
    if ev is not None:
        ev.synchronize()
    for arr, path in zip(arrays, paths):
        for p in path:
            Path(os.path.dirname(p)).mkdir(parents=True, exist_ok=True)
            cv2.imwrite(p, cv2.cvtColor(arr * 255, cv2.COLOR_RGB2BGR))


def eval_qual_quan(config):
    if os.environ.get('REFVSR_DROPIN_EVAL', '1') == '0':
        return _reference_impl()(config)
    mode = config.EVAL.eval_mode
    network, model, save_path_root_deblur, save_path_root_deblur_score, ckpt_name = init(config, mode)
    score_path = os.path.join(save_path_root_deblur_score, 'score_{}_{}.txt'.format(config.EVAL.data, config.EVAL.eval_mode))
    total_norm = 0
    total_itr_time = PSNR_mean_total = SSIM_mean_total = 0
    total_itr_time_video = PSNR_mean = SSIM_mean = 0
    frame_len_prev = 0
    pool = ThreadPoolExecutor(max_workers=int(os.environ.get('REFVSR_EVAL_WRITERS', '4')))
    pending = []
    cuda = torch.cuda.is_available() and getattr(config, 'cuda', False)
    ring = {}                                             # pinned host buffers, two per image kind (frame k-1 may still be encoding)

    def to_host(t, key, k):
        """(1, 3, H, W) device tensor -> (H, W, 3) float32 numpy view of a pinned buffer (async), or a plain copy on CPU"""
        hwc = t[0].permute(1, 2, 0)
        if not cuda:
            return hwc.float().cpu().numpy().copy()
        slot = (key, k % 3, tuple(hwc.shape))
        if slot not in ring:
            ring[slot] = torch.empty(tuple(hwc.shape), dtype=torch.float32).pin_memory()
        ring[slot].copy_(hwc, non_blocking=True)
        return ring[slot].numpy()

    for i, inputs in enumerate(model.data_loader_eval):
        is_first_frame = inputs['is_first'][0].item()
        if 'is_continue' in inputs.keys() and inputs['is_continue'][0].item():
            print('passing, video', inputs['video_name'][0])
            frame_len_prev += 1
            continue
        if is_first_frame:
            if i > 0:
                PSNR_mean_total = PSNR_mean_total + PSNR_mean
                SSIM_mean_total = SSIM_mean_total + SSIM_mean
                total_itr_time = total_itr_time + total_itr_time_video
                PSNR_mean = PSNR_mean / frame_len_prev
                SSIM_mean = SSIM_mean / frame_len_prev
                total_itr_time_video = total_itr_time_video / frame_len_prev
                line = '[MEAN EVAL {}|{}|{}][{}/{}] PSNR: {:.5f} SSIM: {:.5f} ({:.5f}sec)\n\n'.format(
                    config.mode, config.EVAL.data, inputs['video_name'][0], inputs['video_idx'][0], inputs['video_len'][0], PSNR_mean,
                    SSIM_mean, total_itr_time_video)
                print(line, end='')
                if not config.EVAL.qualitative_only:
                    with open(score_path, 'a') as file:
                        file.write(line)
            total_itr_time_video = PSNR_mean = SSIM_mean = 0

        init_time = time.time()
        with torch.no_grad():
            results = model.evaluation(inputs, is_PSNR=not config.EVAL.qualitative_only)
            errs, outs = results['errs'], results['vis']
            try:
                inp, output = outs['LR_UW_png'], outs['SR_UW_png']
            except Exception:                                               # noqa: BLE001  (the reference's own fallback, :70-74)
                inp, output = outs['LR_UW'], outs['SR_UW']
            gt = outs['HR_UW']
            PSNR = SSIM = 0
            ssim_t = None
            if not config.EVAL.qualitative_only and ('SR_UW_png' in outs.keys() or 'SR_UW' in outs.keys()):
                if not config.flag_HD_in:
                    ssim_t = ssim_device(output.float(), gt.float())
        want_images = not config.EVAL.quantitative_only
        out_np = gt_np = inp_np = None
        ev = None
        if want_images or (config.flag_HD_in and not config.EVAL.qualitative_only):
            out_np = to_host(output.float(), 'out', i)
            gt_np = to_host(gt.float(), 'gt', i)
            if want_images and config.EVAL.is_gradio is False:
                inp_np = to_host(inp.float(), 'inp', i)
            if cuda:
                ev = torch.cuda.Event()
                ev.record()
        if not config.EVAL.qualitative_only and ('SR_UW_png' in outs.keys() or 'SR_UW' in outs.keys()):
            PSNR = errs['PSNR'].item()                                        # the frame's one host sync
            if ssim_t is not None:
                SSIM = float(ssim_t.item())
            else:                                                             # flag_HD_in: the reference's CPU path (:86-92)
                if ev is not None:
                    ev.synchronize()
                o_ = cv2.resize(out_np, dsize=(0, 0), fx=1 / config.scale, fy=1 / config.scale, interpolation=cv2.INTER_CUBIC)
                SSIM = ssim_cpu(o_, gt_np)
        elif cuda:
            torch.cuda.current_stream().synchronize()
        itr_time = time.time() - init_time

        PSNR_mean = PSNR_mean + PSNR
        SSIM_mean = SSIM_mean + SSIM
        frame_name = inputs['frame_name'][0]
        line = '[EVAL {}|{}|{}][{}/{}][{}/{}] {} PSNR: {:.5f} SSIM: {:.5f} ({:.5f}sec)'.format(
            config.mode, config.EVAL.data, inputs['video_name'][0], inputs['video_idx'][0] + 1, inputs['video_len'][0],
            inputs['frame_idx'][0] + 1, inputs['frame_len'][0], frame_name, PSNR, SSIM, itr_time)
        print(line)
        with open(score_path, 'w' if (i == 0) else 'a') as file:
            file.write(line + '\n')

        if want_images:
            frame_name_no_ext = frame_name.split('.')[0]
            vid = inputs['video_name'][0]
            if config.EVAL.is_gradio is False:
                arrays, paths = [inp_np, out_np], [[], []]
                if 'gt' in inputs.keys():
                    arrays.append(gt_np)
                    paths.append([])
                for iformat in ['png', 'jpg']:
                    root = os.path.join(save_path_root_deblur, iformat)
                    paths[0].append(os.path.join(root, 'input', vid, '{}.{}'.format(frame_name_no_ext, iformat)))
                    paths[1].append(os.path.join(root, 'output', vid, '{}.{}'.format(frame_name_no_ext, iformat)))
                    if 'gt' in inputs.keys():
                        paths[2].append(os.path.join(root, 'gt', vid, '{}.{}'.format(frame_name_no_ext, iformat)))
            else:
                arrays, paths = [out_np], [[os.path.join(save_path_root_deblur, '{}.png'.format(frame_name_no_ext))]]
            pending.append(pool.submit(_write_images, (ev, arrays, paths)))
            while len(pending) > 2:                       # a pinned slot is reused every third frame: keep the queue short
                pending.pop(0).result()

        total_itr_time_video = total_itr_time_video + itr_time
        total_norm = total_norm + 1
        frame_len_prev = inputs['frame_len'][0]

    for f in pending:
        f.result()
    pool.shutdown()
    total_itr_time = (total_itr_time + total_itr_time_video) / total_norm
    PSNR_mean_total = (PSNR_mean_total + PSNR_mean) / total_norm
    SSIM_mean_total = (SSIM_mean_total + SSIM_mean) / total_norm
    sys.stdout.write('\n[TOTAL {}|{}] PSNR: {:.5f}  SSIM: {:.5f} ({:.5f}sec)\n'.format(ckpt_name, config.EVAL.data, PSNR_mean_total,
                                                                                   SSIM_mean_total, total_itr_time))
    if not config.EVAL.qualitative_only:
        with open(score_path, 'a') as file:
            file.write('\n[TOTAL {}|{}] PSNR: {:.5f} SSIM: {:.5f} ({:.5f}sec)\n'.format(ckpt_name, config.EVAL.data, PSNR_mean_total,
                                                                                    SSIM_mean_total, total_itr_time))
