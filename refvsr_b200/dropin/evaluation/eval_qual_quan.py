"""`eval_qual_quan(config)` - drop-in for evaluation/eval_qual_quan.py:17-144 with the same inputs, printed lines, score file and
image tree, re-organised so that the host loop no longer caps a fast network at ~1 frame/s:

  reference (per frame)                                              here
  ------------------------------------------------------------------ ----------------------------------------------------
  gc.collect() + torch.cuda.empty_cache()      (:59-60)              dropped (the engine allocates nothing per call)
  output / gt / inp .cpu().numpy() as float32  (:76-79, :95)         one rv_eval_images call turns the frames to be written
  and cv2.cvtColor(x * 255, RGB2BGR) per write (:103-125)            into the uint8 BGR images cv2.imwrite stores for them; one
                                                                     non-blocking copy moves those bytes into pinned memory
  SSIM by skimage on the CPU, 1080p, 3 channels (:92, ~1 s)          one rv_region_metrics call: skimage's full-frame SSIM map
                                                                     summed over the interior it averages (3 pixels in from
                                                                     every edge) and the 3 channels
  6 x cv2.imwrite (png + jpg of input / output / gt) (:103-125)      same files, written by a small thread pool after the
                                                                     frame's copy event; the loop never waits for the encoder
  errs['PSNR'].item() right after the forward  (:84)                 read after the SSIM sums, one sync per frame

Every written image takes the device path: input / output / gt in png and jpg, the gradio branch's single png, and the
flag_HD_in (HD -> 8K) models' 4320x7680 outputs, whose 8-bit image is a quarter of the float32 frame.  Without CUDA (`-cpu`) the
frames are copied back as float32, scored by the reference's `ssim` and written as the reference writes them.

flag_HD_in models keep the reference's quantitative branch (:86-89, the CPU SSIM of the cv2-resized output), but the reference's
own Trainer.evaluation cannot compute their PSNR: it subtracts the 1080p ground truth from the 8K output, which does not broadcast.
These models run with --qualitative_only, as the reference's scripts_eval/eval_*8K.sh do.

`REFVSR_DROPIN_EVAL=0` restores the reference's own loop (A/B measurements)."""
import importlib.util
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import cv2
import numpy as np
import torch

from refvsr_b200 import lib as rv_lib

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


def split_images(buf, hws):
    """(H, W, 3) views of a packed rv_eval_images or rv_conf_map_images buffer (flat uint8 numpy array), one per (H, W)"""
    views, off = [], 0
    for h, w in hws:
        views.append(buf[off:off + 3 * h * w].reshape(h, w, 3))
        off += 3 * h * w
    return views


def _host_float(t):
    """(1, 3, H, W) tensor -> (H, W, 3) float32 numpy array, as the reference copies a frame back"""
    return t[0].permute(1, 2, 0).float().cpu().numpy().copy()


def _write_images(job):
    """(event, arrays, paths): after the event, write each array to each of its paths; float arrays are RGB in [0, 1] and
    written as the reference writes them, uint8 arrays are BGR images written as they are"""
    ev, arrays, paths = job
    if ev is not None:
        ev.synchronize()
    for arr, path in zip(arrays, paths):
        img = arr if arr.dtype == np.uint8 else cv2.cvtColor(arr * 255, cv2.COLOR_RGB2BGR)
        for p in path:
            Path(os.path.dirname(p)).mkdir(parents=True, exist_ok=True)
            cv2.imwrite(p, img)


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
    ops = rv_lib.CudaOps() if cuda else None
    ring = {}                                             # pinned host buffers, three per size (two frames may still be encoding)

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
                print(line)
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
        want_images = not config.EVAL.quantitative_only
        has_gt_images = 'gt' in inputs.keys()
        arrays = ev = None
        if want_images:                                   # the frames written, in the order of their paths below
            frames = [inp, output] + ([gt] if has_gt_images else []) if config.EVAL.is_gradio is False else [output]
            if cuda:
                frames = [f.float().contiguous() for f in frames]
                packed = ops.eval_images(frames)
                slot = (total_norm % 3, packed.numel())
                if slot not in ring:
                    ring[slot] = torch.empty(packed.numel(), dtype=torch.uint8).pin_memory()
                ring[slot].copy_(packed, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record()
                arrays = split_images(ring[slot].numpy(), [tuple(f.shape[2:]) for f in frames])
            else:
                arrays = [_host_float(f) for f in frames]
        PSNR = SSIM = 0
        if not config.EVAL.qualitative_only and ('SR_UW_png' in outs.keys() or 'SR_UW' in outs.keys()):
            if config.flag_HD_in:                                             # the reference's CPU path (:86-92)
                o_ = cv2.resize(_host_float(output), dsize=(0, 0), fx=1 / config.scale, fy=1 / config.scale,
                                interpolation=cv2.INTER_CUBIC)
                SSIM = ssim_cpu(o_, _host_float(gt))
            elif cuda:
                SSIM = ops.mean_ssim(output.float().contiguous(), gt.float().contiguous())   # the frame's one host sync
            else:
                SSIM = ssim_cpu(_host_float(output), _host_float(gt))
            PSNR = errs['PSNR'].item()
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
                dirs = ['input', 'output'] + (['gt'] if has_gt_images else [])
                paths = [[os.path.join(save_path_root_deblur, iformat, d, vid, '{}.{}'.format(frame_name_no_ext, iformat))
                          for iformat in ('png', 'jpg')] for d in dirs]
            else:
                paths = [[os.path.join(save_path_root_deblur, '{}.png'.format(frame_name_no_ext))]]
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
