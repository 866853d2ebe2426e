"""`eval_quan_FOV(config)` - drop-in for evaluation/eval_quan_FOV.py:17-228 (`run.py --eval_mode FOV`) with the same printed lines
and the same score file.

Per frame the reference copies both frames to the host and computes 16 full-frame SSIM maps there (`ssim` once, `ssim_masked`
15 times, each recomputing the whole map before masking it) and 16 masked PSNRs over as many full-size masks.  Every mask is a
union or difference of centred boxes (refvsr_b200/fov.py), so here one `rv_region_metrics` call on the GPU sums the squared
error and the SSIM map over the frame's 7 boxes, and the host forms all 36 numbers from those 14 sums.  flag_HD_in (8K) models:
the output is copied to the host and cv2-resized exactly as the reference does (:146-149), and the resized frame is scored the
same way.  The printed seconds time `model.evaluation` alone, as the reference's do.

`REFVSR_DROPIN_EVAL=0` runs the reference's own loop."""
import importlib.util
import os
import sys
import time

from refvsr_b200 import lib as rv_lib
from refvsr_b200.fov import KEYS, METRICS, score_frame

from . import REFERENCE_DIR
from .init import init

# the six rows of a MEAN EVAL / TOTAL block: (label, METRICS index, entry format of one key: {0} = smallest key, {1} = key, in %)
_ROWS = (('PSNR-FOV_in  ', 0, '0-{1:3.1f}%: {2:.5f}, '), ('PSNR-FOV_out ', 1, '{1:3.1f}-100%: {2:.5f}, '),
         ('PSNR-FOV_ring', 2, '{0:3.1f}-{1:3.1f}%: {2:.5f}, '), ('SSIM-FOV_in  ', 3, '0-{1:3.1f}%: {2:.5f}, '),
         ('SSIM-FOV_out ', 4, '{1:3.1f}-100%: {2:.5f}, '), ('SSIM-FOV_ring', 5, '{0:3.1f}-{1:3.1f}%: {2:.5f}, '))


def _reference_impl():
    spec = importlib.util.spec_from_file_location('evaluation._reference_eval_quan_FOV', os.path.join(REFERENCE_DIR, 'eval_quan_FOV.py'),
                                                  submodule_search_locations=None)
    mod = importlib.util.module_from_spec(spec)
    mod.__package__ = 'evaluation'
    spec.loader.exec_module(mod)
    return mod.eval_quan_FOV


def _rows(means):
    """the six '[PSNR-FOV_*] (...' / '[SSIM-FOV_*] (...' rows of a block, up to the last row's closing ')'"""
    return ')\n'.join('[{}] ('.format(label) + ''.join(fmt.format(KEYS[-1] * 100, k * 100, means[j][k]) for k in KEYS)
                      for label, j, fmt in _ROWS)


def eval_quan_FOV(config):
    if os.environ.get('REFVSR_DROPIN_EVAL', '1') == '0':
        return _reference_impl()(config)
    mode = config.EVAL.eval_mode
    network, model, save_path_root_deblur, save_path_root_deblur_score, ckpt_name = init(config, mode)
    score_path = os.path.join(save_path_root_deblur_score, 'score_{}_{}.txt'.format(config.EVAL.data, config.EVAL.eval_mode))
    ops = rv_lib.CudaOps()
    debug = config.EVAL.is_debug

    def zeros():
        return [{key: 0 for key in KEYS} for _ in METRICS]

    totals, means = zeros(), zeros()          # [METRICS index][key], summed like the reference's twelve dicts
    total_norm = 0
    total_itr_time = total_itr_time_video = 0
    frame_count = 0
    frame_len_prev = 0
    for i, inputs in enumerate(model.data_loader_eval):
        is_first_frame = inputs['is_first'][0].item()
        if 'is_continue' in inputs.keys() and inputs['is_continue'][0].item():
            print('passing, video', inputs['video_name'][0])
            frame_len_prev += 1
            continue
        if debug:
            frame_count += 1
            if frame_count == 3:
                frame_len_prev = frame_count - 1
                is_first_frame = True

        if is_first_frame:
            if i > 0:
                total_itr_time = total_itr_time + total_itr_time_video
                total_itr_time_video = total_itr_time_video / frame_len_prev
                for j in range(len(METRICS)):
                    for key in KEYS:
                        totals[j][key] += means[j][key]
                        means[j][key] = means[j][key] / frame_len_prev
                out_str = '[MEAN EVAL {}|{}|{}][{}/{}] ({:.5f}sec) \n'.format(
                    config.mode, config.EVAL.data, inputs['video_name'][0], inputs['video_idx'][0], inputs['video_len'][0],
                    total_itr_time_video) + _rows(means) + ') \n\n'
                print(out_str)
                if not debug:
                    with open(score_path, 'a') as file:
                        file.write(out_str)
            if debug and frame_count == 2:
                break
            total_itr_time_video = 0
            means = zeros()

        init_time = time.time()
        results = model.evaluation(inputs)
        itr_time = time.time() - init_time

        outs = results['vis']
        output = outs['SR_UW_png'] if ('LR_UW_png' in outs and 'SR_UW_png' in outs) else outs['SR_UW']   # the reference's fallback
        scores = score_frame(ops, output, outs['HR_UW'], config.scale if config.flag_HD_in else None)

        for key in KEYS:
            for j, v in enumerate(scores[key]):
                means[j][key] += v
            if key == 1:
                frame_name = inputs['frame_name'][0]
                line = '[EVAL {}|{}|{}][{}/{}][{}/{}] {} PSNR: {:.5f} SSIM: {:.5f} ({:.5f}sec)'.format(
                    config.mode, config.EVAL.data, inputs['video_name'][0], inputs['video_idx'][0] + 1, inputs['video_len'][0],
                    inputs['frame_idx'][0] + 1, inputs['frame_len'][0], frame_name, scores[key][0], scores[key][3], itr_time)
                print(line)
                if not debug:
                    with open(score_path, 'w' if (i == 0) else 'a') as file:
                        file.write(line + '\n')
            if debug:
                print(key, 'raw:', *scores[key])
                print(key, 'sum:', *(means[j][key] for j in range(len(METRICS))), '\n')

        total_itr_time_video = total_itr_time_video + itr_time
        total_norm = total_norm + 1
        frame_len_prev = inputs['frame_len'][0]

    total_itr_time = (total_itr_time + total_itr_time_video) / total_norm
    for j in range(len(METRICS)):
        for key in KEYS:
            totals[j][key] = (totals[j][key] + means[j][key]) / total_norm
    out_str = '\n[TOTAL {}|{}] \n'.format(ckpt_name, config.EVAL.data) + _rows(totals) + ') ({:.5f}sec)\n\n'.format(total_itr_time)
    sys.stdout.write(out_str)
    if not debug:
        with open(score_path, 'a') as file:
            file.write(out_str)
