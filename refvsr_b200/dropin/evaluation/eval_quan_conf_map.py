"""`eval_quan_conf_map(config)` - drop-in for evaluation/eval_quan_conf_map.py:18-182 (`run.py --eval_mode conf`) with the same
printed lines, score file and image tree.

Per frame the reference copies the four confidence maps to the host one by one, min/max-normalises them on the device, runs
matplotlib's `inferno` over each in float64, copies the input and the output back and writes 12 images from float32 arrays
(cv2.imwrite rounds them to 8 bits).  Here one `rv_conf_map_images` call produces all six images as the exact 8-bit BGR bytes
those writes store (refvsr_b200/colormap.py holds the table), one non-blocking copy moves them into a pinned buffer, and the
qual_quan drop-in's writer encodes them on REFVSR_EVAL_WRITERS threads while the next frame runs.  A vis without
`conf_map_prop` takes the reference's other branch (:97-104): `conf_map` alone, coloured without normalisation.  The printed
seconds time `model.evaluation` alone, as the reference's do.

`REFVSR_DROPIN_EVAL=0` runs the reference's own loop."""
import importlib.util
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import torch

from refvsr_b200 import lib as rv_lib
from refvsr_b200.colormap import inferno_lut

from . import REFERENCE_DIR
from .eval_qual_quan import _write_images
from .init import init

# eval_vis keys and image directories of the maps, in the order of rv_conf_map_images' packed buffer
MAP_KEYS = ('conf_map', 'conf_map_prop', 'conf_map_prop_backward', 'conf_map_prop_forward')
MAP_DIRS = ('conf_map_norm', 'conf_map_prop_norm', 'conf_map_prop_b_norm', 'conf_map_prop_f_norm')


def _reference_impl():
    spec = importlib.util.spec_from_file_location('evaluation._reference_eval_quan_conf_map',
                                                  os.path.join(REFERENCE_DIR, 'eval_quan_conf_map.py'), submodule_search_locations=None)
    mod = importlib.util.module_from_spec(spec)
    mod.__package__ = 'evaluation'
    spec.loader.exec_module(mod)
    return mod.eval_quan_conf_map


def split_images(buf, map_hw, n_maps, inp_hw, out_hw):
    """views of a packed rv_conf_map_images buffer (flat uint8 numpy array): n_maps (h, w, 3) maps, the input, the output"""
    views, off = [], 0
    for h, w in [map_hw] * n_maps + [inp_hw, out_hw]:
        views.append(buf[off:off + 3 * h * w].reshape(h, w, 3))
        off += 3 * h * w
    return views


def frame_images(ops, outs, vis):
    """one frame's packed image bytes (a uint8 tensor on the frames' device) and the directory of each image, in buffer order"""
    normalize = 'conf_map_prop' in vis.keys()
    keys = MAP_KEYS if normalize else MAP_KEYS[:1]
    try:
        inp, output = outs['LR_UW_png'], outs['SR_UW_png']
    except Exception:                                                   # noqa: BLE001  (the reference's own fallback, :107-112)
        inp, output = outs['LR_UW'], outs['SR_UW']
    maps = [vis[k].float().contiguous() for k in keys]
    inp, output = inp.float().contiguous(), output.float().contiguous()
    packed = ops.conf_map_images(maps, inp, output, inferno_lut(inp.device), normalize)
    shapes = (tuple(maps[0].shape[2:]), len(maps), tuple(inp.shape[2:]), tuple(output.shape[2:]))
    return packed, shapes, MAP_DIRS[:len(keys)] + ('input', 'output')


def eval_quan_conf_map(config):
    if os.environ.get('REFVSR_DROPIN_EVAL', '1') == '0':
        return _reference_impl()(config)
    mode = config.EVAL.eval_mode
    config.save_sample = True
    network, model, save_path_root_deblur, save_path_root_deblur_score, ckpt_name = init(config, mode)
    score_path = os.path.join(save_path_root_deblur_score, 'score_{}_{}.txt'.format(config.EVAL.data, config.EVAL.eval_mode))
    ops = rv_lib.CudaOps()
    pool = ThreadPoolExecutor(max_workers=int(os.environ.get('REFVSR_EVAL_WRITERS', '4')))
    pending = []
    ring = {}                                             # pinned host buffers, three per size (two frames may still be encoding)

    total_norm = 0
    frame_len_prev = 0
    total_itr_time = 0
    total_itr_time_video = 0
    for i, inputs in enumerate(model.data_loader_eval):
        is_first_frame = inputs['is_first'][0].item()
        if 'is_continue' in inputs.keys() and inputs['is_continue'][0].item():
            print('passing, video', inputs['video_name'][0])
            frame_len_prev += 1
            continue

        if is_first_frame:
            if i > 0:
                total_itr_time = total_itr_time + total_itr_time_video
                total_itr_time_video = total_itr_time_video / frame_len_prev
                line = '[MEAN EVAL {}|{}|{}][{}/{}] ({:.5f}sec)\n\n'.format(config.mode, config.EVAL.data, inputs['video_name'][0],
                                                                          inputs['video_idx'][0], inputs['video_len'][0], total_itr_time_video)
                print(line)
                with open(score_path, 'a') as file:
                    file.write(line)
            total_itr_time_video = 0

        init_time = time.time()
        results = model.evaluation(inputs, is_log=True)
        itr_time = time.time() - init_time

        packed, shapes, dirs = frame_images(ops, results['vis'], results['vis']['eval_vis'])
        ev = None
        if packed.is_cuda:
            slot = (total_norm % 3, packed.numel())
            if slot not in ring:
                ring[slot] = torch.empty(packed.numel(), dtype=torch.uint8).pin_memory()
            ring[slot].copy_(packed, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            host = ring[slot].numpy()
        else:
            host = packed.numpy().copy()

        frame_name = inputs['frame_name'][0]
        line = '[EVAL {}|{}|{}][{}/{}][{}/{}] {} ({:.5f}sec)\n'.format(
            config.mode, config.EVAL.data, inputs['video_name'][0], inputs['video_idx'][0] + 1, inputs['video_len'][0],
            inputs['frame_idx'][0] + 1, inputs['frame_len'][0], frame_name, itr_time)
        print(line)
        with open(score_path, 'w' if (i == 0) else 'a') as file:
            file.write(line)

        # (the reference's `'gt' in inputs` branch, :123-124 and :167-170, names an undefined `gt`; no data set has that key)
        frame_name_no_ext = frame_name.split('.')[0]
        vid = inputs['video_name'][0]
        paths = [[os.path.join(save_path_root_deblur, iformat, d, vid, '{}.{}'.format(frame_name_no_ext, iformat))
                  for iformat in ('png', 'jpg')] for d in dirs]
        pending.append(pool.submit(_write_images, (ev, split_images(host, *shapes), paths)))
        while len(pending) > 2:                           # a pinned slot is reused every third frame: keep the queue short
            pending.pop(0).result()

        total_itr_time_video = total_itr_time_video + itr_time
        total_norm = total_norm + 1
        frame_len_prev = inputs['frame_len'][0]

    for f in pending:
        f.result()
    pool.shutdown()
    total_itr_time = (total_itr_time + total_itr_time_video) / total_norm
    line = '\n[TOTAL {}|{}] ({:.5f}sec)\n'.format(ckpt_name, config.EVAL.data, total_itr_time)
    sys.stdout.write(line)
    with open(score_path, 'a') as file:
        file.write(line)
