"""The regions of the reference's FOV evaluation mode (evaluation/eval_quan_FOV.py:153-213) as boxes, and that mode's per-frame
scores from the per-box sums of `CudaOps.region_metrics`.

For each key (share of the frame the Ref camera also sees) the reference masks the frame with centred boxes: inside (fi) is the
crop `[h//r : h-h//r, w//r : w-w//r]` with r = int(1/((1-key)/2)) (the full frame for key 1), outside (fo) is the frame minus
that crop, and the ring (fr) is the crop minus key 0.5's crop (r = 4).  Key 1's SSIM inside is skimage's plain mean, i.e. over
the 3-pixel valid interior of the SSIM map.  Every region is therefore `plus - minus` for two of the seven boxes of
`fov_boxes`, with `minus` inside `plus` (r >= 4 makes each crop contain key 0.5's)."""
import cv2
import numpy as np
import torch

KEYS = (1, 0.9, 0.8, 0.7, 0.6, 0.5)
FULL, INTERIOR, INNER = 5, 6, 4          # box indices: the frame, the SSIM valid interior, key 0.5's crop (the ring's hole)


def crop_ratio(key):
    """the reference's own expression: 20, 10, 6, 5, 4 for keys 0.9 .. 0.5 (0.7 gives 6, not 6.67)"""
    return int(1 / ((1 - key) / 2))


def fov_boxes(H, W):
    """the seven (y0, y1, x0, x1) half-open boxes of a frame: the crop of each key below 1, the frame, the SSIM valid interior"""
    crops = [(H // r, H - H // r, W // r, W - W // r) for r in map(crop_ratio, KEYS[1:])]
    return crops + [(0, H, 0, W), (3, H - 3, 3, W - 3)]


def fov_regions(key):
    """{metric: (plus, minus)} box indices of one key for the six metrics PSNR_fi, PSNR_fo, PSNR_fr, SSIM_fi, SSIM_fo, SSIM_fr
    (minus None: the box alone); a metric the reference does not score for the key (it adds 0) is absent"""
    if key == 1:
        return {'PSNR_fi': (FULL, None), 'SSIM_fi': (INTERIOR, None), 'PSNR_fr': (FULL, INNER), 'SSIM_fr': (FULL, INNER)}
    k = KEYS.index(key) - 1
    reg = {'PSNR_fi': (k, None), 'SSIM_fi': (k, None), 'PSNR_fo': (FULL, k), 'SSIM_fo': (FULL, k)}
    if key > 0.5:
        reg['PSNR_fr'] = reg['SSIM_fr'] = (k, INNER)
    return reg


METRICS = ('PSNR_fi', 'PSNR_fo', 'PSNR_fr', 'SSIM_fi', 'SSIM_fo', 'SSIM_fr')


def fov_scores(sq, s, boxes):
    """key -> the six metrics (METRICS order) of one frame from region_metrics' per-box sums `sq` (squared error) and `s` (SSIM
    map) over `boxes` = fov_boxes(H, W).  numpy float64 arithmetic throughout, so an empty region gives nan and an exact match
    inf, as the reference's numpy scalars do; unscored metrics are 0 like the reference's."""
    area = [np.float64(3 * (y1 - y0) * (x1 - x0)) for y0, y1, x0, x1 in boxes]

    def region(v, plus, minus):
        if minus is None:
            return np.float64(v[plus]), area[plus]
        return np.float64(v[plus]) - np.float64(v[minus]), area[plus] - area[minus]

    out = {}
    with np.errstate(divide='ignore', invalid='ignore'):
        for key in KEYS:
            vals = []
            reg = fov_regions(key)
            for m in METRICS:
                if m not in reg:
                    vals.append(0)
                elif m.startswith('PSNR'):
                    total, count = region(sq, *reg[m])
                    vals.append(10 * np.log10(np.float64(1.0) / (total / count)))
                else:
                    total, count = region(s, *reg[m])
                    vals.append(total / count)
            out[key] = tuple(vals)
    return out


def score_frame(ops, output, gt, hd_scale=None):
    """the six metrics per key of one frame (fov_scores) with one `ops.region_metrics` call.  output, gt: (1, 3, H, W) images on
    one device.  hd_scale (flag_HD_in models, whose output is hd_scale times the size of gt): the output is first copied to the
    host and cv2-resized by 1 / hd_scale exactly as the reference does (eval_quan_FOV.py:146-149), then uploaded again."""
    if hd_scale:
        output_cpu = output.cpu().numpy()[0].transpose(1, 2, 0)
        output_cpu = cv2.resize(output_cpu, dsize=(0, 0), fx=1 / hd_scale, fy=1 / hd_scale, interpolation=cv2.INTER_CUBIC)
        output = torch.from_numpy(output_cpu.transpose(2, 0, 1)[None].copy()).to(gt.device)
    boxes = fov_boxes(output.shape[2], output.shape[3])
    sq, s = ops.region_metrics(output.float().contiguous(), gt.float().contiguous(), boxes)
    return fov_scores(sq, s, boxes)
