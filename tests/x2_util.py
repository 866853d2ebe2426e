"""Shared helpers of the x2 tests (scale=2, matching_ksize=4): the golden cases and the oracle at x2.

The cases live in tests/golden/make_golden_x2.py (the generator that ran the unmodified reference); they are kept out of
tests/util.py::CASES, which the x4 tests parametrise over."""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

from oracle import refvsr_oracle as O
from util import GOLDEN_DIR

sys.path.insert(0, GOLDEN_DIR)
from make_golden_x2 import X2, X2_CASES, X2_CONFIGS, X2_MID  # noqa: E402,F401


def build_x2_case(name, device, ops=None, **cfg_over):
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.modules import seeded_test_weights
    from refvsr_b200.synth import make_clip
    spec = X2_CASES[name]
    over = dict(spec['over'])
    over.update(cfg_over)
    cfg = get_config(spec['config'], device=device, **over)
    net = SRNet(cfg).eval()
    seeded_test_weights(net, seed=spec['seed'])
    if ops is not None:
        net.Network.set_ops(ops)
    net = net.to(device)
    lrs, refs = make_clip(spec['frames'], spec['h'], spec['w'], spec['ref_scale'], seed=spec['seed'])
    golden = np.load(os.path.join(GOLDEN_DIR, name + '.npz'))
    return spec, cfg, net, lrs, refs, golden


class OracleRefVSRx2(O.OracleRefVSR):
    """OracleRefVSR (oracle/refvsr_oracle.py, the x4 / flag_HD_in restatement) extended to the x2 models: the three places
    where the reference's forward depends on `scale` are overridden."""

    def __init__(self, config, sd):
        super().__init__(config, sd)
        if config.scale != 2 or self.mk != 4 or self.hd:
            raise ValueError('OracleRefVSRx2: scale=2, matching_ksize=4, flag_HD_in=False')
        self._centre = None

    def match_features(self, x, pool):
        # vgg_range = 7 because scale != 4 (attention.py:31-40); no nearest resize without flag_HD_in (attention.py:65-67)
        x = F.conv2d(x, self.sd['feature_match.sub_mean.weight'], self.sd['feature_match.sub_mean.bias'])
        if pool:
            x = O.avgpool2(x)
        x = torch.relu(self.conv('feature_match.feature_extract.0', x))
        x = torch.relu(self.conv('feature_match.feature_extract.2', x))
        x = torch.relu(self.conv('feature_match.feature_extract.5', O.maxpool2(x)))
        return O.lrelu(self.conv('feature_match.feature_extract.map128.0', x), 0.2)

    def compute_up(self, bw_up, fw_up, conf_bw, conf_fw, base):
        # RefVSR.py:104-119 without upsample2 (RefVSR.py:89-90,114-115); base = bicubic x2 of the centre frame (RefVSR.py:288)
        cb = O.bicubic(conf_bw, 2).clamp(0, 1)
        cf = O.bicubic(conf_fw, 2).clamp(0, 1)
        cat = torch.cat([bw_up, fw_up], 1)
        out = self.conv('fusion_UP', cat, pad=0)
        alpha = self.basic2('conf_fusion_BWFW', torch.cat([cb, cf], 1))
        out = out + alpha * self.basic2('feat_fusion_BWFW', cat)
        out = self.reslist('feat_decoder_BWFW', 4, out)
        out = O.lrelu(self.conv('conv_hr', out), 0.1)
        return self.conv('conv_last', out) + O.bicubic(self._centre, 2).clamp(0, 1)

    def forward(self, lrs, refs, is_first_frame, is_train=False):
        self._centre = lrs[:, lrs.shape[1] // 2].float().cpu()
        return super().forward(lrs, refs, is_first_frame, is_train)
