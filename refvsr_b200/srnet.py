"""Drop-in for models/SRNet.py (reference lines cited inline)."""
import collections
import importlib

import numpy as np
import torch
import torch.nn as nn


class SRNet(nn.Module):
    """models/SRNet.py:11-61.  `config.network` selects the architecture module exactly like the
    reference's importlib hook (SRNet.py:20-21); 'RefVSR' resolves to refvsr_b200.network.Network, any
    other name is looked up as `models.archs.<name>` so third-party archs keep working."""

    def __init__(self, config):
        super().__init__()
        self.rank = torch.distributed.get_rank() if getattr(config, 'dist', False) else -1
        self.config = config
        self.device = config.device
        if config.network == 'RefVSR':
            from .network import Network
            self.Network = Network(config)
        else:
            lib = importlib.import_module('models.archs.{}'.format(config.network))
            self.Network = lib.Network(config)
        self.data = collections.OrderedDict()

    def weights_init(self, m):                       # SRNet.py:24-38
        if isinstance(m, (torch.nn.Conv2d, torch.nn.ConvTranspose2d)):
            torch.nn.init.xavier_uniform_(m.weight, gain=self.config.wi)
            if m.bias is not None:
                torch.nn.init.constant_(m.bias, 0)
        elif type(m) in (torch.nn.BatchNorm2d, torch.nn.InstanceNorm2d):
            if m.weight is not None:
                torch.nn.init.constant_(m.weight, 1)
                torch.nn.init.constant_(m.bias, 0)
        elif type(m) == torch.nn.Linear:
            torch.nn.init.normal_(m.weight, 0, self.config.win)
            if m.bias is not None:
                torch.nn.init.constant_(m.bias, 0)

    def init(self):                                   # SRNet.py:40-45
        if self.config.wi is not None and self.config.win is not None:
            self.Network.apply(self.weights_init)
            if self.Network.FlowNet is not None:
                self.Network.FlowNet.load_ckpt(pretrained='./ckpt/SPyNet.pytorch')

    def input_constructor(self, res):                 # SRNet.py:47-54 (ptflops hook)
        b, f, c, h, w = res[:]
        imgs = torch.FloatTensor(np.random.randn(b, f, c, h, w)).to(self.device)
        return {'x': imgs, 'ref': imgs}

    def forward(self, x, ref, is_first_frame=True, is_log=False, is_train=False):   # SRNet.py:57-61
        return self.Network.forward(x, ref, is_first_frame, is_log=is_log, is_train=is_train)

    def push_frame(self, lr, ref):
        """streaming twin of forward() for callers that keep their own decoded-frame ring: after the clip's first window, hand
        over only the entering (LR, Ref) frame -> (3, scale*h, scale*w); see Network.push_frame (no counterpart in the reference)"""
        return self.Network.push_frame(lr, ref)

    def push_frames(self, lrs, refs):
        """push_frame for a batch of n streams: the entering frames (n, 3, h, w) / (n, 3, hr, wr) -> (n, 3, scale*h, scale*w), one
        batched window schedule; see Network.push_frames"""
        return self.Network.push_frames(lrs, refs)

    def forward_u8(self, lrs, refs, is_first_frame=True, bgr=False):
        """forward() for decoded 8-bit video: lrs (n, t, h, w, 3), refs (n, t, hr, wr, 3) contiguous uint8 HWC frames on the
        engine's device (bgr: cv2's B, G, R order) -> (n, scale*h, scale*w, 3) uint8, the bytes cv2.imwrite would store for
        forward()'s result on u8 / 255; see Network.forward_u8 (no counterpart in the reference)"""
        return self.Network.forward_u8(lrs, refs, is_first_frame, bgr=bgr)

    def push_frame_u8(self, lr, ref, bgr=False):
        """push_frame() for 8-bit frames: lr (h, w, 3), ref (hr, wr, 3) uint8 -> (scale*h, scale*w, 3) uint8"""
        return self.Network.push_frame_u8(lr, ref, bgr=bgr)

    def push_frames_u8(self, lrs, refs, bgr=False):
        """push_frames() for 8-bit frames: lrs (n, h, w, 3), refs (n, hr, wr, 3) uint8 -> (n, scale*h, scale*w, 3) uint8"""
        return self.Network.push_frames_u8(lrs, refs, bgr=bgr)

    def forward_yuv420(self, lrs, refs, is_first_frame=True, nv12=False):
        """forward() for decoded 4:2:0 video: lrs (n, t, 3h/2, w), refs (n, t, 3hr/2, wr) contiguous uint8 I420 frames (nv12:
        NV12) on the engine's device -> (n, 3H/2, W) uint8 frames of the same layout, the 4:2:0 frames of forward_u8's RGB
        result for the RGB frames cv2.cvtColor makes of the inputs; see Network.forward_yuv420 (no counterpart in the reference)"""
        return self.Network.forward_yuv420(lrs, refs, is_first_frame, nv12=nv12)

    def push_frame_yuv420(self, lr, ref, nv12=False):
        """push_frame() for 4:2:0 frames: lr (3h/2, w), ref (3hr/2, wr) uint8 -> (3H/2, W) uint8"""
        return self.Network.push_frame_yuv420(lr, ref, nv12=nv12)

    def push_frames_yuv420(self, lrs, refs, nv12=False):
        """push_frames() for 4:2:0 frames: lrs (n, 3h/2, w), refs (n, 3hr/2, wr) uint8 -> (n, 3H/2, W) uint8"""
        return self.Network.push_frames_yuv420(lrs, refs, nv12=nv12)
