"""`Network` - the CUDA implementation of models/archs/RefVSR.py::Network (reference lines cited inline).

The module keeps the reference's constructor signature (`Network(config)`), attribute names,
`state_dict()` schema and the stateful `forward(lrs, refs, is_first_frame, is_log, is_train)` contract
(RefVSR.py:151-325).  The forward pass is an explicit schedule of calls into the operator set
(`lib.CudaOps`: hand-written sm_90a kernels behind the C ABI).  Differences to the reference are
confined to *how* results are obtained, never to what they are:

  * activations are NHWC f16/bf16/f32 buffers; concat / bias / activation / gating / residual /
    pixel-shuffle are fused into the conv kernels;
  * exact reuse across sliding windows (SURVEY 7.8): optical flows, matching confidence / index maps and
    the aligned reference features (aa1 / aa2 outputs) are pure functions of frame content; a window that
    slides by one frame (the reference's own assumption when it reuses forward_*_prev, RefVSR.py:256-260)
    re-computes only what the new frame brings.  Flows the reference computes but never consumes are skipped;
  * every buffer of a step lives at a fixed address (pooled scratch + a ring of T per-frame slots), so a
    whole window is ONE CUDA-graph launch after its first occurrence (~750 kernels, no host work between
    them); graphs are keyed by (ring phase, window kind, work list);
  * inside a steady window the branches that do not depend on each other are enqueued on side streams (fork / join nodes of the
    window's graph): the forward-branch step (RefVSR.py:248-277) and the two optical flows of the entering frame pair run next to
    the matching / alignment products and the backward branch (RefVSR.py:211-238).  Same kernels, inputs and per-branch order;
  * `push_frame` (no counterpart in the reference): the window slides by one and only the entering frame is handed over;
  * no gc.collect()/empty_cache() (RefVSR.py:206-208); the only host synchronisation of a call is the reuse guard's verdict
    (`b200_reuse_check='sync'`, one int32).
"""
import collections
import contextlib
import os

import torch
import torch.nn as nn

from . import packing
from .lib import (ACT_CLAMP3, ACT_LRELU01, ACT_LRELU02, ACT_NONE, ACT_RELU, FRAME_I420, FRAME_NV12, frame_shape)
from .modules import build_parameter_tree

_PREC = {'fp32': torch.float32, 'fp16': torch.float16, 'bf16': torch.bfloat16}


class _NewestOnly:
    """window stand-in of Network.push_frame: only the entering frame (index t-1) exists; the staging loop of _do_window never asks
    for another one because positions a0 .. a0+t-2 are already staged"""

    def __init__(self, frame, t):
        self.frame, self.t, self.is_cuda = frame, t, frame.is_cuda

    def __getitem__(self, j):
        if j != self.t - 1:
            raise RuntimeError('push_frame: the engine asked for a frame it should already hold (ring bookkeeping out of step)')
        return self.frame


def _cget(config, name, default):
    try:
        v = getattr(config, name)
    except (AttributeError, KeyError):
        return default
    return default if v is None else v


class Network(nn.Module):
    def __init__(self, config, ops=None):
        super().__init__()
        self.config = config
        self.rank = torch.distributed.get_rank() if _cget(config, 'dist', False) else -1
        self.scale = config.scale
        self.flag_HD_in = config.flag_HD_in
        self.mid_channels = config.mid_channels
        if self.scale == 2:
            # the x2 models (config_RefVSR_*.py:30-34: scale 2 with matching_ksize 4): VGG[0:7] matching at 1/2 resolution,
            # AlignedConv2d on both alignment levels (aa1 blocks of 2, aa2 blocks of 4), no upsample2.  The other x2
            # combinations fail inside the reference itself, so there is nothing to reproduce.
            if self.flag_HD_in:
                raise NotImplementedError('scale=2 with flag_HD_in is not supported: the reference cannot compute it '
                                          '(its block gather indexes past the unfolded reference, attention.py:143)')
            if config.matching_ksize != 4:
                raise NotImplementedError('scale=2 needs matching_ksize=4 (got %s): with any other block size the reference '
                                          'cannot compute it (F.fold size mismatch, attention.py:144)' % (config.matching_ksize,))
        elif self.scale != 4:
            # fail loudly instead of silently computing something else.  flag_HD_in (the "8K" configs: VGG[0:7] matching at
            # 1/4 resolution, matching_ksize 8, AlignedConv2d on both alignment levels) is handled by the same schedule.
            raise NotImplementedError('refvsr_b200 implements the x4 models (config_RefVSR_{small_,}{L1,MFID}{,_8K}) and '
                                      'the x2 models (scale=2, matching_ksize=4); got scale=%s' % (self.scale,))
        build_parameter_tree(self, config)

        # cross-call recurrent state (RefVSR.py:96-101), one entry per batch element
        self.frame_itr_num = 0
        self.max_frame_itr_num = config.reset_branch
        self._state = {}
        self._packed = {}
        self._graphs = {}
        self._mat12 = None
        self._ops = ops
        prec = _cget(config, 'b200_precision', None)
        if prec is None:
            prec = 'fp16' if _cget(config, 'is_amp', False) else 'bf16'
        self.precision = prec
        self.act_dtype = _PREC[prec]
        # 'split' = fp32-grade matching GEMM ([hi|lo|hi] fp16 operands), 'single' = one fp16 pass
        # (what the reference does under autocast, trainers/trainer.py:237-239)
        # tools/match_mode_check.py compares the two against the reference; the fp32 path needs the fp32-grade
        # argmax, the 16-bit paths already round their features
        self.match_mode = _cget(config, 'b200_match', 'split' if prec == 'fp32' else 'single')
        self.prefer_tc = bool(_cget(config, 'b200_tensor_cores', True))
        self.reuse = bool(_cget(config, 'b200_reuse', True))
        # the reuse cache is only valid when consecutive calls slide the window by exactly one frame (what the reference's
        # own eval loop does, data_loader/datasets.py:222-245).  'sync' (default): every non-first call compares the t-1
        # overlapping LR / Ref frames with the staged copies on the device (one launch, ~20 MB read); a caller that does NOT
        # slide gets a full recompute, i.e. exactly what the reference would compute for that call (one small D2H + host sync per
        # call; a speculative variant that launches the window behind the check and reads the verdict afterwards was built and
        # measured in round 2: no gain within run-to-run noise, so the simpler decide-first form stays).  'async': same check, verdict read at the NEXT call -> RuntimeError
        # (no host sync on the hot path).  'off': trust the caller (round-1 behaviour).
        self.reuse_check = _cget(config, 'b200_reuse_check', 'sync')
        if self.reuse_check not in ('sync', 'async', 'off'):
            raise ValueError("b200_reuse_check must be 'sync', 'async' or 'off'")
        self.reuse_fallbacks = 0      # calls that violated the sliding contract and were recomputed from scratch
        self.batch_fallbacks = 0      # calls of n > 1 windows whose elements needed different schedules (run one by one)
        self.use_graphs = bool(_cget(config, 'b200_cuda_graphs', True))
        # residual blocks through the fused rv_resblock kernel (one launch per block) -> opt-in
        self.fuse_resblocks = bool(_cget(config, 'b200_fuse_resblocks', False))
        # rv_conv_chain: the 60-conv propagation trunks and the ResList decoders as one call each, the same results as the
        # per-layer path (csrc/conv_chain.cu) -> opt-in.
        self.use_chain = bool(_cget(config, 'b200_conv_chain', False)) and not os.environ.get('REFVSR_NO_CHAIN')
        self.chain_max_ctas = int(_cget(config, 'b200_chain_max_ctas', 0))   # see rv_conv_chain_desc.max_ctas (dist.py sets it)
        # The forward-branch step of a steady window (RefVSR.py:248-277) needs only the previous call's state and per-frame products
        # of earlier calls; the products of the entering frame and the backward branch (RefVSR.py:211-238) do not depend on it.
        # With overlap on, the forward step is enqueued on a second stream (a fork / join inside the window's CUDA graph): the
        # launches of the two branches fill each other's prologue / first-box latency / last-tile tail (part of every trunk
        # conv).  Same kernels, same inputs, same order within each branch: bit-identical
        # results (tests/test_gpu_model.py::test_branch_overlap_is_exact).  A static SM split between
        # the two streams (rv_set_conv_cta_cap) is available; the branches are not symmetric and a cap outlives the overlap,
        # so the caps default to 0 (none).
        self.overlap_branches = bool(_cget(config, 'b200_overlap_branches', True)) and not os.environ.get('REFVSR_NO_OVERLAP')
        # grid caps: forward step (second stream) / products and the first `overlap_bw_steps` backward steps (main stream); 0 = none
        self.overlap_cap = int(os.environ.get('REFVSR_OVERLAP_CAP', _cget(config, 'b200_overlap_cap', 0)))
        self.overlap_main_cap = int(os.environ.get('REFVSR_OVERLAP_MAIN_CAP', _cget(config, 'b200_overlap_main_cap', 0)))
        self.overlap_bw_steps = int(os.environ.get('REFVSR_OVERLAP_BW_STEPS', _cget(config, 'b200_overlap_bw_steps', 0)))
        # hash-keyed on-disk cache of packed conv weights (SURVEY 8f row 4); opt-in: config.b200_pack_cache = <dir> or
        # REFVSR_PACK_CACHE=<dir> (packing.py)
        if _cget(config, 'b200_pack_cache', None):
            os.environ['REFVSR_PACK_CACHE'] = str(_cget(config, 'b200_pack_cache', None))
        self._side = None
        self._flow_streams = None
        self._ring_mod = None
        self._shard = None
        self._bufs = {}
        self._device = torch.device('cpu')
        self._b = 0
        self._bn = 1                  # windows of the current call: ring slots and carried state are [bn][...] tensors
        self._bmode = False           # enqueueing the batched steps of a call: every scratch buffer has the batch dimension
        self._u8 = None               # inside an 8-bit call: its frame format, the bgr flag of forward_u8 / push_frame_u8 /
        #                               push_frames_u8 (False / True) or FRAME_I420 / FRAME_NV12 of the *_yuv420 entries
        self.executed_kernels = 0     # kernels of librefvsr_b200.so actually executed (eager launches + graph nodes)
        self.register_load_state_dict_post_hook(lambda module, incompatible: module._invalidate())

    def _invalidate(self):
        self._packed.clear()
        self._graphs.clear()
        self._mat12 = None

    def _apply(self, fn, *a, **k):
        # .to()/.cuda()/.half() move or convert parameters: packed weights, graphs and buffers must be rebuilt
        self._invalidate()
        self._bufs.clear()
        self._state.clear()
        return super()._apply(fn, *a, **k)

    # ------------------------------------------------------------------------------------------
    # plumbing
    # ------------------------------------------------------------------------------------------
    @property
    def ops(self):
        if self._ops is None:
            from .lib import CudaOps
            self._ops = CudaOps()
        return self._ops

    def set_ops(self, ops):
        self._ops = ops
        self._invalidate()

    def reset_state(self):
        self._state.clear()
        self.frame_itr_num = 0

    def _layer(self, name, srcs, stride=1, pad=None, bias_add=0.0, s2d=False, ps_rows=False):
        """Packed weights of conv `name` (attribute path under self) for the given source layout.  ps_rows: the conv feeds a
        pixel shuffle, and the engine's own packing puts its columns in the HR-row order (packing.ps_rows_order); ops that
        pack their own layers keep the conv's order."""
        key = (name, tuple(srcs), s2d, ps_rows)
        hit = self._packed.get(key)
        if hit is not None:
            return hit
        mod = self.get_submodule(name)
        weight, srcs = mod.weight.detach(), list(srcs)
        k = weight.shape[2]
        pad = k // 2 if pad is None else pad
        if s2d:
            weight, srcs = packing.s2d_weights(weight, srcs, k // 2)
        if hasattr(self.ops, 'pack_conv'):
            pc = self.ops.pack_conv(name, weight, mod.bias, srcs, stride, pad, self.act_dtype, self._device, self.prefer_tc, bias_add)
        else:
            pc = packing.pack_conv(name, weight, mod.bias, srcs, stride, pad, self.act_dtype, self._device, self.prefer_tc, bias_add,
                                   ps_rows=ps_rows)
        self._packed[key] = pc
        return pc

    def _buf(self, tag, shape, dtype, whole=False):
        if self._bmode and not whole:
            tag, shape = f'B{self._bn}.{tag}', (self._bn,) + tuple(shape)
        key = (tag, tuple(shape), dtype)
        b = self._bufs.get(key)
        if b is None or b.device != self._device:
            b = torch.empty(tuple(shape), dtype=dtype, device=self._device)
            self._bufs[key] = b
        return b

    def _sbuf(self, kind, rest, shape, dtype):
        """Per-stream state of batch element self._b: ring slots (kind 'ring') and the carried forward state (kind 'prev').  In a
        call of n > 1 windows each buffer is ONE [n][...] tensor: the per-element products write their slice of it and the batched
        steps (self._bmode) read and write it whole."""
        if self._bn > 1:
            full = self._buf(f'{kind}B{self._bn}.{rest}', (self._bn,) + tuple(shape), dtype, whole=True)
            return full if self._bmode else full[self._b]
        return self._buf(f'{kind}{self._b}.{rest}', shape, dtype)

    def _conv(self, name, src0, src1, out, srcs, act_pre=ACT_NONE, act_post=ACT_NONE, gate=None, res=None,
              pixel_shuffle=False, stride=1, pad=None, bias_add=0.0):
        k = self.get_submodule(name).weight.shape[2]
        if (stride == 2 and self.prefer_tc and self.act_dtype != torch.float32 and k in (3, 5)
                and (pad is None or pad == k // 2) and src0.shape[-3] % 2 == 0 and src0.shape[-2] % 2 == 0):
            # stride-2 conv as a stride-1 3x3 conv over the space-to-depth input -> tensor-core kernel
            z0 = self._buf(f's2d.{name}.0', (src0.shape[-3] // 2, src0.shape[-2] // 2, 4 * src0.shape[-1]), src0.dtype)
            self.ops.space_to_depth2(src0, z0)
            z1 = None
            if src1 is not None:
                z1 = self._buf(f's2d.{name}.1', (src1.shape[-3] // 2, src1.shape[-2] // 2, 4 * src1.shape[-1]), src1.dtype)
                self.ops.space_to_depth2(src1, z1)
            layer = self._layer(name, srcs, 1, 1, bias_add, s2d=True)
            self.ops.conv2d(layer, z0, z1, out, gate=gate, res=res, act_pre=act_pre, act_post=act_post,
                            pixel_shuffle=pixel_shuffle)
            return out
        layer = self._layer(name, srcs, stride, pad, bias_add, ps_rows=pixel_shuffle)
        self.ops.conv2d(layer, src0, src1, out, gate=gate, res=res, act_pre=act_pre, act_post=act_post,
                        pixel_shuffle=pixel_shuffle)
        return out

    # ------------------------------------------------------------------------------------------
    # building blocks
    # ------------------------------------------------------------------------------------------
    def _resblock(self, conv1, conv2, x, out, tmp, act_mid, act_post=ACT_NONE):
        """out = act_post(x + conv2(act_mid(conv1(x)))): rv_resblock when the block qualifies
        (16-bit activations, C <= 64), otherwise two convolutions through the scratch buffer `tmp`."""
        C = x.shape[-1]
        m1, m2 = self.get_submodule(conv1), self.get_submodule(conv2)
        if (self.fuse_resblocks and self.prefer_tc and hasattr(self.ops, 'resblock')
                and packing.resblock_fusable(m1.weight, m2.weight, C, self.act_dtype)):
            key = ('rb', conv1, conv2, C)
            rb = self._packed.get(key)
            if rb is None:
                pack = self.ops.pack_resblock if hasattr(self.ops, 'pack_resblock') else packing.pack_resblock
                rb = pack(conv1, m1.weight, m1.bias, m2.weight, m2.bias, C, self.act_dtype, self._device)
                self._packed[key] = rb
            self.ops.resblock(rb, x, out, act_mid, act_post)
            return out
        self._conv(conv1, x, None, tmp, [(C, C)], act_pre=act_mid)
        self._conv(conv2, tmp, None, out, [(C, C)], res=x, act_post=act_post)
        return out

    def _chain_layer(self, name, C):
        key = ('chain', name)
        hit = self._packed.get(key)
        if hit is None:
            mod = self.get_submodule(name)
            pack = self.ops.pack_chain if hasattr(self.ops, 'pack_chain') else packing.pack_chain
            hit = pack(name, mod.weight, mod.bias, C, self.act_dtype, self._device)
            self._packed[key] = hit
        return hit

    def _chain_ok(self, names, C):
        return (self.use_chain and self.prefer_tc and not self.fuse_resblocks and hasattr(self.ops, 'conv_chain')
                and all(packing.chain_ok(self.get_submodule(n).weight, C, self.act_dtype) for n in names))

    def _run_chain(self, bufs, layers):
        H, W = bufs[0].shape[0], bufs[0].shape[1]
        flags = self._buf('chain.flags', (((H + 15) // 16) * ((W + 7) // 8),), torch.int32)
        self.ops.conv_chain(bufs, layers, flags, max_ctas=self.chain_max_ctas)

    def _reslist(self, prefix, n, x, out, tag):
        """ResList (RefVSR_/common.py:64-82): n x [x + conv2(lrelu0.2(conv1(x)))], conv_tail, + input."""
        H, W, C = x.shape[-3:]
        t = self._buf(tag + '.t', (H, W, C), x.dtype)
        s = [self._buf(tag + '.s0', (H, W, C), x.dtype), self._buf(tag + '.s1', (H, W, C), x.dtype)]
        names = [f'{prefix}.RBs.{i}.conv{j}' for i in range(n) for j in (1, 2)] + [f'{prefix}.conv_tail']
        if self._chain_ok(names, C):
            bufs = [x, s[0], s[1], t, out]              # buffer indices 0..4
            layers, cur = [], 0
            for i in range(n):
                nxt = 1 + (i % 2)
                layers.append((self._chain_layer(f'{prefix}.RBs.{i}.conv1', C), cur, -1, 3, ACT_LRELU02, ACT_NONE))
                layers.append((self._chain_layer(f'{prefix}.RBs.{i}.conv2', C), 3, cur, nxt, ACT_NONE, ACT_NONE))
                cur = nxt
            layers.append((self._chain_layer(f'{prefix}.conv_tail', C), cur, 0, 4, ACT_NONE, ACT_NONE))
            self._run_chain(bufs, layers)
            return out
        cur = x
        for i in range(n):
            nxt = s[i % 2]
            self._resblock(f'{prefix}.RBs.{i}.conv1', f'{prefix}.RBs.{i}.conv2', cur, nxt, t, ACT_LRELU02)
            cur = nxt
        self._conv(f'{prefix}.conv_tail', cur, None, out, [(C, C)], res=x)
        return out

    def _prop_resblocks(self, prefix, lr8, feat, out, tag):
        """ResidualBlocksWithInputConv (RefVSR.py:327-360) on cat[lr, feat] (RefVSR.py:225-226,266-267)."""
        C = self.mid_channels
        H, W = feat.shape[-3], feat.shape[-2]
        nblk = self.config.num_blocks
        t = self._buf(tag + '.t', (H, W, C), feat.dtype)
        s = [self._buf(tag + '.s0', (H, W, C), feat.dtype), self._buf(tag + '.s1', (H, W, C), feat.dtype)]
        cur = self._conv(f'{prefix}.main.0', lr8, feat, out if nblk == 0 else s[0], [(3, 8), (C, C)],
                         act_pre=ACT_LRELU01)
        names = [f'{prefix}.main.2.{i}.conv{j}' for i in range(nblk) for j in (1, 2)]
        if nblk > 0 and self._chain_ok(names, C):
            bufs = [s[0], s[1], t, out]                 # buffer indices 0..3
            layers, ci = [], 0
            for i in range(nblk):
                ni = 3 if i == nblk - 1 else 1 - ci
                layers.append((self._chain_layer(f'{prefix}.main.2.{i}.conv1', C), ci, -1, 2, ACT_RELU, ACT_NONE))
                layers.append((self._chain_layer(f'{prefix}.main.2.{i}.conv2', C), 2, ci, ni, ACT_NONE, ACT_NONE))
                ci = ni
            self._run_chain(bufs, layers)
            return out
        for i in range(nblk):
            nxt = out if i == nblk - 1 else (s[1] if cur is s[0] else s[0])
            self._resblock(f'{prefix}.main.2.{i}.conv1', f'{prefix}.main.2.{i}.conv2', cur, nxt, t, ACT_RELU)
            cur = nxt
        return out

    # ---- SPyNet (SPyNet.py:49-139) ----------------------------------------------------------------
    @staticmethod
    def _pyr_shapes(h, w):
        w_up = w if w % 32 == 0 else 32 * (w // 32 + 1)
        h_up = h if h % 32 == 0 else 32 * (h // 32 + 1)
        return [(h_up >> (5 - l), w_up >> (5 - l)) for l in range(6)]      # coarsest first

    def _pyramid(self, img, slot):
        """img (3,h,w) fp32 -> 6 normalised levels, coarsest first, each (H,W,3) fp32, in ring slot `slot`."""
        shapes = self._pyr_shapes(img.shape[1], img.shape[2])
        lv = [self._sbuf('ring', f'pyr{l}.{slot}', (H, W, 3), torch.float32) for l, (H, W) in enumerate(shapes)]
        self.ops.spynet_resize_norm(img, lv[5])
        for l in range(4, -1, -1):
            self.ops.avgpool2(lv[l + 1], lv[l])
        return lv

    def _spynet(self, pyr_ref, pyr_supp, out, sp='spy'):
        """flow from ref to supp into `out` (h,w,2) fp32.  pyr_*: outputs of _pyramid.  sp: scratch-buffer prefix (one set per
        stream when two flows are computed concurrently, _run_products)."""
        dt = self.act_dtype
        flow = None
        for level in range(6):
            r, s = pyr_ref[level], pyr_supp[level]
            H, W = r.shape[0], r.shape[1]
            x8 = self._buf(sp + '.x8', (H, W, 8), dt)
            flow_up = self._buf(sp + '.fu', (H, W, 2), torch.float32)
            self.ops.spynet_level_input(r, s, flow, x8, flow_up)
            pre = f'FlowNet.basic_module.{level}.basic_module'
            a = self._conv(f'{pre}.0.conv', x8, None, self._buf(sp + '.a', (H, W, 32), dt), [(8, 8)], act_pre=ACT_RELU)
            b = self._conv(f'{pre}.1.conv', a, None, self._buf(sp + '.b', (H, W, 64), dt), [(32, 32)], act_pre=ACT_RELU)
            c = self._conv(f'{pre}.2.conv', b, None, self._buf(sp + '.c', (H, W, 32), dt), [(64, 64)], act_pre=ACT_RELU)
            d = self._conv(f'{pre}.3.conv', c, None, self._buf(sp + '.d', (H, W, 16), dt), [(32, 32)], act_pre=ACT_RELU)
            flow = self._buf(sp + '.fl', (H, W, 2), torch.float32)
            self._conv(f'{pre}.4.conv', d, None, flow, [(16, 16)], res=flow_up)   # flow_up + residue (SPyNet.py:95)
        self.ops.flow_resize(flow, out)     # SPyNet.py:129-137; RefVSR.py:184,189 resize is the identity
        return out

    # ---- feature matching (attention.py:58-100) -----------------------------------------------------
    def _sub_mean_mat(self):
        if self._mat12 is None:
            sm = self.feature_match.sub_mean
            wm = sm.weight.detach().float().reshape(3, 3).cpu()
            bm = sm.bias.detach().float().cpu()
            self._mat12 = [float(v) for r in range(3) for v in (wm[r, 0], wm[r, 1], wm[r, 2], bm[r])]
        return self._mat12

    def _match_features(self, img, pool2, tag):
        dt = self.act_dtype
        if self.flag_HD_in:                                   # attention.py:65-67: nearest x0.5 before anything else
            small = self._buf(tag + '.nn', (3, img.shape[1] // 2, img.shape[2] // 2), torch.float32)
            self.ops.resize_planes(img, small, 2.0, mode='nearest')
            img = small
        H, W = (img.shape[1] // 2, img.shape[2] // 2) if pool2 else (img.shape[1], img.shape[2])
        x8 = self._buf(tag + '.x8', (H, W, 8), dt)
        self.ops.prep_image(img, x8, mat12=self._sub_mean_mat(), pool2=pool2)
        f1 = self._conv('feature_match.feature_extract.0', x8, None, self._buf(tag + '.f1', (H, W, 64), dt),
                        [(3, 8)], act_pre=ACT_RELU)
        f2 = self._conv('feature_match.feature_extract.2', f1, None, self._buf(tag + '.f2', (H, W, 64), dt),
                        [(64, 64)], act_pre=ACT_RELU)
        if self.feature_match.vgg_range == 7:                 # flag_HD_in or x2 (attention.py:31-40): maxpool, conv 64->128, ReLU
            Hm, Wm = H // 2, W // 2
            mp = self._buf(tag + '.mp', (Hm, Wm, 64), dt)
            self.ops.maxpool2(f2, mp)
            f5 = self._conv('feature_match.feature_extract.5', mp, None, self._buf(tag + '.f5', (Hm, Wm, 128), dt),
                            [(64, 64)], act_pre=ACT_RELU)
            return self._conv('feature_match.feature_extract.map128.0', f5, None, self._buf(tag + '.f3', (Hm, Wm, 16), dt),
                              [(128, 128)], act_pre=ACT_LRELU02)
        f3 = self._conv('feature_match.feature_extract.map64.0', f2, None, self._buf(tag + '.f3', (H, W, 16), dt),
                        [(64, 64)], act_pre=ACT_LRELU02)
        return f3

    def _feature_match(self, lr, ref, conf, idx):
        """conf (h,w) fp32, idx (hm*wm,) int32 indexing the reference feature grid; (hm, wm) = (h, w), (h/2, w/2) at x2 or
        (h/4, w/4) with flag_HD_in, where the relevance map is then bicubic-upsampled to (h, w) (attention.py:93-98)."""
        h, w = lr.shape[1], lr.shape[2]
        split = self.match_mode == 'split'
        kpad = 432 if split else 144          # 3 x 144 / 144 patch values: no zero columns for the GEMM to multiply
        lr_f = self._match_features(lr, False, 'fm.lr')
        hm, wm = lr_f.shape[0], lr_f.shape[1]
        conf_out = conf
        if (hm, wm) != (h, w):
            conf = self._buf('fm.conf_small', (hm, wm), torch.float32)
        A = self._buf('fm.A', (hm * wm, kpad), torch.float16)
        self.ops.patch_pack(lr_f, A, 1 if split else 0)
        ref_f = self._match_features(ref, True, 'fm.ref')
        R = ref_f.shape[0] * ref_f.shape[1]
        B = self._buf('fm.B', (R, kpad), torch.float16)
        self.ops.patch_pack(ref_f, B, 2 if split else 0)
        self.ops.match_argmax(A, B, conf, idx, impl=1 if self.prefer_tc else 0)
        if conf is not conf_out:
            self.ops.resize_planes(conf.view(1, hm, wm), conf_out.view(1, h, w), float(hm) / float(h), mode='bicubic',
                                   clamp01=True)

    # ---- reference encoders (RefVSR.py:233-234,274-275) ----------------------------------------------
    def _ref_features(self, ref):
        C, dt = self.mid_channels, self.act_dtype
        hr, wr = ref.shape[1], ref.shape[2]
        ref8 = self._buf('re.ref8', (hr, wr, 8), dt)
        self.ops.prep_image(ref, ref8)
        e0 = self._conv('ref_encoder1.0.0', ref8, None, self._buf('re.e0', (hr, wr, C), dt), [(3, 8)], act_pre=ACT_LRELU02)
        e1 = self._conv('ref_encoder1.1.0', e0, None, self._buf('re.e1', (hr, wr, C), dt), [(C, C)], act_pre=ACT_LRELU02)
        ref_feat = self._buf('re.feat', (hr, wr, C), dt)
        self._reslist('res1', 4, e1, ref_feat, 're.r1')
        h2, w2 = (hr - 1) // 2 + 1, (wr - 1) // 2 + 1
        d0 = self._conv('ref_encoder2.0.0', ref_feat, None, self._buf('re.d0', (h2, w2, C), dt), [(C, C)],
                        act_pre=ACT_LRELU02, stride=2)
        d1 = self._conv('ref_encoder2.1.0', d0, None, self._buf('re.d1', (h2, w2, C), dt), [(C, C)], act_pre=ACT_LRELU02)
        ref_feat_down = self._buf('re.featd', (h2, w2, C), dt)
        self._reslist('res2', 4, d1, ref_feat_down, 're.r2')
        return ref8, ref_feat, ref_feat_down

    # ---- AlignedConv2d (alignment.py:39-100) --------------------------------------------------------
    def _align_conv1(self, aa, x8, out, tag):
        H, W = x8.shape[0], x8.shape[1]
        dt = self.act_dtype
        a = self._conv(aa + '.align.conv1.0', x8, None, self._buf(tag + '.a', (H, W, 32), dt), [(3, 8)],
                       act_pre=ACT_LRELU02, pad=2)
        self._resblock(aa + '.align.conv1.2.conv1', aa + '.align.conv1.2.conv2', a, out, self._buf(tag + '.t', (H, W, 32), dt),
                       ACT_LRELU02, ACT_LRELU02)
        return out

    def _aligned_attention(self, aa, query_img, ref8, idx, value, out):
        """AlignedAttention + AlignedConv2d (attention.py:131-159, alignment.py:39-100) -> out (2hq', 2wq', C) where
        `query_img` (3, hq', wq') fp32 is the LR-side image (lr for aa2, lr_down for aa1), blocks are ks x ks pixels,
        ks = module scale (aa2: 2, 4 at x2, or 8 with flag_HD_in; aa1: 2 at x2, 4 with flag_HD_in).  `ref8` is gathered on ITS OWN
        block grid, as the reference does (RefVSR.py:127 passes the full-resolution reference image to aa1)."""
        C, dt = self.mid_channels, self.act_dtype
        ks = self.get_submodule(aa).scale
        H2, W2 = 2 * query_img.shape[1], 2 * query_img.shape[2]
        hq, wq = H2 // ks, W2 // ks
        warped = self._buf(aa + '.wf', (H2, W2, C), dt)
        self.ops.gather_blocks(value, idx, hq, wq, ks, warped)
        wref8 = self._buf(aa + '.wr', (H2, W2, 8), dt)
        self.ops.gather_blocks(ref8, idx, hq, wq, ks, wref8)
        q8 = self._buf(aa + '.q8', (H2, W2, 8), dt)
        self.ops.bicubic_up2_image(query_img, q8)                # alignment.py:41 (no clamp)
        qf = self._align_conv1(aa, q8, self._buf(aa + '.qf', (H2, W2, 32), dt), aa + '.c1q')
        rf = self._align_conv1(aa, wref8, self._buf(aa + '.rf', (H2, W2, 32), dt), aa + '.c1r')
        ha, wa = (H2 + 4 - 5) // ks + 1, (W2 + 4 - 5) // ks + 1
        p0 = self._conv(aa + '.align.p_conv.0', rf, qf, self._buf(aa + '.p0', (ha, wa, 32), dt), [(32, 32), (32, 32)],
                        act_pre=ACT_LRELU02, stride=ks, pad=2)
        p1 = self._resblock(aa + '.align.p_conv.2.conv1', aa + '.align.p_conv.2.conv2', p0, self._buf(aa + '.p1', (ha, wa, 32), dt),
                            self._buf(aa + '.pt', (ha, wa, 32), dt), ACT_LRELU02, ACT_LRELU02)
        affine = self._buf(aa + '.aff', (ha, wa, 3), torch.float32)
        self._conv(aa + '.align.p_conv.4', p1, None, affine, [(32, 32)], act_post=ACT_CLAMP3, pad=0, bias_add=1.0)
        self.ops.aligned_sample(warped, affine, ks, out)
        return out

    def _match_step(self):
        """LR pixels per matching-grid cell along each axis: the nearest x0.5 of flag_HD_in (attention.py:65-67) times the
        max-pool of VGG[0:7] (attention.py:31-40)"""
        return (2 if self.flag_HD_in else 1) * (2 if self.feature_match.vgg_range == 7 else 1)

    def _frame_slot(self, slot, h, w):
        """ring buffers of one frame"""
        C, dt = self.mid_channels, self.act_dtype
        f = self._match_step()
        return {'conf': self._sbuf('ring', f'conf.{slot}', (h, w), torch.float32),
                'idx': self._sbuf('ring', f'idx.{slot}', ((h // f) * (w // f),), torch.int32),
                'aligned': self._sbuf('ring', f'al.{slot}', (h, w, C), dt),
                'aligned_up': self._sbuf('ring', f'alup.{slot}', (2 * h, 2 * w, C), dt),
                'lr8': self._sbuf('ring', f'lr8.{slot}', (h, w, 8), dt)}

    def _frame_alignment(self, lr, ref, slot):
        """Everything the RAP module needs from one (LR, Ref) frame pair, all pure functions of the frame
        (RefVSR.py:196-204,233-234 and the aa1 / aa2 calls of RefVSR.py:127,136): matching confidence, the
        reference features gathered at LR resolution (aa1) and gathered + affinely re-sampled at 2x (aa2),
        plus the NHWC copy of the LR frame.  Computed once per frame, reused by every window that contains it."""
        h, w = lr.shape[1], lr.shape[2]
        fp = self._frame_slot(slot, h, w)
        self._feature_match(lr, ref, fp['conf'], fp['idx'])
        ref8, ref_feat, ref_feat_down = self._ref_features(ref)
        if self.aa1.has_align:                   # x2 / flag_HD_in: aa1 scale 2 / 4 with AlignedConv2d (RefVSR.py:39,125-127)
            lr_down = self._buf('aa1.lrd', (3, h // 2, w // 2), torch.float32)
            self.ops.resize_planes(lr, lr_down, 2.0, mode='bicubic', clamp01=True)
            self._aligned_attention('aa1', lr_down, ref8, fp['idx'], ref_feat_down, fp['aligned'])
        else:
            self.ops.gather_blocks(ref_feat_down, fp['idx'], h, w, self.aa1.scale, fp['aligned'])   # aa1: scale 1, align=False
        self._aligned_attention('aa2', lr, ref8, fp['idx'], ref_feat, fp['aligned_up'])
        self.ops.prep_image(lr, fp['lr8'])
        return fp

    # ---- RAP module (RefVSR.py:123-149) --------------------------------------------------------------
    def _rap(self, fp, conf_prop, feat_prop, feat_prop_UP, tag):
        C, dt = self.mid_channels, self.act_dtype
        conf, aligned, aligned_up = fp['conf'], fp['aligned'], fp['aligned_up']
        h, w = conf.shape[-2:]
        # scratch maps: one set per branch when the two branches may run concurrently (tag = 'bw.rap0' / 'fw.rap1' ...)
        sc = (tag.split('.')[0] + '.rap') if self.overlap_branches else 'rap'
        # level 1 (reference alignment already done per frame, see _frame_alignment)
        cp8 = self._buf(sc + '.cp8', (h, w, 8), dt)
        self.ops.conf_pair(conf_prop, conf, cp8, up2=False)
        a0 = self._conv('conf_fusion.0.0', cp8, None, self._buf(sc + '.a0', (h, w, 16), dt), [(2, 8)], act_pre=ACT_LRELU02)
        alpha = self._conv('conf_fusion.1.0', a0, None, self._buf(sc + '.alpha', (h, w, C), dt), [(16, 16)], act_pre=ACT_LRELU02)
        f0 = self._conv('feat_fusion.0.0', feat_prop, aligned, self._buf(sc + '.f0', (h, w, C), dt), [(C, C), (C, C)],
                        act_pre=ACT_LRELU02)
        fused = self._conv('feat_fusion.1.0', f0, None, self._buf(sc + '.fused', (h, w, C), dt), [(C, C)],
                           act_pre=ACT_LRELU02, gate=alpha, res=feat_prop)
        feat_out = self._buf(tag + '.feat', (h, w, C), dt)
        self._reslist('feat_decoder', 8, fused, feat_out, sc + '.dec1')

        # level 2
        up = self._conv('upsample1.upsample_conv', feat_out, None, self._buf(sc + '.up', (2 * h, 2 * w, C), dt), [(C, C)],
                        pixel_shuffle=True)
        fu = self._conv('feat_fusion2_1.0.0', feat_prop_UP, up, self._buf(sc + '.fu', (2 * h, 2 * w, C), dt),
                        [(C, C), (C, C)], act_pre=ACT_LRELU02)
        cp8u = self._buf(sc + '.cp8u', (2 * h, 2 * w, 8), dt)
        self.ops.conf_pair(conf_prop, conf, cp8u, up2=True)
        b0 = self._conv('conf_fusion2.0.0', cp8u, None, self._buf(sc + '.b0', (2 * h, 2 * w, 16), dt), [(2, 8)], act_pre=ACT_LRELU02)
        alpha2 = self._conv('conf_fusion2.1.0', b0, None, self._buf(sc + '.alpha2', (2 * h, 2 * w, C), dt), [(16, 16)],
                            act_pre=ACT_LRELU02)
        g0 = self._conv('feat_fusion2.0.0', fu, aligned_up, self._buf(sc + '.g0', (2 * h, 2 * w, C), dt), [(C, C), (C, C)],
                        act_pre=ACT_LRELU02)
        fused2 = self._conv('feat_fusion2.1.0', g0, None, self._buf(sc + '.fused2', (2 * h, 2 * w, C), dt), [(C, C)],
                            act_pre=ACT_LRELU02, gate=alpha2, res=fu)
        feat_up_out = self._buf(tag + '.featUP', (2 * h, 2 * w, C), dt)
        self._reslist('feat_decoder2', 4, fused2, feat_up_out, sc + '.dec2')
        conf_out = self._buf(tag + '.conf', (h, w), torch.float32)
        self.ops.conf_max(conf_prop, conf, conf_out)
        return feat_out, feat_up_out, conf_out

    # ---- upsampling tail (RefVSR.py:104-119,288,297) -------------------------------------------------
    def _compute_up(self, bw_up, fw_up, conf_bw, conf_fw, lr_center, clamp01):
        C, dt = self.mid_channels, self.act_dtype
        H2, W2 = bw_up.shape[-3], bw_up.shape[-2]
        h, w = H2 // 2, W2 // 2
        cp8 = self._buf('up.cp8', (H2, W2, 8), dt)
        self.ops.conf_pair(conf_bw, conf_fw, cp8, up2=True)
        base = self._conv('fusion_UP', bw_up, fw_up, self._buf('up.base', (H2, W2, C), dt), [(C, C), (C, C)], pad=0)
        a0 = self._conv('conf_fusion_BWFW.0.0', cp8, None, self._buf('up.a0', (H2, W2, 16), dt), [(2, 8)], act_pre=ACT_LRELU02)
        alpha = self._conv('conf_fusion_BWFW.1.0', a0, None, self._buf('up.alpha', (H2, W2, C), dt), [(16, 16)],
                           act_pre=ACT_LRELU02)
        f0 = self._conv('feat_fusion_BWFW.0.0', bw_up, fw_up, self._buf('up.f0', (H2, W2, C), dt), [(C, C), (C, C)],
                        act_pre=ACT_LRELU02)
        fused = self._conv('feat_fusion_BWFW.1.0', f0, None, self._buf('up.fused', (H2, W2, C), dt), [(C, C)],
                           act_pre=ACT_LRELU02, gate=alpha, res=base)
        dec = self._reslist('feat_decoder_BWFW', 4, fused, self._buf('up.dec', (H2, W2, C), dt), 'up.decs')
        s = self.scale
        if s == 4:
            # lrelu(pixel_shuffle(conv)) == pixel_shuffle(lrelu(conv))  (RefVSR.py:114-115)
            hr = self._conv('upsample2.upsample_conv', dec, None, self._buf('up.hr', (4 * h, 4 * w, C), dt), [(C, C)],
                            act_pre=ACT_LRELU01, pixel_shuffle=True)
        else:
            hr = dec                                             # x2: no upsample2 (RefVSR.py:89-90,114-115)
        hr2 = self._conv('conv_hr', hr, None, self._buf('up.hr2', (s * h, s * w, C), dt), [(C, C)], act_pre=ACT_LRELU01)
        last = self._conv('conv_last', hr2, None, self._buf('up.last', (s * h, s * w, 4), torch.float32), [(C, C)])
        if self._u8 is not None:                                 # the same values, written as 8-bit frames
            out = self._buf('up.out8', frame_shape(s * h, s * w, self._u8), torch.uint8)
            self.ops.reconstruct_u8(last, lr_center, s, clamp01, out, self._u8)
            return out
        out = self._buf('up.out', (3, s * h, s * w), torch.float32)
        self.ops.reconstruct(last, lr_center, s, clamp01, out)      # + bicubic x scale of the centre frame (RefVSR.py:288)
        return out

    # ------------------------------------------------------------------------------------------
    # per-frame products with exact reuse across sliding windows: plan (pure bookkeeping) + execute
    # ------------------------------------------------------------------------------------------
    def _plan_products(self, st, a0, t, range_start):
        """Decide what this window still has to compute and update the bookkeeping.  Frames are addressed by
        their absolute index a = a0 + j (a0 = calls since the stream started); the product of frame / pair
        `a` lives in ring slot a % t.  Returns a list of ('pyr'|'fw'|'bw'|'frame', a)."""
        mid = t // 2
        for name in ('pyr', 'fw', 'bw', 'frame'):
            st[name] = {a for a in st[name] if a >= a0}
        work = []

        def need_pyr(a):
            if a not in st['pyr']:
                st['pyr'].add(a)
                work.append(('pyr', a))

        ev = _cget(self.config, 'EVAL', None)
        zero_flow = bool(_cget(ev, 'is_gradio', False)) if ev is not None else False   # RefVSR.py:183-191
        # flows actually consumed by this call (the reference computes all 2(t-1), RefVSR.py:179-193)
        need_fw = sorted(set(range(range_start, mid)) | ({mid} if mid < t - 1 else set()))
        need_bw = list(range(mid, t - 1))
        for j in need_fw:            # forward_flows[j] = Flow(lrs[j+1], lrs[j])   (RefVSR.py:182-184)
            if a0 + j not in st['fw']:
                if not zero_flow:
                    need_pyr(a0 + j + 1)
                    need_pyr(a0 + j)
                st['fw'].add(a0 + j)
                work.append(('fw0' if zero_flow else 'fw', a0 + j))
        for j in need_bw:            # backward_flows[j] = Flow(lrs[j], lrs[j+1])  (RefVSR.py:187-189)
            if a0 + j not in st['bw']:
                if not zero_flow:
                    need_pyr(a0 + j)
                    need_pyr(a0 + j + 1)
                st['bw'].add(a0 + j)
                work.append(('bw0' if zero_flow else 'bw', a0 + j))
        for j in range(range_start, t):
            if a0 + j not in st['frame']:
                st['frame'].add(a0 + j)
                work.append(('frame', a0 + j))
        return work

    def _rm(self, t):
        """ring length: T per-frame slots for the windowed forward, (owned frames + T - 1) for a frame-sharded clip"""
        return self._ring_mod or t

    def _ring(self, kind, a, t, shape, dtype=torch.float32):
        return self._sbuf('ring', f'{kind}.{a % self._rm(t)}', shape, dtype)

    def _run_products(self, work, t, h, w, hr, wr):
        """Pyramids first, then the flows and the per-frame alignment products, which are independent of each other.  With
        b200_overlap_branches the flows (~60 launches of SPyNet's small convs per steady window: grids of 2 - 75 CTAs) go to two
        side streams - alternating, each with its own scratch maps - and fill the SMs the matching / alignment kernels of the
        main stream leave idle; everything is joined before this returns.  Same kernels and inputs: bit-identical."""
        def flow(kind, a, sp):
            pa = [self._sbuf('ring', f'pyr{l}.{a % self._rm(t)}', (H, W, 3), torch.float32) for l, (H, W) in enumerate(self._pyr_shapes(h, w))]
            pb = [self._sbuf('ring', f'pyr{l}.{(a + 1) % self._rm(t)}', (H, W, 3), torch.float32) for l, (H, W) in enumerate(self._pyr_shapes(h, w))]
            out = self._ring(kind, a, t, (h, w, 2))
            if kind == 'fw':
                self._spynet(pb, pa, out, sp)      # Flow(frame a+1, frame a)
            else:
                self._spynet(pa, pb, out, sp)      # Flow(frame a, frame a+1)

        for kind, a in work:
            if kind == 'pyr':
                self._pyramid(self._ring('lr32', a, t, (3, h, w)), a % self._rm(t))
        flows = [(kind, a) for kind, a in work if kind in ('fw', 'bw')]
        par = self.overlap_branches and self._device.type == 'cuda' and len(flows) > 0 and not self.use_chain
        used = []
        if par:
            main = torch.cuda.current_stream()
            if self._flow_streams is None:
                self._flow_streams = [torch.cuda.Stream(device=self._device) for _ in range(2)]
            for n, (kind, a) in enumerate(flows):
                st_ = self._flow_streams[n % 2]
                if st_ not in used:
                    st_.wait_stream(main)              # fork behind the pyramids
                    used.append(st_)
                with torch.cuda.stream(st_):
                    flow(kind, a, f'spy{n % 2}')
        else:
            for kind, a in flows:
                flow(kind, a, 'spy')
        for kind, a in work:
            if kind in ('fw0', 'bw0'):
                self._ring(kind[:2], a, t, (h, w, 2)).zero_()
            elif kind == 'frame':
                self._frame_alignment(self._ring('lr32', a, t, (3, h, w)), self._ring('ref32', a, t, (3, hr, wr)), a % self._rm(t))
        for st_ in used:
            torch.cuda.current_stream().wait_stream(st_)                # join

    # ------------------------------------------------------------------------------------------
    # forward (RefVSR.py:151-325)
    # ------------------------------------------------------------------------------------------
    def forward(self, lrs, refs, is_first_frame, is_log=False, is_train=False):
        """lrs / refs (n, t, 3, h, w) / (n, t, 3, hr, wr) -> outs['result'] (n, 3, scale*h, scale*w).  n > 1 windows run as ONE
        window schedule: the per-frame products (SPyNet, matching, alignment) once per element, every propagation step and the
        upsampling tail once for the whole batch, in one CUDA graph, bit-identical to running each element alone.  Elements whose
        schedules differ (e.g. the reuse guard finds that one did not slide) run one by one instead (`batch_fallbacks`), as do
        is_log / is_train calls.  A stream keeps its batch size: a call with another n starts new streams (is_first_frame)."""
        outs = collections.OrderedDict()
        if is_log:
            outs['vis'] = collections.OrderedDict()
        if lrs.dim() != 5 or refs.dim() != 5:
            raise ValueError('lrs / refs must be (n, t, c, h, w)')
        n, t, c, h, w = lrs.size()
        if c != 3 or refs.size(2) != 3 or refs.size(1) != t or refs.size(0) != n:
            raise ValueError(f'unexpected input shapes {tuple(lrs.shape)} / {tuple(refs.shape)}')
        self._check_sizes(h, w, refs.size(3), refs.size(4))
        out, vis = self._call(lrs, refs, n, is_first_frame, is_log, is_train)
        outs['result'] = out
        if is_log and vis is not None:
            outs['vis'].update(vis.get('vis', {}))
            if _cget(self.config, 'save_sample', False) and 'eval_vis' in vis:
                outs['eval_vis'] = vis['eval_vis']
        return outs

    def _check_sizes(self, h, w, hr, wr):
        """the LR (h, w) / Ref (hr, wr) sizes the schedule computes what the reference computes for"""
        if hr % 2 or wr % 2:
            raise ValueError('reference frames must have even height/width (2x2 avg-pool and 2x2 block '
                             'gather, attention.py:51,142-144; odd sizes take the reference\'s reflection-'
                             'padded unfold path, which is not implemented)')
        if self.flag_HD_in and (h % 4 or w % 4 or hr % 8 or wr % 8):
            raise ValueError('flag_HD_in: LR height/width must be multiples of 4 and Ref height/width multiples of 8 '
                             '(4x4 / 8x8 alignment blocks on the 1/4-resolution matching grid, attention.py:142-154); '
                             f'got LR {h}x{w}, Ref {hr}x{wr}')
        if self.scale == 2 and (h % 2 or w % 2 or hr % 4 or wr % 4):
            raise ValueError('scale=2: LR height/width must be even and Ref height/width multiples of 4 '
                             '(2x2 / 4x4 alignment blocks on the 1/2-resolution matching grid, attention.py:142-154); '
                             f'got LR {h}x{w}, Ref {hr}x{wr}')

    def _call(self, lrs, refs, n, is_first_frame, is_log, is_train):
        """one call of n windows (forward / forward_u8) once its inputs are checked -> (result, vis)"""
        self._device = lrs.device
        if is_train and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            # trainers/trainer.py:159-172 would call loss.backward() on the result: fail here, with a clear message
            raise NotImplementedError('refvsr_b200 is inference only: forward(is_train=True) builds no autograd graph '
                                      '(call it under torch.no_grad() for a training-mode forward without gradients)')
        if n != self._bn:
            # the ring slots and carried state of a call of n windows are [n][...] tensors: another n starts new streams
            self._state.clear()
            self._bn = n

        caller_first = bool(is_first_frame)
        if not is_train:                                                     # RefVSR.py:168-170
            if self.max_frame_itr_num is not None and self.frame_itr_num == self.max_frame_itr_num:
                is_first_frame = True

        with torch.no_grad():
            results, vis = [], None
            if n > 1 and self._batchable(is_log, is_train):
                fresh, shape = self._batch_fresh(lrs, refs, caller_first)
                out = self._run_batch(fresh, [lrs[b] for b in range(n)], [refs[b] for b in range(n)], shape,
                                      bool(is_first_frame))
            else:
                for b in range(n):
                    res_b, vis_b = self._forward_one(b, lrs[b], refs[b], bool(is_first_frame), caller_first,
                                                     bool(is_log), bool(is_train))
                    results.append(res_b)
                    vis = vis_b if vis is None else vis
                out = torch.stack(results, 0)

        if not is_train:                                                     # RefVSR.py:292-297
            if is_first_frame:
                self.frame_itr_num = 0
            self.frame_itr_num += 1
        return out, vis

    def _batchable(self, is_log, is_train):
        """n > 1 windows can share one schedule: an operator set that takes (n, ...) operands, and none of the per-element-only
        options (debug outputs, training mode, the opt-in fused residual-block / chain kernels)"""
        return (getattr(self.ops, 'batched', False) and not is_log and not is_train and not self.use_chain
                and not self.fuse_resblocks and self._ring_mod is None)

    def _push_state(self, b, lr, ref):
        if self._u8 is None and (lr.dim() != 3 or ref.dim() != 3 or lr.size(0) != 3 or ref.size(0) != 3):
            raise ValueError('push_frame takes one LR frame (3, h, w) and one Ref frame (3, hr, wr)')
        st = self._state.get(b)
        if st is None or not st.get('has_prev') or not self.reuse:
            raise RuntimeError('push_frame needs a previous forward() call (the first window of the clip) and b200_reuse=True')
        t, h, w, hr, wr = st['shape']
        if self._hw(lr) != (h, w) or self._hw(ref) != (hr, wr) or lr.device != self._device:
            raise ValueError(f'push_frame: frame shapes / device differ from the running stream {(h, w)} / {(hr, wr)} on {self._device}')
        return st

    def push_frame(self, lr, ref, b=0):
        """Streaming entry (SURVEY 8f row 2: a decoded-frame ring buffer feeding the per-frame pipeline): the window slides by one
        and ONLY the entering frame is handed over - lr (3, h, w), ref (3, hr, wr) in [0, 1], the frame that would have been
        lrs[b, t-1] / refs[b, t-1] of the next forward() call.  The other t-1 frames are the engine's own staged ring slots, so there
        is nothing to verify (no reuse-guard launch, no host sync) and the caller moves 1/t of the window's bytes.  Returns the
        same tensor forward()['result'][b] would: (3, scale*h, scale*w).  Needs a previous forward() call on this batch slot (the clip's first
        window, is_first_frame=True); forced resets (reset_branch) follow the same counter as forward()."""
        st = self._push_state(b, lr, ref)
        t = st['shape'][0]
        is_first_frame = self.max_frame_itr_num is not None and self.frame_itr_num == self.max_frame_itr_num   # RefVSR.py:168-170
        self._b = b
        win_lr, win_ref = _NewestOnly(lr, t), _NewestOnly(ref, t)
        with torch.no_grad():
            out, _ = self._do_window(b, st, False, win_lr, win_ref, st['shape'], bool(is_first_frame), False, False)
        if is_first_frame:                                                   # RefVSR.py:292-297
            self.frame_itr_num = 0
        self.frame_itr_num += 1
        return out

    def push_frames(self, lrs, refs):
        """push_frame for all n windows of the running batch at once: lrs (n, 3, h, w), refs (n, 3, hr, wr), element b being
        the frame entering window b.  The same contract per element as push_frame; returns what forward()['result'] would,
        (n, 3, scale*h, scale*w), computed by one batched window schedule like forward()."""
        fdims = 3 if self._u8 is None else len(frame_shape(2, 2, self._u8))     # the dimensions of one frame
        if lrs.dim() != fdims + 1 or refs.dim() != fdims + 1 or lrs.size(0) != refs.size(0):
            raise ValueError('push_frames takes LR frames (n, 3, h, w) and Ref frames (n, 3, hr, wr)')
        n = lrs.size(0)
        if n != self._bn:
            raise ValueError(f'push_frames: {n} frames for a stream of {self._bn} windows')
        sts = [self._push_state(b, lrs[b], refs[b]) for b in range(n)]
        shape = sts[0]['shape']
        t = shape[0]
        is_first_frame = self.max_frame_itr_num is not None and self.frame_itr_num == self.max_frame_itr_num   # RefVSR.py:168-170
        with torch.no_grad():
            wl, wr = [_NewestOnly(lrs[b], t) for b in range(n)], [_NewestOnly(refs[b], t) for b in range(n)]
            if n > 1 and self._batchable(False, False):
                out = self._run_batch([False] * n, wl, wr, shape, bool(is_first_frame))
            else:
                outs = []
                for b in range(n):
                    self._b = b
                    outs.append(self._do_window(b, sts[b], False, wl[b], wr[b], shape, bool(is_first_frame), False, False)[0])
                out = torch.stack(outs, 0)
        if is_first_frame:                                                   # RefVSR.py:292-297
            self.frame_itr_num = 0
        self.frame_itr_num += 1
        return out

    # ---- 8-bit frames (no counterpart in the reference) ---------------------------------------------
    # Video decoders hand out uint8 HWC frames and encoders take them back.  These entries accept and return such frames, so a
    # caller converts nothing on the host: the entering frames go through rv_frames_from_u8 straight into the fp32 ring slots
    # (byte u -> fl32(u / 255), the value forward() stages from u8.float() / 255), and the tail's rv_reconstruct_u8 writes the
    # bytes of the fp32 result forward() returns (csrc/frame_u8.cuh).  The schedule, the stream state and the ring are forward()'s,
    # so 8-bit and fp32 calls may be interleaved on one clip.

    def forward_u8(self, lrs, refs, is_first_frame, bgr=False):
        """forward() for 8-bit frames: lrs (n, t, h, w, 3), refs (n, t, hr, wr, 3), contiguous uint8 on the engine's device; bgr:
        B, G, R byte order (cv2's) in and out.  -> (n, scale*h, scale*w, 3) uint8: frame_u8 of forward()['result'] for the frames
        u8.float() / 255, as HWC bytes."""
        self._check_u8('forward_u8', 'lrs', lrs, 5)
        self._check_u8('forward_u8', 'refs', refs, 5)
        n, t, h, w, _ = lrs.shape
        if tuple(refs.shape[:2]) != (n, t):
            raise ValueError(f'forward_u8: lrs {tuple(lrs.shape)} and refs {tuple(refs.shape)} differ in (n, t)')
        self._check_sizes(h, w, refs.shape[2], refs.shape[3])
        with self._frames_u8(bool(bgr)):
            return self._call(lrs, refs, n, is_first_frame, False, False)[0]

    def push_frame_u8(self, lr, ref, bgr=False, b=0):
        """push_frame() for 8-bit frames: lr (h, w, 3), ref (hr, wr, 3) contiguous uint8 -> (scale*h, scale*w, 3) uint8"""
        self._check_u8('push_frame_u8', 'lr', lr, 3)
        self._check_u8('push_frame_u8', 'ref', ref, 3)
        with self._frames_u8(bool(bgr)):
            return self.push_frame(lr, ref, b)

    def push_frames_u8(self, lrs, refs, bgr=False):
        """push_frames() for 8-bit frames: lrs (n, h, w, 3), refs (n, hr, wr, 3) contiguous uint8 -> (n, scale*h, scale*w, 3) uint8"""
        self._check_u8('push_frames_u8', 'lrs', lrs, 4)
        self._check_u8('push_frames_u8', 'refs', refs, 4)
        with self._frames_u8(bool(bgr)):
            return self.push_frames(lrs, refs)

    # ---- YUV 4:2:0 frames (no counterpart in the reference) ------------------------------------------
    # Video decoders and encoders mostly work in 4:2:0: ffmpeg's yuv420p is I420, hardware codecs use NV12.  These entries take and
    # return such frames as the (3h/2, w) uint8 arrays cv2 uses, converted on the GPU at the same two points as the 8-bit entries:
    # rv_frames_from_u8 turns an entering frame into the fp32 values of the RGB bytes cv2.cvtColor(COLOR_YUV2RGB_I420 / _NV12)
    # gives, and rv_reconstruct_u8 writes cv2.cvtColor(COLOR_RGB2YUV_I420) of the RGB bytes forward_u8 returns (interleaved for
    # NV12).  Everything else is forward_u8's: schedule, stream state, ring; fp32, 8-bit and 4:2:0 calls may be interleaved.

    def forward_yuv420(self, lrs, refs, is_first_frame, nv12=False):
        """forward() for 4:2:0 frames: lrs (n, t, 3h/2, w), refs (n, t, 3hr/2, wr), contiguous uint8 on the engine's device, I420
        (Y plane, U plane, V plane) or with nv12 NV12 (Y plane, interleaved U, V rows), LR and Ref alike.  -> (n, 3H/2, W) uint8
        frames of the same layout, (H, W) = (scale*h, scale*w): the 4:2:0 frames of forward_u8's RGB result for the RGB frames
        cv2 makes of lrs / refs."""
        self._check_yuv420('forward_yuv420', 'lrs', lrs, 4)
        self._check_yuv420('forward_yuv420', 'refs', refs, 4)
        n, t = lrs.shape[:2]
        if tuple(refs.shape[:2]) != (n, t):
            raise ValueError(f'forward_yuv420: lrs {tuple(lrs.shape)} and refs {tuple(refs.shape)} differ in (n, t)')
        self._check_sizes(2 * lrs.shape[2] // 3, lrs.shape[3], 2 * refs.shape[2] // 3, refs.shape[3])
        with self._frames_u8(FRAME_NV12 if nv12 else FRAME_I420):
            return self._call(lrs, refs, n, is_first_frame, False, False)[0]

    def push_frame_yuv420(self, lr, ref, nv12=False, b=0):
        """push_frame() for 4:2:0 frames: lr (3h/2, w), ref (3hr/2, wr) contiguous uint8 -> (3H/2, W) uint8"""
        self._check_yuv420('push_frame_yuv420', 'lr', lr, 2)
        self._check_yuv420('push_frame_yuv420', 'ref', ref, 2)
        with self._frames_u8(FRAME_NV12 if nv12 else FRAME_I420):
            return self.push_frame(lr, ref, b)

    def push_frames_yuv420(self, lrs, refs, nv12=False):
        """push_frames() for 4:2:0 frames: lrs (n, 3h/2, w), refs (n, 3hr/2, wr) contiguous uint8 -> (n, 3H/2, W) uint8"""
        self._check_yuv420('push_frames_yuv420', 'lrs', lrs, 3)
        self._check_yuv420('push_frames_yuv420', 'refs', refs, 3)
        with self._frames_u8(FRAME_NV12 if nv12 else FRAME_I420):
            return self.push_frames(lrs, refs)

    def _check_yuv420(self, fn, name, x, dims):
        if not isinstance(x, torch.Tensor) or x.dtype != torch.uint8:
            raise ValueError(f'{fn}: {name} must be a uint8 tensor, got {getattr(x, "dtype", type(x).__name__)}')
        if x.dim() != dims or x.shape[-2] % 3 or x.shape[-2] == 0 or x.shape[-1] % 2 or x.shape[-1] == 0:
            raise ValueError(f'{fn}: {name} must be {dims}-d 4:2:0 frames of (3h/2, w) rows and columns, h and w even, '
                             f'got {tuple(x.shape)}')
        if not x.is_contiguous():
            raise ValueError(f'{fn}: {name} must be contiguous')
        dev = next(self.parameters()).device
        if x.device != dev:
            raise ValueError(f'{fn}: {name} is on {x.device}, the engine on {dev}')

    def _check_u8(self, fn, name, x, dims):
        if not isinstance(x, torch.Tensor) or x.dtype != torch.uint8:
            raise ValueError(f'{fn}: {name} must be a uint8 tensor, got {getattr(x, "dtype", type(x).__name__)}')
        if x.dim() != dims or x.shape[-1] != 3:
            raise ValueError(f'{fn}: {name} must be {dims}-d with the 3 channels last (HWC frames), got {tuple(x.shape)}')
        if not x.is_contiguous():
            raise ValueError(f'{fn}: {name} must be contiguous')
        dev = next(self.parameters()).device
        if x.device != dev:
            raise ValueError(f'{fn}: {name} is on {x.device}, the engine on {dev}')

    @contextlib.contextmanager
    def _frames_u8(self, fmt):
        self._u8 = fmt
        try:
            yield
        finally:
            self._u8 = None

    def _hw(self, x):
        """(h, w) of a frame or a stack of frames: (..., 3, h, w) fp32, or inside an 8-bit call (..., h, w, 3) uint8 HWC or
        (..., 3h/2, w) uint8 4:2:0"""
        if self._u8 is None:
            return tuple(x.shape[-2:])
        if self._u8 in (FRAME_I420, FRAME_NV12):
            return (2 * x.shape[-2] // 3, x.shape[-1])
        return tuple(x.shape[-3:-1])

    def _is_fresh(self, b, lrs, refs, caller_first, is_train):
        """(state, fresh, shape) of batch element b's stream: fresh = its cached per-frame products cannot be reused"""
        t, (h, w), (hr, wr) = lrs.shape[0], self._hw(lrs), self._hw(refs)
        self._b = b           # ring / state namespace of this batch element

        # stream bookkeeping for exact reuse: a caller-declared first frame starts a new stream; forced
        # resets (reset_branch) keep sliding, so the caches stay valid across them.
        st = self._state.get(b)
        shape = (t, h, w, hr, wr)
        fresh = (st is None or caller_first or not self.reuse or is_train or st.get('shape') != shape)
        if not fresh and self.reuse_check != 'off':
            fresh = not self._window_slid_by_one(st, lrs, refs, t, h, w, hr, wr)
        return st, fresh, shape

    def _batch_fresh(self, lrs, refs, caller_first):
        """_is_fresh for the n elements of a batched call; with b200_reuse_check='sync' the n reuse-guard verdicts are read back
        in ONE device-to-host copy (one host sync per call, not per element).  -> ([fresh per element], shape)"""
        n, t, (h, w), (hr, wr) = lrs.shape[0], lrs.shape[1], self._hw(lrs), self._hw(refs)
        shape = (t, h, w, hr, wr)
        fresh, pending = [], []
        for b in range(n):
            if self.reuse_check != 'sync':
                fresh.append(self._is_fresh(b, lrs[b], refs[b], caller_first, False)[1])
                continue
            self._b = b
            st = self._state.get(b)
            f = st is None or caller_first or not self.reuse or st.get('shape') != shape
            if not f:
                pending.append((b, self._enqueue_overlap_compare(st, lrs[b], refs[b], t, h, w, hr, wr)))
            fresh.append(f)
        if pending:
            for (b, _), differs in zip(pending, torch.cat([flag for _, flag in pending]).tolist()):
                if differs:                   # the staged frames of the previous call are the reference
                    self.reuse_fallbacks += 1
                    fresh[b] = True
        return fresh, shape

    def _forward_one(self, b, lrs, refs, is_first_frame, caller_first, is_log, is_train):
        st, fresh, shape = self._is_fresh(b, lrs, refs, caller_first, is_train)
        return self._do_window(b, st, fresh, lrs, refs, shape, is_first_frame, is_log, is_train)

    def _prepare_window(self, b, st, fresh, lrs, refs, shape, is_first_frame, is_train, a0_fresh=0):
        """Bookkeeping of element b's next window: stream position, staging of the entering frames, product work list.
        A fresh stream starts at position a0_fresh (any value: only a % t addresses the ring)."""
        t, h, w, hr, wr = shape
        mid = t // 2
        if fresh:
            st = {'a0': a0_fresh, 'pyr': set(), 'fw': set(), 'bw': set(), 'frame': set(), 'staged': set(),
                  'has_prev': bool(st and st.get('has_prev')) and st.get('shape') == shape, 'shape': shape}
            self._state[b] = st
        else:
            st['a0'] += 1
        a0 = st['a0']

        if is_first_frame:
            range_start = 0
        else:
            range_start = mid if not is_train else 0                          # RefVSR.py:173-176
            if not st['has_prev']:
                raise RuntimeError('is_first_frame=False but no propagated state exists '
                                   '(the reference fails the same way: RefVSR.py:256-260)')

        # stage the frames that entered the window into their ring slots (fp32 copies; outside any graph)
        st['staged'] = {a for a in st['staged'] if a >= a0}
        enter = [j for j in range(t) if a0 + j not in st['staged']]
        if self._u8 is None:
            for j in enter:
                self._ring('lr32', a0 + j, t, (3, h, w)).copy_(lrs[j])
                self._ring('ref32', a0 + j, t, (3, hr, wr)).copy_(refs[j])
        elif enter:                                   # 8-bit frames: converted straight into their slots, one launch per size
            self.ops.frames_from_u8([lrs[j] for j in enter], [self._ring('lr32', a0 + j, t, (3, h, w)) for j in enter], self._u8)
            self.ops.frames_from_u8([refs[j] for j in enter], [self._ring('ref32', a0 + j, t, (3, hr, wr)) for j in enter], self._u8)
        st['staged'].update(a0 + j for j in enter)

        work = self._plan_products(st, a0, t, range_start)
        return st, a0, range_start, work

    def _execute(self, key, fn):
        """fn() enqueues one window and returns (static output, vis).  key None: run eagerly; otherwise the window is captured
        into a CUDA graph once per key and replayed."""
        if key is None:
            n0 = self.ops.launch_count()
            out_static, vis = fn()
            self.executed_kernels += self.ops.launch_count() - n0
            return out_static.clone(), vis
        entry = self._graphs.get(key)
        if entry is None:
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            n0 = self.ops.launch_count()
            with torch.cuda.graph(graph):
                out_static, _ = fn()
            entry = (graph, out_static, self.ops.launch_count() - n0)
            self._graphs[key] = entry
        entry[0].replay()
        self.executed_kernels += entry[2]          # kernel nodes of librefvsr_b200.so replayed by the graph
        return entry[1].clone(), None

    def _graph_ok(self, fresh, is_log, is_train, lrs):
        return (self.use_graphs and not fresh and not is_log and not is_train and lrs.is_cuda
                and hasattr(torch.cuda, 'CUDAGraph'))

    def _do_window(self, b, st, fresh, lrs, refs, shape, is_first_frame, is_log, is_train):
        t, h, w, hr, wr = shape
        st, a0, range_start, work = self._prepare_window(b, st, fresh, lrs, refs, shape, is_first_frame, is_train)
        variant = 'first' if is_first_frame else 'steady'
        key = None
        if self._graph_ok(fresh, is_log, is_train, lrs):
            key = (b, self._bn, shape, a0 % t, variant, tuple((k, a - a0) for k, a in work), self._u8)
        out, vis = self._execute(key, lambda: self._run_window(b, st, a0, t, h, w, hr, wr, work, is_first_frame, range_start,
                                                                is_log, is_train))
        st['has_prev'] = True
        return out, vis

    def _run_batch(self, fresh, lrs, refs, shape, is_first_frame):
        """One window for each of the n elements (lrs[b] / refs[b]: element b's window frames).  When every element has the same
        schedule (same ring phase, product work and fresh decision) the products are enqueued per element and every step once
        for the batch; otherwise each element runs alone.  -> (n, 3, scale*h, scale*w)"""
        n = len(fresh)
        t, h, w, hr, wr = shape
        # a stream that starts afresh takes the ring phase of the batch's sliding streams, so that their next windows line up
        slid = [self._state[b]['a0'] + 1 for b in range(n) if not fresh[b]]
        preps = []
        for b in range(n):
            self._b = b
            preps.append(self._prepare_window(b, self._state.get(b), fresh[b], lrs[b], refs[b], shape, is_first_frame, False,
                                              slid[0] if slid else 0))
        sigs = {(a0 % t, rs, tuple((k, a - a0) for k, a in work)) for _, a0, rs, work in preps}
        variant = 'first' if is_first_frame else 'steady'
        if len(sigs) > 1 or len(set(fresh)) > 1:
            self.batch_fallbacks += 1
            outs = []
            for b, (st, a0, rs, work) in enumerate(preps):
                self._b = b
                key = None
                if self._graph_ok(fresh[b], False, False, lrs[b]):
                    key = (b, self._bn, shape, a0 % t, variant, tuple((k, a - a0) for k, a in work), self._u8)
                outs.append(self._execute(key, lambda: self._run_window(b, st, a0, t, h, w, hr, wr, work, is_first_frame, rs,
                                                                         False, False))[0])
                st['has_prev'] = True
            return torch.stack(outs, 0)

        st0, a0, range_start, work = preps[0]

        def products():
            # per element: SPyNet, matching and the alignment products (each writes its slice of the ring)
            self._bmode = False
            try:
                for b, p in enumerate(preps):
                    self._b = b
                    self._run_products(p[3], t, h, w, hr, wr)
            finally:
                self._bmode = True

        key = None
        if self._graph_ok(fresh[0], False, False, lrs[0]):
            key = ('batch', n, shape, a0 % t, variant, tuple((k, a - a0) for k, a in work), self._u8)
        self._bmode = True
        try:
            out, _ = self._execute(key, lambda: self._run_window(0, st0, a0, t, h, w, hr, wr, work, is_first_frame, range_start,
                                                                  False, False, products=products))
        finally:
            self._bmode = False
        for st, *_ in preps:
            st['has_prev'] = True
        return out

    def _enqueue_overlap_compare(self, st, lrs, refs, t, h, w, hr, wr):
        """Reuse guard, device side: frames 0..t-2 of this call must be frames 1..t-1 of the previous one, i.e. equal to the
        staged ring slots a0+1 .. a0+t-1 (bitwise: the slots are fp32 copies of what the caller passed).  Enqueues the comparison;
        returns the int32 device flag (non-zero = the window did NOT slide by one)."""
        flag = self._buf(f'reuse.flag{self._b}', (1,), torch.int32)
        a1 = st['a0'] + 1
        # 8-bit frames: compare their fp32 values.  For RGB / BGR bytes the conversion is one to one, so equal values <=> equal
        # bytes; the YUV -> RGB map of 4:2:0 frames is not (Y bytes below 16 and saturated channels give
        # equal RGB bytes for different frames), and equal values are what reuse needs, so comparing bytes would refuse some windows that can be reused.
        if self._u8 is not None:
            lr32 = self._buf(f'reuse.lr32.{self._b}', (t - 1, 3, h, w), torch.float32)
            rf32 = self._buf(f'reuse.ref32.{self._b}', (t - 1, 3, hr, wr), torch.float32)
            self.ops.frames_from_u8([lrs[j] for j in range(t - 1)], [lr32[j] for j in range(t - 1)], self._u8)
            self.ops.frames_from_u8([refs[j] for j in range(t - 1)], [rf32[j] for j in range(t - 1)], self._u8)
        else:
            lr32 = lrs if (lrs.dtype == torch.float32 and lrs.is_contiguous()) else lrs.float().contiguous()
            rf32 = refs if (refs.dtype == torch.float32 and refs.is_contiguous()) else refs.float().contiguous()
        pairs = []
        for j in range(t - 1):
            pairs.append((lr32[j], self._ring('lr32', a1 + j, t, (3, h, w))))
            pairs.append((rf32[j], self._ring('ref32', a1 + j, t, (3, hr, wr))))
        for i in range(0, len(pairs), 16):
            chunk = pairs[i:i + 16]
            if i == 0:
                self.ops.frames_differ(chunk, flag)
            else:
                flag2 = self._buf(f'reuse.flag{self._b}.{i}', (1,), torch.int32)
                self.ops.frames_differ(chunk, flag2)
                flag.bitwise_or_(flag2)
        return flag

    def _window_slid_by_one(self, st, lrs, refs, t, h, w, hr, wr):
        """Reuse guard, host side.  Returns False when the cached per-frame products must not be reused for this call."""
        flag = self._buf(f'reuse.flag{self._b}', (1,), torch.int32)
        if self.reuse_check == 'async' and st.get('check_pending'):
            st['check_pending'] = False
            if int(flag.item()):
                self.reuse_fallbacks += 1
                raise RuntimeError('refvsr_b200: the previous call did not slide the window by one frame '
                                   '(is_first_frame=False with different overlapping frames); its output reused stale '
                                   "per-frame products.  Pass is_first_frame=True for a new clip or set b200_reuse_check='sync'")
        flag = self._enqueue_overlap_compare(st, lrs, refs, t, h, w, hr, wr)
        if self.reuse_check == 'async':
            st['check_pending'] = True
            return True
        if int(flag.item()):          # one small host sync per call; the staged frames of the previous call are the reference
            self.reuse_fallbacks += 1
            return False
        return True

    def _warp3_ok(self):
        return self.act_dtype != torch.float32 and hasattr(self.ops, 'warp3') and not os.environ.get('REFVSR_NO_WARP3')

    def _backward_branch(self, a0, t, h, w, vis=None, after_step=None):
        """backward branch of the window at stream position a0 (RefVSR.py:211-238): window-local, starts from zeros at the
        window's last frame -> (feat_prop_UP, conf_map_prop) buffers at the centre frame"""
        ops = self.ops
        C, dt = self.mid_channels, self.act_dtype
        mid = t // 2
        feat_prop = self._buf('bw.z.feat', (h, w, C), dt).zero_()
        feat_prop_UP = self._buf('bw.z.featUP', (2 * h, 2 * w, C), dt).zero_()
        conf_prop = self._buf('bw.z.conf', (h, w), torch.float32).zero_()
        for i in range(t - 1, mid - 1, -1):
            if i < t - 1:
                flow = self._ring('bw', a0 + i, t, (h, w, 2))
                wf = self._buf('bw.w.feat', (h, w, C), dt)
                wc = self._buf('bw.w.conf', (h, w), torch.float32)
                wu = self._buf('bw.w.featUP', (2 * h, 2 * w, C), dt)
                if self._warp3_ok():
                    ops.warp3(feat_prop, feat_prop_UP, conf_prop, flow, wf, wu, wc)     # one launch, one flow read
                else:
                    ops.warp(feat_prop, flow, wf)
                    ops.warp(conf_prop, flow, wc)
                    ops.warp(feat_prop_UP, flow, wu, flow_up2=True)            # RefVSR.py:220
                feat_prop, conf_prop, feat_prop_UP = wf, wc, wu
                if vis is not None and i == mid:
                    vis['vis']['BW_LR_next_warp'] = self._warp_image(self._ring('lr32', a0 + i + 1, t, (3, h, w)), flow)
            fp = self._frame_slot((a0 + i) % self._rm(t), h, w)
            agg = self._prop_resblocks('backward_resblocks', fp['lr8'], feat_prop,
                                       self._buf('bw.agg', (h, w, C), dt), 'bw.rb')
            feat_prop, feat_prop_UP, conf_prop = self._rap(fp, conf_prop, agg, feat_prop_UP, f'bw.rap{i % 2}')
            if after_step is not None:
                after_step(t - 1 - i)
        return feat_prop_UP, conf_prop

    def _forward_step(self, a, t, h, w, state, flow, quirk, tagi):
        """One forward-branch step at stream position `a` (RefVSR.py:248-277).  `state` = (feat, featUP, conf) or None (start
        from zeros, no warp).  quirk=True: the step follows another step of the SAME call - the reference then warps the
        already-warped LR-resolution feat_prop onto the 2x grid and drops the propagated feat_prop_UP (RefVSR.py:252-254);
        quirk=False: the state comes from the previous call and feat_prop_UP is warped itself (RefVSR.py:256-260)."""
        ops = self.ops
        C, dt = self.mid_channels, self.act_dtype
        if state is None:
            feat_prop = self._buf('fw.z.feat', (h, w, C), dt).zero_()
            feat_prop_UP = self._buf('fw.z.featUP', (2 * h, 2 * w, C), dt).zero_()
            conf_prop = self._buf('fw.z.conf', (h, w), torch.float32).zero_()
        else:
            feat, featUP, conf = state
            wf = self._buf('fw.w.feat', (h, w, C), dt)
            wu = self._buf('fw.w.featUP', (2 * h, 2 * w, C), dt)
            wc = self._buf('fw.w.conf', (h, w), torch.float32)
            if not quirk and self._warp3_ok():
                ops.warp3(feat, featUP, conf, flow, wf, wu, wc)
            else:
                ops.warp(feat, flow, wf)
                ops.warp(wf if quirk else featUP, flow, wu, flow_up2=True)
                ops.warp(conf, flow, wc)
            feat_prop, feat_prop_UP, conf_prop = wf, wu, wc
        fp = self._frame_slot(a % self._rm(t), h, w)
        agg = self._prop_resblocks('forward_resblocks', fp['lr8'], feat_prop, self._buf('fw.agg', (h, w, C), dt), 'fw.rb')
        return self._rap(fp, conf_prop, agg, feat_prop_UP, f'fw.rap{tagi % 2}')

    def _run_window(self, b, st, a0, t, h, w, hr, wr, work, is_first_frame, range_start, is_log, is_train, products=None):
        """All kernel launches of one window.  Reads / writes static buffers only (graph-capturable).  products: enqueues the
        per-frame products (default: this element's work list); in a batched window it runs them for every element."""
        C, dt = self.mid_channels, self.act_dtype
        mid = t // 2
        vis = {'vis': collections.OrderedDict()} if is_log else None
        if products is None:
            def products():
                self._run_products(work, t, h, w, hr, wr)

        def lr32(i):
            return self._ring('lr32', a0 + i, t, (3, h, w))

        if is_first_frame:
            range_start = 0
        prev = {'feat': self._sbuf('prev', 'feat', (h, w, C), dt), 'featUP': self._sbuf('prev', 'featUP', (2 * h, 2 * w, C), dt),
                'conf': self._sbuf('prev', 'conf', (h, w), torch.float32), 'flow': self._sbuf('prev', 'flow', (h, w, 2), torch.float32)}

        def carry_flow(i):
            if (a0 + i) in st['fw']:
                prev['flow'].copy_(self._ring('fw', a0 + i, t, (h, w, 2)))

        def forward_branch(copy_flow=True):
            # ---------------- forward branch (RefVSR.py:241-283) ----------------
            state, flow = None, None
            for i in range(range_start, mid + 1):
                if i > range_start:
                    flow = self._ring('fw', a0 + i - 1, t, (h, w, 2))
                    state = self._forward_step(a0 + i, t, h, w, state, flow, True, i)
                elif not is_first_frame:
                    flow = prev['flow']
                    state = self._forward_step(a0 + i, t, h, w, (prev['feat'], prev['featUP'], prev['conf']), flow, False, i)
                else:
                    state = self._forward_step(a0 + i, t, h, w, None, None, False, i)
                if is_log and i == mid and flow is not None:
                    vis['vis']['FW_LR_prev_warp'] = self._warp_image(lr32(i - 1), flow)
                feat_prop, feat_prop_UP, conf_prop = state
                if (is_train and i == 0) or (not is_train and i == mid):           # RefVSR.py:279-283
                    prev['feat'].copy_(feat_prop)
                    prev['featUP'].copy_(feat_prop_UP)
                    prev['conf'].copy_(conf_prop)
                    if copy_flow:
                        carry_flow(i)
            return feat_prop_UP, conf_prop

        # A steady window runs ONE forward step from the carried state: nothing it reads is produced by this call (the flow comes from
        # the previous call, the alignment products of the centre frame were computed when that frame entered) -> it overlaps the
        # entering frame's products and the backward branch.  The one exception is the flow carried to the NEXT call (forward_flows[mid],
        # computed by this call's products): it is copied after the join, which also orders it behind the step's own read of prev.
        overlap = (self.overlap_branches and self._device.type == 'cuda' and hasattr(self.ops, 'set_conv_cta_cap') and not is_log
                   and not is_train and not is_first_frame and range_start == mid and ('frame', a0 + mid) not in work
                   and not self.use_chain)                   # (the chain kernel's tile flags are one shared buffer)
        if overlap:
            ops = self.ops
            main = torch.cuda.current_stream()
            if self._side is None:
                self._side = torch.cuda.Stream(device=self._device)
            side = self._side
            side.wait_stream(main)                                   # fork (a graph branch under capture)
            try:
                ops.set_conv_cta_cap(self.overlap_cap)                # (the cap is read when a launch is enqueued)
                with torch.cuda.stream(side):
                    feat_prop_UP, conf_prop = forward_branch(copy_flow=False)
                ops.set_conv_cta_cap(self.overlap_main_cap)
                products()

                def after_step(k):
                    if k + 1 == self.overlap_bw_steps:
                        ops.set_conv_cta_cap(0)                      # the forward step is over by now: full grids again
                if self.overlap_bw_steps <= 0:
                    ops.set_conv_cta_cap(0)
                backward_feat_UP, conf_bw = self._backward_branch(a0, t, h, w, vis, after_step)
            finally:
                ops.set_conv_cta_cap(0)
                main.wait_stream(side)                               # join
            carry_flow(mid)
        else:
            products()
            # ---------------- backward branch (RefVSR.py:211-238) ----------------
            backward_feat_UP, conf_bw = self._backward_branch(a0, t, h, w, vis)
            # (the forward branch writes 'fw.*' buffers only, so these stay intact)
            feat_prop_UP, conf_prop = forward_branch()

        # ---------------- U (RefVSR.py:286-297) ----------------
        out = self._compute_up(backward_feat_UP, feat_prop_UP, conf_bw, conf_prop, lr32(mid), clamp01=not is_train)

        if is_log and _cget(self.config, 'save_sample', False):
            ev = collections.OrderedDict()
            ev['conf_map'] = self._frame_slot((a0 + mid) % self._rm(t), h, w)['conf'].view(1, 1, h, w).clone()
            ev['conf_map_prop_backward'] = conf_bw.view(1, 1, h, w).clone()
            ev['conf_map_prop_forward'] = conf_prop.view(1, 1, h, w).clone()
            ev['conf_map_prop'] = torch.maximum(ev['conf_map_prop_backward'], ev['conf_map_prop_forward'])
            vis['eval_vis'] = ev
        return out, vis

    # ------------------------------------------------------------------------------------------
    # frame-sharded clip (refvsr_b200/dist.py, SURVEY 8e): the same steps, scheduled per ROLE instead of per window.
    # A rank owns output frames [f0, f1).  Stream position a holds clip frame clamp(a - T//2, 0, n-1) (the clamped windows of
    # data_loader/datasets.py:233-234); window k covers positions k .. k+T-1.  Per-frame products live in a ring of
    # (f1 - f0) + T - 1 positions.  Forward-branch steps form a serial chain across ranks (state hand-off); backward
    # branches, products and the upsampling tail are local.
    # ------------------------------------------------------------------------------------------
    def shard_begin(self, frames_lr, frames_ref, g0, own, num_frames):
        """frames_*: clip frames [g0, g0 + m) (own range + input halo), (m, 3, h, w) on the compute device."""
        t = self.config.frame_num
        m, _, h, w = frames_lr.shape
        hr, wr = frames_ref.shape[2], frames_ref.shape[3]
        if self.max_frame_itr_num is None:
            raise ValueError('reset_branch=None: the forward recurrence never restarts; frame sharding needs chain heads only at '
                             'frame 0, i.e. a pure pipeline - run replicas over different clips instead')
        self._device = frames_lr.device
        self._b = 0
        self._bn = 1
        self._ring_mod = (own[1] - own[0]) + t - 1
        self._shard = {'pyr': set(), 'fw': set(), 'bw': set(), 'frame': set(), 'staged': set(), 'geom': (t, h, w, hr, wr),
                       'g0': g0, 'n': num_frames, 'own': tuple(own), 'lr': frames_lr, 'ref': frames_ref, 'fw_out': {}}
        self._state.clear()          # the windowed forward's caches are void once the ring is re-purposed

    def shard_end(self):
        self._ring_mod, self._shard = None, None
        self._state.clear()

    def _shard_products(self, want):
        """make sure the per-position products in `want` = [(kind, a)], kind in frame / fw / bw, exist in the ring"""
        st = self._shard
        t, h, w, hr, wr = st['geom']
        mid, n, g0 = t // 2, st['n'], st['g0']
        ev = _cget(self.config, 'EVAL', None)
        zero_flow = bool(_cget(ev, 'is_gradio', False)) if ev is not None else False
        work = []

        def stage(a):
            if a not in st['staged']:
                c = min(max(a - mid, 0), n - 1) - g0
                if not 0 <= c < st['lr'].shape[0]:
                    raise RuntimeError(f'frame-sharded clip: position {a} needs clip frame {c + g0}, outside the local range '
                                       f'[{g0}, {g0 + st["lr"].shape[0]}) - input halo too small')
                self._ring('lr32', a, t, (3, h, w)).copy_(st['lr'][c])
                self._ring('ref32', a, t, (3, hr, wr)).copy_(st['ref'][c])
                st['staged'].add(a)

        def need_pyr(a):
            stage(a)
            if a not in st['pyr']:
                st['pyr'].add(a)
                work.append(('pyr', a))
        for kind, a in want:
            if a in st[kind]:
                continue
            st[kind].add(a)
            if kind == 'frame':
                stage(a)
                work.append(('frame', a))
            elif zero_flow:
                work.append((kind + '0', a))
            else:
                need_pyr(a)
                need_pyr(a + 1)
                work.append((kind, a))
        n0 = self.ops.launch_count()
        self._run_products(work, t, h, w, hr, wr)
        self.executed_kernels += self.ops.launch_count() - n0

    def shard_state_buffers(self, tag):
        """persistent (feat, featUP, conf) buffers for a propagated forward state (`tag`: 'in' = received, 'out' = to send)"""
        t, h, w, hr, wr = self._shard['geom']
        C, dt = self.mid_channels, self.act_dtype
        return (self._buf(f'sh.{tag}.feat', (h, w, C), dt), self._buf(f'sh.{tag}.featUP', (2 * h, 2 * w, C), dt),
                self._buf(f'sh.{tag}.conf', (h, w), torch.float32))

    def shard_prefetch_forward(self, k0, k1, head):
        """everything the forward steps of output frames [k0, k1) need that does NOT depend on the incoming state"""
        t = self._shard['geom'][0]
        mid, n = t // 2, self._shard['n']
        want = []
        for k in range(k0, k1):
            first = head and k == k0
            for i in range(0 if first else mid, mid + 1):
                want.append(('frame', k + i))
            for j in range(0 if first else mid - 1, mid):
                want.append(('fw', k + j))            # fw(a) = Flow(position a+1, position a); the step at k+i warps with fw(k+i-1)
        self._shard_products(want)

    def shard_forward_piece(self, k0, k1, state_in):
        """Forward-branch steps of output frames [k0, k1) with torch.no_grad().  state_in None: k0 is a chain head
        (k0 % reset_branch == 0: the branch restarts from zeros over the window's first T//2+1 frames, RefVSR.py:168-176);
        else (feat, featUP, conf) after frame k0-1.  Returns the state after frame k1-1 (persistent 'out' buffers)."""
        st = self._shard
        t, h, w, hr, wr = st['geom']
        mid = t // 2
        with torch.no_grad():
            self.shard_prefetch_forward(k0, k1, state_in is None)
            n0 = self.ops.launch_count()
            out_state = self.shard_state_buffers('out')
            state = state_in
            for k in range(k0, k1):
                if k == k0 and state_in is None:
                    state = None
                    for i in range(0, mid + 1):
                        flow = self._ring('fw', k + i - 1, t, (h, w, 2)) if i > 0 else None
                        state = self._forward_step(k + i, t, h, w, state, flow, True, i)
                else:
                    flow = self._ring('fw', k + mid - 1, t, (h, w, 2))       # = forward_flow_prev of the previous call
                    state = self._forward_step(k + mid, t, h, w, state, flow, False, mid)
                for dst, src in zip(out_state, state):                      # RefVSR.py:279-283 (detach().clone())
                    dst.copy_(src)
                state = out_state
                C, dt = self.mid_channels, self.act_dtype
                keep = (self._buf(f'sh.fwUP.{k - st["own"][0]}', (2 * h, 2 * w, C), dt),
                        self._buf(f'sh.fwconf.{k - st["own"][0]}', (h, w), torch.float32))
                keep[0].copy_(out_state[1])
                keep[1].copy_(out_state[2])
                st['fw_out'][k] = keep
            self.executed_kernels += self.ops.launch_count() - n0
        return out_state

    def shard_finish_window(self, k):
        """backward branch (window-local) + upsampling tail of output frame k; its forward step must be done.
        -> (3, scale*h, scale*w) fp32 (a fresh tensor)"""
        st = self._shard
        t, h, w, hr, wr = st['geom']
        mid = t // 2
        with torch.no_grad():
            self._shard_products([('frame', k + i) for i in range(mid, t)] + [('bw', k + j) for j in range(mid, t - 1)])
            n0 = self.ops.launch_count()
            bw_up, conf_bw = self._backward_branch(k, t, h, w)
            fw_up, conf_fw = st['fw_out'][k]
            out = self._compute_up(bw_up, fw_up, conf_bw, conf_fw, self._ring('lr32', k + mid, t, (3, h, w)), clamp01=True)
            self.executed_kernels += self.ops.launch_count() - n0
            return out.clone()

    def _warp_image(self, img, flow):
        """debug visualisation `warp(lrs[:, i±1], flow)` (RefVSR.py:222,263) -> (1,3,h,w)"""
        x = img.permute(1, 2, 0).contiguous()
        o = torch.empty_like(x)
        self.ops.warp(x, flow, o)
        return o.permute(2, 0, 1).unsqueeze(0).contiguous()
