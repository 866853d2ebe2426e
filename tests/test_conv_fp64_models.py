"""Every convolution of every model, precision and conv kernel the engine runs, checked element by element against a
float64 reference at the engine's shapes: the cases test_conv_fp64.ENGINE_CONVS (RefVSR_MFID, 16-bit, tensor cores) leaves out.

MODEL_CONVS lists them: RefVSR_MFID and RefVSR_small_MFID at x4 with Ref 1x and 2x and at x2, RefVSR_MFID_8K and
RefVSR_small_MFID_8K (flag_HD_in) at LR 1080x1920 -> 4320x7680, each at its own 16-bit type (bf16; fp16 for the is_amp
small models) with tensor cores on and off, and at fp32.  An entry is (name, Sig, kernel, precision class, input
geometries): kernel 'tc' is conv_tc.cu, 'simt' conv_simt.cu, as packing.pack_conv_uncached picks it for the layer; class
'16' runs in bf16 and fp16 on one set of operands exact in both, class '32' runs in fp32.

The bound is test_conv_fp64's.  16-bit cases use its operands and its bound unchanged.  fp32 cases (conv_simt.cu's
<float, float, float> kernel) take inputs, weights, bias, gates and residuals that are fp32 values with full 24-bit
mantissas.  Their products are no longer exact in fp32, but the kernel accumulates with fmaf, so every step
acc <- fmaf(x, w, acc) rounds once, by at most u (2u if it truncated) of a partial sum no larger than A = conv(|x|, |w|) + |b|.
With the bias add, the activation's multiply and the gate multiply that is again at most 2 (K + 2) u A max(1, |gate|)
<= C_ACC K u A max(1, |gate|), plus 2u |ref| for the residual add and the clamp.  The last of these operations yields the
fp32 output itself, so nothing rounds after them: the fp32 bound of test_conv_fp64, with no ulp term.

On dense random operands that bound cannot see reduced input precision.  Inputs rounded to tf32 (or bf16, or weights to
fp16) err by about 2^-11 |x w| per product, and with random signs by about 2^-11 A / sqrt(K) in all, below
C_ACC K u A = 3 K 2^-24 A once K is a few hundred (K = 432 for a 48-channel 3x3 conv).  Hence the sparse precision probe:
each output channel has exactly PROBE_NZ = 8 non-zero weights, at random (tap, input channel) pairs.  fmaf(x, 0, acc) = acc
exactly for finite x, so the accumulation rounds at most PROBE_NZ times and the bound holds with K replaced by
K_nz = PROBE_NZ (2 (8 + 2) <= 3 * 8): 24 u A = 2^-19.4 A.  A single product rounded to tf32 already errs by up to 2^-11
of itself, about 2^-14 A for one of 8 products, some 40 times the bound.  The probe runs once per fp32 signature at a
small geometry; the dense operands run at every geometry the engine runs the conv at.

Maps of more than BAND outputs (the HD and 8K maps: a 4320x7680 map of 48 channels is 1.6 G elements, 3.2 GB in 16 bits
and 12.7 GB in float64) are referenced and checked in horizontal bands of conv output rows.  Each band's reference reads its
input rows with the (k - 1) / 2-row halo the kernel reads (zeros beyond the map), so fp64 memory stays at a few GB while
every element, the last rows included, is checked.

Without a GPU: the list against the 24 schedules' launches (no case missing, none stale), the fp32 bound's self-tests
(a fake fp32 kernel passes both operand families; planted precision, phase and tap defects fail) and the tensor-core
launch plans the new cases reach.  With a GPU: every case, the sparse probe per fp32 signature, and n = 2 batches of the
new tensor-core cases up to 1080x1920 against two separate launches, bit for bit.  n = 2 at 4320x7680 (3.2 G elements per
operand) is not run."""
import collections
import ctypes as C
import functools
import zlib

import pytest
import torch
import torch.nn.functional as F

from refvsr_b200 import packing
from refvsr_b200.lib import IMPL_SIMT, IMPL_TC
from test_conv_batch import _desc, _plan, run_batch
from test_conv_fp64 import (C_ACC, DTYPES, ENGINE_CONVS, GUARD, H100_SMEM, H100_SMS, SPY, U, C3, L1, L2, N, R, Sig, _act,
                            _nchw, _nhwc, _recording_ops, check, out_hw, reference)

SPY_HD = sorted(SPY + [(1088, 1920)])       # SPyNet levels of the x4, x2 and flag_HD_in (LR 1080x1920) schedules
PROBE_NZ = 8
PROBE_HW = (68, 120)
BAND = 1 << 25                              # conv outputs per reference band

# (name, signature, kernel, precision class, input geometries) of every conv launch of the 24 schedules (module docstring)
# that ENGINE_CONVS does not list.  Stride-2 convs of 16-bit tensor-core schedules run over the space-to-depth map (s2d);
# with tensor cores off or in fp32 they run as direct stride-2 / 4 / 8 convs on the CUDA cores.
# test_model_convs_are_all_listed and test_model_convs_are_all_launched keep this exact.
MODEL_CONVS = [
    ('align.conv1.0', Sig(((3, 8),), 32, 5, 2, 1, L2, N, False, '', False, 'act', 32), 'tc', '16', [(2160, 3840)]),
    ('align.rb.conv1', Sig(((32, 32),), 32, 3, 1, 1, L2, N, False, '', False, 'act', 32), 'tc', '16', [(2160, 3840)]),
    ('align.rb.conv2', Sig(((32, 32),), 32, 3, 1, 1, N, L2, False, 'act', False, 'act', 32), 'tc', '16', [(2160, 3840)]),
    ('conf_fusion.0', Sig(((2, 8),), 16, 3, 1, 1, L2, N, False, '', False, 'act', 16), 'tc', '16', [(2160, 3840)]),
    ('conf_fusion.1.24', Sig(((16, 16),), 24, 3, 1, 1, L2, N, False, '', False, 'act', 24),
     'tc', '16', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conf_fusion.1.48', Sig(((16, 16),), 48, 3, 1, 1, L2, N, False, '', False, 'act', 48), 'tc', '16', [(2160, 3840)]),
    ('conv.lrelu.24', Sig(((24, 24),), 24, 3, 1, 1, L2, N, False, '', False, 'act', 24),
     'tc', '16', [(135, 240), (270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conv.lrelu.48', Sig(((48, 48),), 48, 3, 1, 1, L2, N, False, '', False, 'act', 48), 'tc', '16', [(2160, 3840)]),
    ('conv.relu.24', Sig(((24, 24),), 24, 3, 1, 1, R, N, False, '', False, 'act', 24),
     'tc', '16', [(270, 480), (540, 960), (1080, 1920)]),
    ('conv.relu.48', Sig(((48, 48),), 48, 3, 1, 1, R, N, False, '', False, 'act', 48), 'tc', '16', [(1080, 1920)]),
    ('conv.res.24', Sig(((24, 24),), 24, 3, 1, 1, N, N, False, 'act', False, 'act', 24),
     'tc', '16', [(135, 240), (270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conv.res.48', Sig(((48, 48),), 48, 3, 1, 1, N, N, False, 'act', False, 'act', 48), 'tc', '16', [(2160, 3840)]),
    ('conv_hr.24', Sig(((24, 24),), 24, 3, 1, 1, L1, N, False, '', False, 'act', 24), 'tc', '16', [(1080, 1920), (4320, 7680)]),
    ('conv_hr.48', Sig(((48, 48),), 48, 3, 1, 1, L1, N, False, '', False, 'act', 48), 'tc', '16', [(4320, 7680)]),
    ('conv_last.c24', Sig(((24, 24),), 3, 3, 1, 1, N, N, False, '', False, 'f32', 4), 'tc', '16', [(1080, 1920), (4320, 7680)]),
    ('conv_last.c48', Sig(((48, 48),), 3, 3, 1, 1, N, N, False, '', False, 'f32', 4), 'tc', '16', [(4320, 7680)]),
    ('feat_fusion.0.24', Sig(((24, 24), (24, 24)), 24, 3, 1, 1, L2, N, False, '', False, 'act', 24),
     'tc', '16', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('feat_fusion.0.48', Sig(((48, 48), (48, 48)), 48, 3, 1, 1, L2, N, False, '', False, 'act', 48),
     'tc', '16', [(2160, 3840)]),
    ('feat_fusion.1.24', Sig(((24, 24),), 24, 3, 1, 1, L2, N, True, 'act', False, 'act', 24),
     'tc', '16', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('feat_fusion.1.48', Sig(((48, 48),), 48, 3, 1, 1, L2, N, True, 'act', False, 'act', 48), 'tc', '16', [(2160, 3840)]),
    ('fusion_UP.24', Sig(((24, 24), (24, 24)), 24, 1, 0, 1, N, N, False, '', False, 'act', 24),
     'tc', '16', [(540, 960), (1080, 1920), (2160, 3840)]),
    ('fusion_UP.48', Sig(((48, 48), (48, 48)), 48, 1, 0, 1, N, N, False, '', False, 'act', 48), 'tc', '16', [(2160, 3840)]),
    ('main.0.24', Sig(((3, 8), (24, 24)), 24, 3, 1, 1, L1, N, False, '', False, 'act', 24),
     'tc', '16', [(270, 480), (540, 960), (1080, 1920)]),
    ('main.0.48', Sig(((3, 8), (48, 48)), 48, 3, 1, 1, L1, N, False, '', False, 'act', 48), 'tc', '16', [(1080, 1920)]),
    ('ref_encoder1.0.24', Sig(((3, 8),), 24, 3, 1, 1, L2, N, False, '', False, 'act', 24),
     'tc', '16', [(270, 480), (540, 960), (1080, 1920)]),
    ('ref_encoder1.0.48', Sig(((3, 8),), 48, 3, 1, 1, L2, N, False, '', False, 'act', 48), 'tc', '16', [(1080, 1920)]),
    ('ref_encoder2.0.s2d.24', Sig(((96, 96),), 24, 3, 1, 1, L2, N, False, '', False, 'act', 24),
     'tc', '16', [(135, 240), (270, 480), (540, 960)]),
    ('ref_encoder2.0.s2d.48', Sig(((192, 192),), 48, 3, 1, 1, L2, N, False, '', False, 'act', 48), 'tc', '16', [(540, 960)]),
    ('spynet.0', Sig(((8, 8),), 32, 7, 3, 1, R, N, False, '', False, 'act', 32), 'tc', '16', [(1088, 1920)]),
    ('spynet.1', Sig(((32, 32),), 64, 7, 3, 1, R, N, False, '', False, 'act', 64), 'tc', '16', [(1088, 1920)]),
    ('spynet.2', Sig(((64, 64),), 32, 7, 3, 1, R, N, False, '', False, 'act', 32), 'tc', '16', [(1088, 1920)]),
    ('spynet.3', Sig(((32, 32),), 16, 7, 3, 1, R, N, False, '', False, 'act', 16), 'tc', '16', [(1088, 1920)]),
    ('spynet.4+flow_up', Sig(((16, 16),), 2, 7, 3, 1, N, N, False, 'f32', False, 'f32', 2), 'tc', '16', [(1088, 1920)]),
    ('upsample1.192', Sig(((48, 48),), 192, 3, 1, 1, N, N, False, '', True, 'act', 48), 'tc', '16', [(1080, 1920)]),
    ('upsample1.96', Sig(((24, 24),), 96, 3, 1, 1, N, N, False, '', True, 'act', 24),
     'tc', '16', [(270, 480), (540, 960), (1080, 1920)]),
    ('upsample2.192', Sig(((48, 48),), 192, 3, 1, 1, L1, N, False, '', True, 'act', 48), 'tc', '16', [(2160, 3840)]),
    ('upsample2.96', Sig(((24, 24),), 96, 3, 1, 1, L1, N, False, '', True, 'act', 24), 'tc', '16', [(540, 960), (2160, 3840)]),
    ('align.conv1.0', Sig(((3, 8),), 32, 5, 2, 1, L2, N, False, '', False, 'act', 32),
     'simt', '16', [(540, 960), (1080, 1920), (2160, 3840)]),
    ('align.p_conv.0.stride2', Sig(((32, 32), (32, 32)), 32, 5, 2, 2, L2, N, False, '', False, 'act', 32),
     'simt', '16', [(540, 960)]),
    ('align.p_conv.0.stride8', Sig(((32, 32), (32, 32)), 32, 5, 2, 8, L2, N, False, '', False, 'act', 32),
     'simt', '16', [(2160, 3840)]),
    ('align.p_conv.4', Sig(((32, 32),), 3, 1, 0, 1, N, C3, False, '', False, 'f32', 3), 'simt', '16', [(270, 480)]),
    ('align.rb.conv1', Sig(((32, 32),), 32, 3, 1, 1, L2, N, False, '', False, 'act', 32),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('align.rb.conv2', Sig(((32, 32),), 32, 3, 1, 1, N, L2, False, 'act', False, 'act', 32),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conf_fusion.0', Sig(((2, 8),), 16, 3, 1, 1, L2, N, False, '', False, 'act', 16),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conf_fusion.1.24', Sig(((16, 16),), 24, 3, 1, 1, L2, N, False, '', False, 'act', 24),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conf_fusion.1.48', Sig(((16, 16),), 48, 3, 1, 1, L2, N, False, '', False, 'act', 48),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conv.lrelu.24', Sig(((24, 24),), 24, 3, 1, 1, L2, N, False, '', False, 'act', 24),
     'simt', '16', [(135, 240), (270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conv.lrelu.48', Sig(((48, 48),), 48, 3, 1, 1, L2, N, False, '', False, 'act', 48),
     'simt', '16', [(135, 240), (270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conv.relu.24', Sig(((24, 24),), 24, 3, 1, 1, R, N, False, '', False, 'act', 24),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920)]),
    ('conv.relu.48', Sig(((48, 48),), 48, 3, 1, 1, R, N, False, '', False, 'act', 48),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920)]),
    ('conv.res.24', Sig(((24, 24),), 24, 3, 1, 1, N, N, False, 'act', False, 'act', 24),
     'simt', '16', [(135, 240), (270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conv.res.48', Sig(((48, 48),), 48, 3, 1, 1, N, N, False, 'act', False, 'act', 48),
     'simt', '16', [(135, 240), (270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conv_hr.24', Sig(((24, 24),), 24, 3, 1, 1, L1, N, False, '', False, 'act', 24),
     'simt', '16', [(1080, 1920), (4320, 7680)]),
    ('conv_hr.48', Sig(((48, 48),), 48, 3, 1, 1, L1, N, False, '', False, 'act', 48),
     'simt', '16', [(1080, 1920), (4320, 7680)]),
    ('conv_last.c24', Sig(((24, 24),), 3, 3, 1, 1, N, N, False, '', False, 'f32', 4),
     'simt', '16', [(1080, 1920), (4320, 7680)]),
    ('conv_last.c48', Sig(((48, 48),), 3, 3, 1, 1, N, N, False, '', False, 'f32', 4),
     'simt', '16', [(1080, 1920), (4320, 7680)]),
    ('feat_fusion.0.24', Sig(((24, 24), (24, 24)), 24, 3, 1, 1, L2, N, False, '', False, 'act', 24),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('feat_fusion.0.48', Sig(((48, 48), (48, 48)), 48, 3, 1, 1, L2, N, False, '', False, 'act', 48),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('feat_fusion.1.24', Sig(((24, 24),), 24, 3, 1, 1, L2, N, True, 'act', False, 'act', 24),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('feat_fusion.1.48', Sig(((48, 48),), 48, 3, 1, 1, L2, N, True, 'act', False, 'act', 48),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('feature_extract.0', Sig(((3, 8),), 64, 3, 1, 1, R, N, False, '', False, 'act', 64),
     'simt', '16', [(135, 240), (270, 480), (540, 960)]),
    ('feature_extract.2', Sig(((64, 64),), 64, 3, 1, 1, R, N, False, '', False, 'act', 64),
     'simt', '16', [(135, 240), (270, 480), (540, 960)]),
    ('feature_extract.5', Sig(((64, 64),), 128, 3, 1, 1, R, N, False, '', False, 'act', 128),
     'simt', '16', [(135, 240), (270, 480)]),
    ('fusion_UP.24', Sig(((24, 24), (24, 24)), 24, 1, 0, 1, N, N, False, '', False, 'act', 24),
     'simt', '16', [(540, 960), (1080, 1920), (2160, 3840)]),
    ('fusion_UP.48', Sig(((48, 48), (48, 48)), 48, 1, 0, 1, N, N, False, '', False, 'act', 48),
     'simt', '16', [(540, 960), (1080, 1920), (2160, 3840)]),
    ('main.0.24', Sig(((3, 8), (24, 24)), 24, 3, 1, 1, L1, N, False, '', False, 'act', 24),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920)]),
    ('main.0.48', Sig(((3, 8), (48, 48)), 48, 3, 1, 1, L1, N, False, '', False, 'act', 48),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920)]),
    ('map128', Sig(((128, 128),), 16, 1, 0, 1, L2, N, False, '', False, 'act', 16), 'simt', '16', [(135, 240), (270, 480)]),
    ('map64', Sig(((64, 64),), 16, 1, 0, 1, L2, N, False, '', False, 'act', 16), 'simt', '16', [(135, 240), (270, 480)]),
    ('ref_encoder1.0.24', Sig(((3, 8),), 24, 3, 1, 1, L2, N, False, '', False, 'act', 24),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920)]),
    ('ref_encoder1.0.48', Sig(((3, 8),), 48, 3, 1, 1, L2, N, False, '', False, 'act', 48),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920)]),
    ('ref_encoder2.0.24', Sig(((24, 24),), 24, 3, 1, 2, L2, N, False, '', False, 'act', 24),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920)]),
    ('ref_encoder2.0.48', Sig(((48, 48),), 48, 3, 1, 2, L2, N, False, '', False, 'act', 48),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920)]),
    ('spynet.0', Sig(((8, 8),), 32, 7, 3, 1, R, N, False, '', False, 'act', 32), 'simt', '16', SPY_HD),
    ('spynet.1', Sig(((32, 32),), 64, 7, 3, 1, R, N, False, '', False, 'act', 64), 'simt', '16', SPY_HD),
    ('spynet.2', Sig(((64, 64),), 32, 7, 3, 1, R, N, False, '', False, 'act', 32), 'simt', '16', SPY_HD),
    ('spynet.3', Sig(((32, 32),), 16, 7, 3, 1, R, N, False, '', False, 'act', 16), 'simt', '16', SPY_HD),
    ('spynet.4+flow_up', Sig(((16, 16),), 2, 7, 3, 1, N, N, False, 'f32', False, 'f32', 2), 'simt', '16', SPY_HD),
    ('upsample1.192', Sig(((48, 48),), 192, 3, 1, 1, N, N, False, '', True, 'act', 48),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920)]),
    ('upsample1.96', Sig(((24, 24),), 96, 3, 1, 1, N, N, False, '', True, 'act', 24),
     'simt', '16', [(270, 480), (540, 960), (1080, 1920)]),
    ('upsample2.192', Sig(((48, 48),), 192, 3, 1, 1, L1, N, False, '', True, 'act', 48),
     'simt', '16', [(540, 960), (2160, 3840)]),
    ('upsample2.96', Sig(((24, 24),), 96, 3, 1, 1, L1, N, False, '', True, 'act', 24),
     'simt', '16', [(540, 960), (2160, 3840)]),
    ('align.conv1.0', Sig(((3, 8),), 32, 5, 2, 1, L2, N, False, '', False, 'f32', 32),
     'simt', '32', [(540, 960), (1080, 1920), (2160, 3840)]),
    ('align.p_conv.0.stride2', Sig(((32, 32), (32, 32)), 32, 5, 2, 2, L2, N, False, '', False, 'f32', 32),
     'simt', '32', [(540, 960)]),
    ('align.p_conv.0.stride4', Sig(((32, 32), (32, 32)), 32, 5, 2, 4, L2, N, False, '', False, 'f32', 32),
     'simt', '32', [(1080, 1920)]),
    ('align.p_conv.0.stride8', Sig(((32, 32), (32, 32)), 32, 5, 2, 8, L2, N, False, '', False, 'f32', 32),
     'simt', '32', [(2160, 3840)]),
    ('align.p_conv.4', Sig(((32, 32),), 3, 1, 0, 1, N, C3, False, '', False, 'f32', 3), 'simt', '32', [(270, 480)]),
    ('align.rb.conv1', Sig(((32, 32),), 32, 3, 1, 1, L2, N, False, '', False, 'f32', 32),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('align.rb.conv2', Sig(((32, 32),), 32, 3, 1, 1, N, L2, False, 'f32', False, 'f32', 32),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conf_fusion.0', Sig(((2, 8),), 16, 3, 1, 1, L2, N, False, '', False, 'f32', 16),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conf_fusion.1.24', Sig(((16, 16),), 24, 3, 1, 1, L2, N, False, '', False, 'f32', 24),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conf_fusion.1.48', Sig(((16, 16),), 48, 3, 1, 1, L2, N, False, '', False, 'f32', 48),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conv.lrelu.24', Sig(((24, 24),), 24, 3, 1, 1, L2, N, False, '', False, 'f32', 24),
     'simt', '32', [(135, 240), (270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conv.lrelu.48', Sig(((48, 48),), 48, 3, 1, 1, L2, N, False, '', False, 'f32', 48),
     'simt', '32', [(135, 240), (270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conv.relu.24', Sig(((24, 24),), 24, 3, 1, 1, R, N, False, '', False, 'f32', 24),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920)]),
    ('conv.relu.48', Sig(((48, 48),), 48, 3, 1, 1, R, N, False, '', False, 'f32', 48),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920)]),
    ('conv.res.24', Sig(((24, 24),), 24, 3, 1, 1, N, N, False, 'f32', False, 'f32', 24),
     'simt', '32', [(135, 240), (270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conv.res.48', Sig(((48, 48),), 48, 3, 1, 1, N, N, False, 'f32', False, 'f32', 48),
     'simt', '32', [(135, 240), (270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('conv_hr.24', Sig(((24, 24),), 24, 3, 1, 1, L1, N, False, '', False, 'f32', 24),
     'simt', '32', [(1080, 1920), (4320, 7680)]),
    ('conv_hr.48', Sig(((48, 48),), 48, 3, 1, 1, L1, N, False, '', False, 'f32', 48),
     'simt', '32', [(1080, 1920), (4320, 7680)]),
    ('conv_last.c24', Sig(((24, 24),), 3, 3, 1, 1, N, N, False, '', False, 'f32', 4),
     'simt', '32', [(1080, 1920), (4320, 7680)]),
    ('conv_last.c48', Sig(((48, 48),), 3, 3, 1, 1, N, N, False, '', False, 'f32', 4),
     'simt', '32', [(1080, 1920), (4320, 7680)]),
    ('feat_fusion.0.24', Sig(((24, 24), (24, 24)), 24, 3, 1, 1, L2, N, False, '', False, 'f32', 24),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('feat_fusion.0.48', Sig(((48, 48), (48, 48)), 48, 3, 1, 1, L2, N, False, '', False, 'f32', 48),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('feat_fusion.1.24', Sig(((24, 24),), 24, 3, 1, 1, L2, N, True, 'f32', False, 'f32', 24),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('feat_fusion.1.48', Sig(((48, 48),), 48, 3, 1, 1, L2, N, True, 'f32', False, 'f32', 48),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920), (2160, 3840)]),
    ('feature_extract.0', Sig(((3, 8),), 64, 3, 1, 1, R, N, False, '', False, 'f32', 64),
     'simt', '32', [(135, 240), (270, 480), (540, 960)]),
    ('feature_extract.2', Sig(((64, 64),), 64, 3, 1, 1, R, N, False, '', False, 'f32', 64),
     'simt', '32', [(135, 240), (270, 480), (540, 960)]),
    ('feature_extract.5', Sig(((64, 64),), 128, 3, 1, 1, R, N, False, '', False, 'f32', 128),
     'simt', '32', [(135, 240), (270, 480)]),
    ('fusion_UP.24', Sig(((24, 24), (24, 24)), 24, 1, 0, 1, N, N, False, '', False, 'f32', 24),
     'simt', '32', [(540, 960), (1080, 1920), (2160, 3840)]),
    ('fusion_UP.48', Sig(((48, 48), (48, 48)), 48, 1, 0, 1, N, N, False, '', False, 'f32', 48),
     'simt', '32', [(540, 960), (1080, 1920), (2160, 3840)]),
    ('main.0.24', Sig(((3, 8), (24, 24)), 24, 3, 1, 1, L1, N, False, '', False, 'f32', 24),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920)]),
    ('main.0.48', Sig(((3, 8), (48, 48)), 48, 3, 1, 1, L1, N, False, '', False, 'f32', 48),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920)]),
    ('map128', Sig(((128, 128),), 16, 1, 0, 1, L2, N, False, '', False, 'f32', 16), 'simt', '32', [(135, 240), (270, 480)]),
    ('map64', Sig(((64, 64),), 16, 1, 0, 1, L2, N, False, '', False, 'f32', 16), 'simt', '32', [(135, 240), (270, 480)]),
    ('ref_encoder1.0.24', Sig(((3, 8),), 24, 3, 1, 1, L2, N, False, '', False, 'f32', 24),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920)]),
    ('ref_encoder1.0.48', Sig(((3, 8),), 48, 3, 1, 1, L2, N, False, '', False, 'f32', 48),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920)]),
    ('ref_encoder2.0.24', Sig(((24, 24),), 24, 3, 1, 2, L2, N, False, '', False, 'f32', 24),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920)]),
    ('ref_encoder2.0.48', Sig(((48, 48),), 48, 3, 1, 2, L2, N, False, '', False, 'f32', 48),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920)]),
    ('spynet.0', Sig(((8, 8),), 32, 7, 3, 1, R, N, False, '', False, 'f32', 32), 'simt', '32', SPY_HD),
    ('spynet.1', Sig(((32, 32),), 64, 7, 3, 1, R, N, False, '', False, 'f32', 64), 'simt', '32', SPY_HD),
    ('spynet.2', Sig(((64, 64),), 32, 7, 3, 1, R, N, False, '', False, 'f32', 32), 'simt', '32', SPY_HD),
    ('spynet.3', Sig(((32, 32),), 16, 7, 3, 1, R, N, False, '', False, 'f32', 16), 'simt', '32', SPY_HD),
    ('spynet.4+flow_up', Sig(((16, 16),), 2, 7, 3, 1, N, N, False, 'f32', False, 'f32', 2), 'simt', '32', SPY_HD),
    ('upsample1.192', Sig(((48, 48),), 192, 3, 1, 1, N, N, False, '', True, 'f32', 48),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920)]),
    ('upsample1.96', Sig(((24, 24),), 96, 3, 1, 1, N, N, False, '', True, 'f32', 24),
     'simt', '32', [(270, 480), (540, 960), (1080, 1920)]),
    ('upsample2.192', Sig(((48, 48),), 192, 3, 1, 1, L1, N, False, '', True, 'f32', 48),
     'simt', '32', [(540, 960), (2160, 3840)]),
    ('upsample2.96', Sig(((24, 24),), 96, 3, 1, 1, L1, N, False, '', True, 'f32', 24),
     'simt', '32', [(540, 960), (2160, 3840)]),
]


def _kernel_of_engine_conv(sig):
    return 'tc' if sig.stride == 1 else 'simt'


def _cases(entries, kernel_of=None):
    """{(Sig, kernel, class, geometry)} of list entries (ENGINE_CONVS: the 16-bit engine's kernel for its stride)"""
    if kernel_of:
        return {(s, kernel_of(s), '16', g) for _, s, gs in entries for g in gs}
    return {(s, k, p, g) for _, s, k, p, gs in entries for g in gs}


# ------------------------------------------------------------------------------------------------------------------
# CPU: the list above is what the 24 schedules launch
# ------------------------------------------------------------------------------------------------------------------
_X2_MODEL = dict(scale=2, matching_ksize=4)
SCHEDULES = ([(cfg, p16, 270, 480, ov) for cfg, p16 in (('config_RefVSR_MFID', 'bf16'), ('config_RefVSR_small_MFID', 'fp16'))
              for ov in (dict(), dict(ref_scale=2), dict(_X2_MODEL, h=540, w=960))]
             + [(cfg, p16, 1080, 1920, {}) for cfg, p16 in (('config_RefVSR_MFID_8K', 'bf16'),
                                                             ('config_RefVSR_small_MFID_8K', 'fp16'))])


@functools.lru_cache(maxsize=None)
def _clip(frames, h, w, ref_scale):
    from refvsr_b200.synth import make_clip
    return make_clip(frames, h, w, ref_scale, seed=5)


def _record(cfg_name, prec, tc, h, w, ref_scale=1, **over):
    """(Sig, kernel, class, geometry) of every conv of one full-size schedule (two windows), shapes only: the weights keep
    their default initialisation, which the recorded shapes do not depend on"""
    from refvsr_b200 import SRNet, get_config
    from refvsr_b200.synth import sliding_windows
    cfg = get_config(cfg_name, device='cpu', b200_precision=prec, b200_tensor_cores=tc, **over)
    net = SRNet(cfg).eval()
    ops = _recording_ops(False, kernels=True)
    net.Network.set_ops(ops)
    lrs, refs = _clip(cfg.frame_num, h, w, ref_scale)
    with torch.no_grad():
        for n, (k, wl, wr, first) in enumerate(sliding_windows(lrs, refs, cfg.frame_num)):
            net(wl, wr, first)
            if n == 1:
                break
    return set(ops.seen)


@functools.lru_cache(maxsize=None)
def _launched():
    """{schedule: cases} of the 24 schedules"""
    out = {}
    for cfg, p16, h, w, ov in SCHEDULES:
        ov = dict(ov)
        h, w = ov.pop('h', h), ov.pop('w', w)
        for prec, tc in ((p16, True), (p16, False), ('fp32', True)):
            out[(cfg, prec, tc, h, w, tuple(sorted(ov.items())))] = _record(cfg, prec, tc, h, w, **ov)
    return out


def test_model_convs_are_all_listed():
    """every (signature, kernel, precision class, geometry) the 24 schedules launch is in MODEL_CONVS or ENGINE_CONVS, and
    no case is in both"""
    seen = set().union(*_launched().values())
    model, engine = _cases(MODEL_CONVS), _cases(ENGINE_CONVS, _kernel_of_engine_conv)
    assert not model & engine, f'cases in both lists: {sorted(model & engine)}'
    missing = seen - model - engine
    assert not missing, f'conv launches neither list holds: {sorted(missing)}'
    names = collections.Counter((n, k, p) for n, _, k, p, _ in MODEL_CONVS)
    assert max(names.values()) == 1, 'MODEL_CONVS names must be unique per kernel and class'
    per = collections.Counter((k, p) for _, k, p, _ in model)
    print('[conv_fp64_models] new cases per (kernel, class):', dict(per), 'of', len(seen), 'launched')


def test_model_convs_are_all_launched():
    """every MODEL_CONVS case (and every ENGINE_CONVS case, as the 16-bit tensor-core engine runs it) is launched by one
    of the 24 schedules: no stale entries"""
    seen = set().union(*_launched().values())
    stale = _cases(MODEL_CONVS) - seen
    assert not stale, f'MODEL_CONVS cases no schedule launches: {sorted(stale)}'
    stale = _cases(ENGINE_CONVS, _kernel_of_engine_conv) - seen
    assert not stale, f'ENGINE_CONVS cases no schedule launches: {sorted(stale)}'


# ------------------------------------------------------------------------------------------------------------------
# operands, banded reference, fake kernel
# ------------------------------------------------------------------------------------------------------------------
def _ints(shape, lo, hi, g, device, dtype):
    """uniform integers in [lo, hi) as `dtype`, drawn in slabs of rows so that no int64 tensor of the whole map exists"""
    t = torch.empty(shape, dtype=dtype, device=device)
    step = max(1, (1 << 24) // max(1, t[0].numel())) if t.dim() > 1 else t.shape[0]
    for r in range(0, shape[0], step):
        t[r:r + step] = torch.randint(lo, hi, t[r:r + step].shape, generator=g, device=device, dtype=torch.int32).to(dtype)
    return t


def model_operands(sig, H, W, prec, device, seed, family='dense'):
    """class '16': test_conv_fp64.make_operands' values (inputs k / 128, weights k 2^-e with |k| < 256, gates k / 128 in
    [0, 2), residuals k / 64; exact in bf16 and fp16), held as fp16 ('f32' residuals: fp32 normals).  Class '32': fp32
    values with full mantissas - inputs and residuals N(0, 1), weights N(0, 1 / K), bias N(0, 0.01), gates U[0, 2).
    family 'probe' (fp32): PROBE_NZ non-zero weights per output channel.  Source padding channels are zero, as the engine
    keeps them."""
    g = torch.Generator(device=device).manual_seed(seed)
    cin = sum(r for r, _ in sig.srcs)
    K = sig.k * sig.k * cin
    ho, wo = (H + 2 * sig.pad - sig.k) // sig.stride + 1, (W + 2 * sig.pad - sig.k) // sig.stride + 1
    if prec == '16':
        e = max(0, round(float(torch.tensor(73.0 * K ** 0.5).log2())))
        ops = {'w': _ints((sig.cout, cin, sig.k, sig.k), -255, 256, g, device, torch.float32) * 2.0 ** -e}
        act = torch.float16
    else:
        ops = {'w': torch.randn((sig.cout, cin, sig.k, sig.k), generator=g, device=device) / K ** 0.5}
        act = torch.float32
    if family == 'probe':
        w = torch.zeros(sig.cout, K, device=device)
        for n in range(sig.cout):
            pick = torch.randperm(K, generator=g, device=device)[:PROBE_NZ]
            w[n, pick] = torch.randn(PROBE_NZ, generator=g, device=device)
        ops['w'] = w.view(sig.cout, sig.k, sig.k, cin).permute(0, 3, 1, 2).contiguous()
    ops['b'] = torch.randn(sig.cout, generator=g, device=device) * 0.1
    ops['xs'] = []
    for r, a in sig.srcs:
        x = (_ints((H, W, a), -255, 256, g, device, act) / 128 if prec == '16'
             else torch.randn((H, W, a), generator=g, device=device))
        x[..., r:] = 0
        ops['xs'].append(x)
    if sig.gate:
        ops['gate'] = (_ints((ho, wo, sig.cout), 0, 256, g, device, act) / 128 if prec == '16'
                       else torch.rand((ho, wo, sig.cout), generator=g, device=device) * 2)
    if sig.res:
        ops['res'] = (_ints((ho, wo, sig.cout), -255, 256, g, device, act) / 64 if prec == '16' and sig.res == 'act'
                      else torch.randn((ho, wo, sig.cout), generator=g, device=device))
    return ops


def reference_rows(sig, ops, o0, o1, k_acc=None):
    """test_conv_fp64.reference of conv output rows o0 .. o1 - 1: the input rows they read, zero-padded where they leave
    the map, as a pad-0 conv (ref, base); pixel-shuffled output rows 2 o0 .. 2 o1 - 1"""
    s, p, k = sig.stride, sig.pad, sig.k
    lo, hi = o0 * s - p, (o1 - 1) * s - p + k
    H = ops['xs'][0].shape[0]
    band = dict(ops, xs=[F.pad(t[max(lo, 0):min(hi, H)], (0, 0, p, p, max(0, -lo), max(0, hi - H))) for t in ops['xs']])
    for key in ('gate', 'res'):
        if key in ops:
            band[key] = ops[key][o0:o1]
    return reference(sig._replace(pad=0), band, k_acc)


def _round_tf32(t):
    """fp32 -> tf32 (10 explicit mantissa bits), round to nearest"""
    i = t.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def _fake_fp32_kernel(sig, ops, mutation=None):
    """what conv_simt.cu's fp32 kernel computes, on the CPU (fp32 conv, fp32 epilogue); `mutation` plants one defect: 'tf32'
    / 'bf16' rounds the inputs, 'fp16w' the weights, 'phase' reads a strided conv one input pixel up and left (its padding
    off by one), 'tap' drops tap (0, 2) of output channel 5"""
    w = ops['w'].clone()
    if mutation == 'fp16w':
        w = w.half().float()
    if mutation == 'tap':
        w[5, :, 0, 2] = 0
    x = torch.cat([t[..., :r] for t, (r, _) in zip(ops['xs'], sig.srcs)], 2)
    if mutation == 'tf32':
        x = _round_tf32(x)
    if mutation == 'bf16':
        x = x.bfloat16().float()
    x, p = _nchw(x), sig.pad
    if mutation == 'phase':
        x, p = F.pad(x, (p + 1, p - 1, p + 1, p - 1)), 0
    y = _act(F.conv2d(x, w, ops['b'], stride=sig.stride, padding=p), sig.act_pre)
    if sig.gate:
        y = y * _nchw(ops['gate'])
    if sig.res:
        y = y + _nchw(ops['res'])
    y = _act(y, sig.act_post)
    if sig.ps:
        y = F.pixel_shuffle(y, 2)
    return _nhwc(y)


def _entry(name, kernel, prec):
    return next(e for e in MODEL_CONVS if e[0] == name and e[2] == kernel and e[3] == prec)


_FP32_SELF = ['feat_fusion.1.24', 'upsample1.96', 'align.p_conv.0.stride2', 'ref_encoder2.0.48', 'spynet.4+flow_up',
              'conv_last.c24', 'align.p_conv.4', 'main.0.48', 'align.rb.conv2']


@pytest.mark.parametrize('family', ['dense', 'probe'])
@pytest.mark.parametrize('name', _FP32_SELF)
def test_fp32_bound_passes_a_correct_kernel(name, family):
    _, sig, _, _, _ = _entry(name, 'simt', '32')
    ops = model_operands(sig, 20, 28, '32', 'cpu', zlib.crc32(f'{name}/{family}'.encode()), family)
    if family == 'probe':
        assert int((ops['w'] != 0).flatten(1).sum(1).max()) == PROBE_NZ
    ref, base = reference(sig, ops, PROBE_NZ if family == 'probe' else None)
    y = _fake_fp32_kernel(sig, ops)
    assert tuple(y.shape[:2]) == out_hw(sig, 20, 28)
    check(y, ref, base, torch.float32, f'fake fp32 kernel {name} {family}')


@pytest.mark.parametrize('name,family,mutation', [
    ('feat_fusion.1.48', 'probe', 'tf32'), ('conv.res.48', 'probe', 'tf32'), ('upsample1.96', 'probe', 'tf32'),
    ('feat_fusion.1.48', 'probe', 'bf16'), ('align.p_conv.0.stride8', 'probe', 'bf16'),
    ('feat_fusion.1.48', 'probe', 'fp16w'), ('spynet.1', 'probe', 'fp16w'),
    ('align.p_conv.0.stride2', 'dense', 'phase'), ('ref_encoder2.0.24', 'dense', 'phase'),
    ('feat_fusion.1.48', 'dense', 'tap'), ('conv_hr.24', 'dense', 'tap')])
def test_fp32_bound_fails_a_planted_defect(name, family, mutation):
    _, sig, _, _, _ = _entry(name, 'simt', '32')
    ops = model_operands(sig, 40, 56, '32', 'cpu', 11, family)
    ref, base = reference(sig, ops, PROBE_NZ if family == 'probe' else None)
    y = _fake_fp32_kernel(sig, ops, mutation)
    with pytest.raises(pytest.fail.Exception, match='outside the bound') as info:
        check(y, ref, base, torch.float32, f'fake fp32 kernel {name} {family} with {mutation}')
    print(info.value)


@pytest.mark.parametrize('name,kernel,prec', [('upsample1.96', 'tc', '16'), ('align.p_conv.0.stride8', 'simt', '32'),
                                              ('ref_encoder2.0.24', 'simt', '16'), ('conv_last.c24', 'tc', '16')])
def test_banded_reference_is_the_whole_reference(name, kernel, prec):
    """reference_rows over bands of 1, 5 and the rest of the rows, concatenated, is reference() of the whole map"""
    _, sig, _, _, _ = _entry(name, kernel, prec)
    ops = model_operands(sig, 77, 29, prec, 'cpu', 5)
    ref, base = reference(sig, ops)
    ho = (77 + 2 * sig.pad - sig.k) // sig.stride + 1
    parts = [reference_rows(sig, ops, a, b) for a, b in ((0, 1), (1, 6), (6, ho))]
    torch.testing.assert_close(torch.cat([r for r, _ in parts]), ref, rtol=1e-15, atol=1e-15)
    torch.testing.assert_close(torch.cat([b for _, b in parts]), base, rtol=1e-15, atol=1e-15)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the tensor-core launch plans the new cases reach
# ------------------------------------------------------------------------------------------------------------------
_TC_NEW = [(n, s, g) for n, s, k, p, gs in MODEL_CONVS if k == 'tc' for g in gs]


def _variant(sig, plan):
    """conv_tc.cu's kernel for a plan: the compile-time 3x3 loop (p.fixed: layout 1, NB 16 / 48 / 96 and 3 K-steps in every
    64-channel chunk) or the runtime loop"""
    mode, nb = plan[0], plan[6]
    fixed = (mode == 1 and sig.k == 3 and nb in (16, 48, 96)
             and all((min(a - 64 * j, 64) + 15) // 16 == 3 for _, a in sig.srcs for j in range((a + 63) // 64)))
    return 'compile-time 3x3' if fixed else 'runtime loop'


def test_new_tc_cases_reach_their_plans():
    """rv_conv2d_tc_plan / _epi_depth / _out_store / _consumers of every new tensor-core case on an H100 (232448 B opt-in
    shared memory, 132 SMs), printed; the 24-channel cases reach the NB 32 runtime-loop kernel and the NB 96 runtime-loop
    kernel with a 24-channel input, which ENGINE_CONVS does not"""
    from refvsr_b200.lib import load_library
    lib = load_library()
    reached = set()
    for name, sig, (H, W) in _TC_NEW:
        for dt in (torch.bfloat16, torch.float16):
            d = _desc(sig, H, W, dt, 1 << 20)
            plan, depth, store = _plan(lib, d)
            cons = (C.c_int32 * 4)()
            assert lib.rv_conv2d_tc_consumers(C.byref(d), H100_SMEM, H100_SMS, cons) == 0, lib.rv_last_error()
            var = _variant(sig, plan)
            reached.add((plan[0], plan[6], var, sig.srcs[0][1] if len(sig.srcs) == 1 else None))
            print(f'[conv_fp64_models] {name} {H}x{W} {str(dt)[6:]}: mode {plan[0]} NB {plan[6]} {var}, slots {plan[1]}, '
                  f'resident {plan[2]}, S {plan[3]}, consumers {list(cons)[0]}, epi depth {depth}, out store {store}, '
                  f'smem {plan[7]}')
    assert (1, 32, 'runtime loop', 24) in reached, sorted(reached)
    assert (1, 96, 'runtime loop', 24) in reached, sorted(reached)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def run_model_case(cuda_ops, name, sig, kernel, prec, H, W, family='dense'):
    """the conv `sig` on an H x W input through CudaOps.conv2d, packed as the engine packs it for `kernel`, in bf16 and
    fp16 (class '16') or fp32, against the float64 reference in bands of at most BAND conv outputs.  The output sits in a
    NaN-filled buffer with GUARD NaNs on either side; the guards and output channels at or beyond cout must stay NaN.
    Returns the largest |y - ref| / bound per type."""
    dev = 'cuda'
    ops = model_operands(sig, H, W, prec, dev, zlib.crc32(f'{name}/{kernel}{prec}/{H}x{W}/{family}'.encode()), family)
    ho, wo = (H + 2 * sig.pad - sig.k) // sig.stride + 1, (W + 2 * sig.pad - sig.k) // sig.stride + 1
    Ho, Wo = out_hw(sig, H, W)
    ce = sig.cout // 4 if sig.ps else sig.cout
    n = Ho * Wo * sig.out_cs
    outs, tile, nb = {}, (1, 64 if sig.cout > 16 else 128), None
    for dt, dtn in (DTYPES if prec == '16' else ((torch.float32, 'fp32'),)):
        layer = packing.pack_conv_uncached(name, ops['w'], ops['b'], list(sig.srcs), sig.stride, sig.pad, dt, dev,
                                           kernel == 'tc', ps_rows=sig.ps)
        assert layer.impl == (IMPL_TC if kernel == 'tc' else IMPL_SIMT), (name, kernel, layer.impl)
        if kernel == 'tc':
            tile, nb = ((16, 8) if layer.layout in (1, 3) else (8, 16)), layer.nb
        xs = [x.to(dt) for x in ops['xs']]
        gate = ops['gate'].to(dt) if sig.gate else None
        res = ops['res'].to(torch.float32 if sig.res == 'f32' else dt) if sig.res else None
        odt = torch.float32 if sig.out == 'f32' else dt
        buf = torch.full((n + 2 * GUARD,), float('nan'), dtype=odt, device=dev)
        out = buf[GUARD:GUARD + n].view(Ho, Wo, sig.out_cs)
        cuda_ops.conv2d(layer, xs[0], xs[1] if len(xs) > 1 else None, out, gate=gate, res=res, act_pre=sig.act_pre,
                        act_post=sig.act_post, pixel_shuffle=sig.ps)
        torch.cuda.synchronize()
        del xs, gate, res, layer
        what = f'{name} {kernel}{prec} {H}x{W} {dtn} {family}'
        assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + n:]).all(), (what, 'wrote outside its output')
        assert torch.isnan(out[..., ce:]).all(), (what, 'wrote output-buffer channels at or beyond cout')
        outs[dtn] = (out, odt)
    worst = dict.fromkeys(outs, 0.0)
    rows = max(1, BAND // (wo * sig.cout))
    k_acc = PROBE_NZ if family == 'probe' else None
    for o0 in range(0, ho, rows):
        o1 = min(ho, o0 + rows)
        ref, base = reference_rows(sig, ops, o0, o1, k_acc)
        r0, r1 = (2 * o0, 2 * o1) if sig.ps else (o0, o1)
        for dtn, (out, odt) in outs.items():
            band = f' rows {r0}..{r1 - 1} of {Ho}' if rows < ho else ''
            worst[dtn] = max(worst[dtn], check(out[r0:r1, :, :ce], ref, base, odt,
                                               f'{name} {kernel}{prec} {H}x{W} {dtn} {family}{band}', tile, nb, sig.ps))
        del ref, base
    del outs, ops
    torch.cuda.empty_cache()
    print(f'[conv_fp64_models] worst {kernel}{prec} {name} {H}x{W} {family}: ' +
          ', '.join(f'{k} {v:.4f}' for k, v in worst.items()))
    return worst


_GPU_CASES = [(n, s, k, p, g) for n, s, k, p, gs in MODEL_CONVS for g in gs]


@pytest.mark.gpu
@pytest.mark.parametrize('case', _GPU_CASES, ids=[f'{n}-{k}{p}-{g[0]}x{g[1]}' for n, _, k, p, g in _GPU_CASES])
def test_model_conv(cuda_ops, case):
    name, sig, kernel, prec, (H, W) = case
    run_model_case(cuda_ops, name, sig, kernel, prec, H, W)


_PROBES = sorted({(s, n) for n, s, k, p, _ in MODEL_CONVS if p == '32'}, key=lambda e: e[1])


@pytest.mark.gpu
@pytest.mark.parametrize('case', _PROBES, ids=[n for _, n in _PROBES])
def test_fp32_precision_probe(cuda_ops, case):
    sig, name = case
    run_model_case(cuda_ops, name, sig, 'simt', '32', *PROBE_HW, family='probe')


_BATCH = [(n, s, g) for n, s, g in _TC_NEW if g[0] * g[1] <= 1080 * 1920]


@pytest.mark.gpu
@pytest.mark.parametrize('case', _BATCH, ids=[f'{n}-{g[0]}x{g[1]}' for n, _, g in _BATCH])
def test_batched_new_tc_conv_equals_separate_launches(cuda_ops, case):
    name, sig, (H, W) = case
    run_batch(cuda_ops, name, sig, H, W, 2)
