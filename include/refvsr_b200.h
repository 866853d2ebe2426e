/*
 * refvsr_b200 — C ABI of the H100 (sm_90a) kernels behind RefVSR's per-frame forward hot path.
 *
 * The reference (codeslake/RefVSR) is pure Python: it has no FFI of its own.  Its boundary for this
 * path is the nn.Module contract `SRNet.forward(x, ref, is_first_frame, is_log, is_train)`
 * (models/SRNet.py:57-61) and, below it, a sequence of ATen calls.  This header declares one entry
 * point per *fused group* of those ATen calls; each comment cites the reference lines the entry
 * point replaces.  The Python host (refvsr_b200/lib.py) binds them with ctypes; INTEGRATION.md shows
 * the stub a reference maintainer would add.
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless stated otherwise; `stream` is a cudaStream_t passed as
 *     void* (NULL = legacy default stream); every call is asynchronous on that stream;
 *   - activations are NHWC ("pixel rows"): element (y, x, c) at  (y*W + x)*C + c;
 *   - dtype codes: RV_F32 = 0, RV_F16 = 1, RV_BF16 = 2;
 *   - return value: 0 on success, otherwise a negative RV_E_* code; rv_last_error() returns a
 *     human-readable message for the calling thread (the Python binding raises RuntimeError /
 *     ValueError from it, matching the reference's "Python exceptions only" error convention,
 *     mmedit/models/common/flow_warp.py:27-29, models/archs/SPyNet.py:32-34).
 */
#ifndef REFVSR_B200_H_
#define REFVSR_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RV_F32 0
#define RV_F16 1
#define RV_BF16 2

#define RV_OK 0
#define RV_E_INVALID (-1) /* bad argument (shape / dtype / alignment)            */
#define RV_E_CUDA (-2)    /* CUDA runtime / driver error, see rv_last_error()   */
#define RV_E_UNSUPPORTED (-3)

/* 8-bit frame formats of rv_frames_from_u8 and rv_reconstruct_u8{,_batched}.  An (H, W) frame is one contiguous block:
 *   RGB, BGR    (H, W, 3) HWC bytes, R, G, B or B, G, R per pixel: 3 * H * W bytes
 *   I420        the (H, W) Y plane, then U (H/2, W/2), then V (H/2, W/2): 3 * H * W / 2 bytes (ffmpeg's yuv420p)
 *   NV12        the (H, W) Y plane, then (H/2, W) rows of interleaved U, V pairs: 3 * H * W / 2 bytes
 * The 4:2:0 formats are exactly OpenCV's cvtColor conversions (BT.601 limited range, 20-bit fixed point; csrc/frame_u8.cuh):
 * in, the frame stands for the RGB bytes COLOR_YUV2RGB_I420 / _NV12 gives (nearest chroma); out, it is COLOR_RGB2YUV_I420 of
 * the RGB bytes (chroma from each 2 x 2 block's top-left pixel), interleaved for NV12.  H and W must be even. */
#define RV_FRAME_RGB 0
#define RV_FRAME_BGR 1
#define RV_FRAME_I420 2
#define RV_FRAME_NV12 3

/* activation codes used by rv_conv2d epilogues */
#define RV_ACT_NONE 0
#define RV_ACT_RELU 1     /* SPyNet ConvModule, ResidualBlockNoBN (sr_backbone_utils.py:85-97)      */
#define RV_ACT_LRELU01 2  /* LeakyReLU(0.1): RefVSR.py:94,115-116,343                               */
#define RV_ACT_LRELU02 3  /* LeakyReLU(0.2): BasicBlock / ResBlock (RefVSR_/common.py:25-39,96-109) */
#define RV_ACT_CLAMP3 4   /* clamp(-3, 3): affine map of AlignedConv2d (alignment.py:56)            */

#define RV_CONV_IMPL_SIMT 0 /* fp32-accumulate CUDA-core implicit GEMM (any geometry, any dtype)    */
#define RV_CONV_IMPL_TC 1   /* wgmma implicit GEMM fed by TMA (f16/bf16, stride 1)                 */

const char* rv_last_error(void);
int rv_version(void);
/* number of kernels launched by this library since load (bench.py's `gpu_launches`) */
uint64_t rv_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * rv_conv2d — fused convolution.  Replaces every nn.Conv2d on the path *together with* the
 * elementwise ops around it:
 *   torch.cat of the two inputs          (RefVSR.py:128,138,139,110,225,266; SPyNet.py:96-102)
 *   bias + ReLU / LeakyReLU              (SPyNet.py:152-191; RefVSR_/common.py:25-39,96-109)
 *   alpha-gating and residual adds       (RefVSR.py:131,143,112; common.py:38,80-81;
 *                                          sr_backbone_utils.py:96-97; SPyNet.py:95)
 *   F.pixel_shuffle                      (mmedit/models/common/upsample.py:48-51)
 *
 *   acc[n]  = bias[n] + sum_{ky,kx,c} W[n][c][ky][kx] * in[(y*stride+ky-pad, x*stride+kx-pad), c]
 *             with in = concat(src0, src1) along channels, zero padding outside the image
 *   v       = act_pre(acc);  if (gate) v *= gate[pix][n];  if (res) v += res[pix][n];
 *   v       = act_post(v);
 *   out     = pixel_shuffle ? out[(2y+a, 2x+b)][n/4] (n = 4c+2a+b) : out[pix][n]
 * `out` must not overlap src0, src1, gate or res: a tile reads the src0 / src1 halo that neighbouring tiles store,
 * and the TC path fetches the gate / residual of later tiles while earlier tiles store.
 * ------------------------------------------------------------------------------------------------ */
typedef struct rv_conv_desc {
  const void* src0;   /* [H][W][c0]                                                       */
  const void* src1;   /* [H][W][c1] or NULL                                               */
  int32_t c0, c1;     /* allocated channels of src0/src1 (TC: multiples of 8)             */
  int32_t in_dtype;   /* dtype of src0/src1/gate                                          */
  int32_t H, W;       /* input spatial size                                               */
  const void* wpack;  /* packed weights, layout produced by refvsr_b200/packing.py        */
  const float* bias;  /* [cout] fp32                                                      */
  int32_t cout;       /* real output channels                                             */
  int32_t kh, kw, stride, pad;
  int32_t act_pre, act_post;
  const void* gate;   /* [Ho][Wo][gate_cs] (in_dtype) or NULL                             */
  int32_t gate_cs;
  const void* res;    /* [Ho][Wo][res_cs] (res_dtype) or NULL                             */
  int32_t res_cs, res_dtype;
  void* out;          /* [Ho][Wo][out_cs]   (or [2Ho][2Wo][out_cs] when pixel_shuffle)    */
  int32_t out_cs, out_dtype;
  int32_t pixel_shuffle; /* 0 | 1 (factor 2)                                              */
  int32_t impl;          /* RV_CONV_IMPL_*                                                */
  int32_t nb;            /* TC: output channels per CTA column block (packing.py decides) */
  int32_t k_real;        /* SIMT: rows of wpack = kh*kw*(c0+c1)                           */
  int32_t layout;        /* TC: 0 = [nblk][kx][chunk][ky][NB][64] (one TMA box per kx),    */
                         /*     1 = [nblk][chunk][ky][kx][NB][64] (one box per tile+chunk; */
                         /*         3x3 convs with the all-16-bit epilogue run kx-folded,  */
                         /*         N = 3*NB per MMA),                                     */
                         /*     2 = 32B-swizzled 16-channel quads,                         */
                         /*     3 = weight image of 1, kx-folding disabled (test / A-B)    */
  int32_t ps_order;      /* TC pixel shuffle: 0 = columns n = 4c+2a+b; 1 = HR-row order   */
                         /*   (packing.ps_rows_order: cout = 2*nb, block a = HR sub-row a, */
                         /*   both sub-pixels x all cout/4 channels; weights and bias      */
                         /*   permuted to match).  Other descs must leave it 0.            */
  /* Batch: n images through one launch, each computed exactly as alone (a tile never reads across an image's border).   */
  /* n = 0 or 1: one image, the strides are ignored.  n > 1: image i of an operand starts i * bs_* ELEMENTS after its     */
  /* pointer; every stride of a non-null operand must be > 0 (TC: src0 / src1 strides multiples of 8).  The tensor-core   */
  /* path runs all n x tiles in one persistent launch with the weights loaded once per CTA; the SIMT path issues one       */
  /* launch per image.                                                                                                    */
  int32_t n;
  int64_t bs_src0, bs_src1, bs_gate, bs_res, bs_out;
} rv_conv_desc;

int rv_conv2d(const rv_conv_desc* d, void* stream);
/* Upper bound of the persistent grid of the following rv_conv2d (tensor-core) launches made by this process; 0 restores one CTA
 * per SM.  Returns the previous value.  The engine's own scheduling knob, no counterpart in the reference: the forward-branch
 * step of a window (RefVSR.py:248-277) is independent of its backward branch (RefVSR.py:211-238), so network.py enqueues the two on
 * different streams with half the SMs each - two capped launches overlap each other's prologue / first-box latency / last-tile tail,
 * which a single dependent chain of launches exposes once per layer. */
int rv_set_conv_cta_cap(int cap);
/* Upper bound of the shared memory per CTA that the following rv_conv2d (tensor-core) launches plan with; 0 restores the device's
 * opt-in limit.  Returns the previous value.  A smaller bound takes the plan branches of a device with less shared memory (fewer
 * ring slots, no TMA output buffer), so that each can be run and compared on one device. */
int rv_set_conv_smem_cap(int bytes);
/* 2: the following rv_conv2d (tensor-core) launches run every conv on the two-consumer kernel; 0 (or any other value)
 * restores the plan's choice, which runs the single-source 48 -> 48 3x3 convs (plain or with a residual) on three consumer
 * warpgroups when their buffers fit.  Returns the previous value.  Lets the two kernels be compared on one device. */
int rv_set_conv_consumers(int n);

/* Host-only: the launch plan rv_conv2d's tensor-core path would use on a device with `max_smem_optin` bytes of opt-in shared memory
 * per block and `num_sms` SMs, with the two-consumer kernel (rv_set_conv_consumers(2); rv_conv2d_tc_consumers gives the plan
 * of a three-consumer launch) -> out8 = {mode, smem slots per consumer, weights resident, stages per tile, consumer
 * warpgroups, accumulator sets, nb, dynamic smem bytes}.  No CUDA call is made (pointers in `d` are only tested for null / alignment).  Lets the
 * ring invariants (every issuing warp owns its slots and accumulators) be checked without a GPU. */
int rv_conv2d_tc_plan(const rv_conv_desc* d, int max_smem_optin, int num_sms, int32_t* out8);
/* Host-only, same plan: *depth = gate / residual tiles a consumer's shared-memory buffers hold ahead of its epilogue (1 or 2), 0 when
 * the epilogue loads those operands itself (no gate / residual, NB > 48, or operands TMA cannot address). */
int rv_conv2d_tc_epi_depth(const rv_conv_desc* d, int max_smem_optin, int num_sms, int32_t* depth);
/* Host-only, same plan: how the output is stored.  *kind = 0 per-thread stores from registers, 1 TMA boxes of NHWC tiles staged
 * in shared memory, 2 TMA boxes of pixel-shuffled HR rows staged in shared memory (ps_order 1), 3 pixel-shuffled HR rows as
 * 16-byte stores from registers (ps_order 1, when the staging buffers do not fit). */
int rv_conv2d_tc_out_store(const rv_conv_desc* d, int max_smem_optin, int num_sms, int32_t* kind);
/* Host-only: the plan a launch takes under the current rv_set_conv_consumers setting -> out4 = {consumer warpgroups (2 or 3),
 * smem slots per consumer, gate / residual TMA buffers per consumer (0: none), dynamic smem bytes}. */
int rv_conv2d_tc_consumers(const rv_conv_desc* d, int max_smem_optin, int num_sms, int32_t* out4);

/* ------------------------------------------------------------------------------------------------
 * rv_resblock - residual block  out = act_post( x + conv2( act_mid( conv1(x) ) ) ), 3x3 / stride 1 / pad 1,
 * C -> C -> C channels (C <= 64), f16/bf16 NHWC.  One launch instead of two rv_conv2d calls for
 * ResidualBlockNoBN (mmedit/models/common/sr_backbone_utils.py:85-97, act_mid = ReLU) and ResBlock
 * (models/archs/RefVSR_/common.py:33-39, act_mid = LeakyReLU(0.2); act_post = LeakyReLU(0.2) inside
 * AlignedConv2d, alignment.py:19-21).  w1 / w2: packing.pack_tc(..., layout=1) images ([9 taps][nb][64]).
 * ------------------------------------------------------------------------------------------------ */
typedef struct rv_resblock_desc {
  const void* src;   /* [H][W][c] */
  int32_t c;         /* allocated channels of src (multiple of 8, <= 64) */
  int32_t dtype;     /* RV_F16 | RV_BF16 (input, intermediate and output) */
  int32_t H, W;
  const void* w1;
  const float* b1;   /* [cout] */
  const void* w2;
  const float* b2;
  int32_t cout, nb, act_mid, act_post;
  void* out;         /* [H][W][out_cs] */
  int32_t out_cs;
} rv_resblock_desc;

int rv_resblock(const rv_resblock_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * rv_conv_chain - a CHAIN of 3x3 C->C convolutions (+ bias, activation, residual, activation) over a small set of NHWC
 * f16/bf16 buffers of identical geometry, executed by ONE persistent wgmma launch with per-tile dependencies between
 * layers (refvsr_b200/csrc/conv_chain.cu).  Covers
 *   make_layer(ResidualBlockNoBN, num_blocks)  (mmedit/models/common/sr_backbone_utils.py:26-39,85-97; RefVSR.py:346-349)
 *   ResList: N x ResBlock + conv_tail + skip    (RefVSR_/common.py:25-39,64-82; RefVSR.py:48-60,233-234)
 * Layer l computes  buf[dst] = act_post( act_pre( conv3x3(buf[src]) + bias ) + buf[res] )   (res < 0: no residual), zero
 * padding 1.  dst must differ from src.  wpack = the layout-1 tensor-core weight image of rv_conv2d ([9 taps][nb][64]
 * 16-bit, SWIZZLE_128B byte image), bias = nb floats (zero beyond cout).  All buffers: (H, W, C), C % 8 == 0, C <= 48.
 * `flags` is device scratch of >= ceil(H/16) * ceil(W/8) int32, zeroed by the call on `stream`; flags[t] counts the layers tile t
 * has completed (all = nlayers at the end).
 * Results are bit-identical to the same layers issued one by one through rv_conv2d.
 * ------------------------------------------------------------------------------------------------ */
#define RV_CHAIN_MAX_LAYERS 64
#define RV_CHAIN_MAX_BUFFERS 6
typedef struct {
  const void* wpack;
  const float* bias;
  int32_t src, res, dst;
  int32_t act_pre, act_post; /* RV_ACT_NONE / RELU / LRELU01 / LRELU02 */
} rv_chain_layer;
typedef struct {
  void* buf[RV_CHAIN_MAX_BUFFERS];
  int32_t nbuf;
  int32_t H, W, C, dtype; /* C = allocated channels (row pitch) of every buffer */
  int32_t nb;             /* rows of the weight image (16 / 32 / 48), >= C */
  const rv_chain_layer* layers; /* HOST array */
  int32_t nlayers;
  int32_t* flags;
  int32_t max_ctas; /* 0: one persistent CTA per SM.  > 0: cap (leave SMs free for kernels of OTHER streams that must stay
                       co-resident, e.g. NCCL point-to-point kernels: the chain's CTAs wait on each other's flags and all
                       of them have to be resident) */
} rv_conv_chain_desc;
int rv_conv_chain(const rv_conv_chain_desc* d, void* stream);

/* space-to-depth by 2: out[(Y,X)][(ry*2+rx)*C + c] = src[(2Y+ry, 2X+rx)][c].  Turns the two stride-2
 * convolutions of the path (ref_encoder2.0.0, RefVSR.py:45; aa2.align.p_conv.0, alignment.py:21) into
 * stride-1 3x3 convolutions over 4C channels (weights re-indexed by packing.s2d_weights), so they run on
 * the tensor-core kernel.  H, W even; C*elemsize a multiple of 16. */
int rv_space_to_depth2(const void* src, int H, int W, int C, int dtype, void* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Image / map preparation
 * ------------------------------------------------------------------------------------------------ */
/* NCHW fp32 image (3,H,W) -> NHWC `out` with `out_c` channels (>=3, rest zero).
 * mat12 != NULL: out_c = mat[c][0..2]·rgb + mat[c][3]  (MeanShift 1x1 conv, common.py:84-94,
 *                attention.py:62-63).  pool2: 2x2 mean after the affine map (attention.py:51,75). */
int rv_prep_image(const float* src_nchw, int H, int W, const float* mat12_host, int pool2,
                  void* out, int out_c, int out_dtype, void* stream);

/* SPyNet input resize: bilinear (align_corners=False) to (Ho,Wo) then (x-mean)/std
 * (SPyNet.py:117-126, 62-63). src NCHW fp32 (3,H,W) -> out HWC fp32 (Ho,Wo,3) */
int rv_spynet_resize_norm(const float* src_nchw, int H, int W, float* out, int Ho, int Wo,
                          void* stream);
/* 2x2 mean pool, HWC fp32 with C channels (SPyNet.py:66-78) */
int rv_avgpool2(const float* src, int H, int W, int C, float* out, void* stream);
/* 2x2 / stride 2 max pool of an NHWC map (torchvision vgg19.features[4] inside FeatureMatching with vgg_range = 7,
 * i.e. the flag_HD_in "8K" configs, attention.py:31-40).  src (H,W,C) -> out (H/2,W/2,C), same dtype. */
int rv_maxpool2(const void* src, int H, int W, int C, int dtype, void* out, void* stream);
/* Resize of `n` planar fp32 maps (n,H,W) -> (n,Ho,Wo) with the source coordinate scale `inv_scale` = 1 / scale_factor:
 *   mode 0: bicubic, A = -0.75, align_corners=False, clamped taps (F.interpolate(mode='bicubic')): the x4 upsample
 *           of the relevance map (attention.py:96-98) and lr_down = bicubic x0.5 of the LR frame (RefVSR.py:125);
 *   mode 1: nearest, src = floor(dst * inv_scale) (F.interpolate(scale_factor=0.5, mode='nearest'), attention.py:65-67).
 * clamp01: clamp the result to [0,1] (both bicubic call sites do). */
int rv_resize_planes(const float* src, int n, int H, int W, float inv_scale, int Ho, int Wo, int mode, int clamp01,
                     float* out, void* stream);
/* One pyramid level's network input (SPyNet.py:84-102):
 *   flow_up = level0 ? 0 : 2 * bilinear_x2_align_corners(flow_prev)      -> flow_up (H,W,2) fp32
 *   out8    = [ref(3), flow_warp(supp, flow_up, border, align_corners=True)(3), flow_up(2)]
 * flow_prev is (H/2, W/2, 2) fp32 or NULL. */
int rv_spynet_level_input(const float* ref, const float* supp, const float* flow_prev, int H, int W,
                          void* out8, int out_dtype, float* flow_up, void* stream);
/* final flow resize back to (h,w) + per-axis rescale (SPyNet.py:129-137) */
int rv_flow_resize(const float* flow, int H, int W, float* out, int h, int w, void* stream);

/* ------------------------------------------------------------------------------------------------
 * rv_warp — models/utils.py:34-43 (`warp`: grid_sample bilinear / zeros / align_corners=False with
 * the reference's linspace grid) fused with the x2 flow upsample of RefVSR.py:220,254,259.
 *   src (Hi,Wi,C) `dtype`; flow (hf,wf,2) fp32 in LR pixels;
 *   flow_up2 == 0: output grid = flow grid (hf,wf);
 *   flow_up2 == 1: output grid = (2hf,2wf), flow' = 2*bilinear_align_corners_true(flow).
 * ------------------------------------------------------------------------------------------------ */
int rv_warp(const void* src, int Hi, int Wi, int C, int dtype, const float* flow, int hf, int wf,
            int flow_up2, void* out, void* stream);
/* Batched entry points (`*_batched`): the same arguments plus `n`, the number of images, before `stream`.  Every operand
 * holds n images back to back ([n][...] in the layout of the one-image call), and image i is computed exactly as the
 * one-image call on the i-th slices would compute it, in one launch (the image is gridDim.z).  1 <= n <= 65535. */
int rv_warp_batched(const void* src, int Hi, int Wi, int C, int dtype, const float* flow, int hf, int wf,
                    int flow_up2, void* out, int n, void* stream);
/* The three warps of one propagation step fused into ONE launch (RefVSR.py:216-220 backward branch, :256-260 steady forward
 * step): out_feat = warp(feat, flow), out_conf = warp(conf, flow), out_featUP = warp(featUP, interpolate(flow, x2, bilinear,
 * align_corners=True) * 2).  feat (h,w,C), featUP (2h,2w,C) f16/bf16, conf (h,w) fp32, flow (h,w,2) fp32.  The flow is read
 * once; same arithmetic as three rv_warp calls (feat / conf bit-identical, featUP to the last bit of the storage type).  (Not for the first-window quirk RefVSR.py:252-254, whose 2x warp
 * reads the OUTPUT of the LR warp.) */
int rv_warp3(const void* feat, const void* featUP, const float* conf, const float* flow, int h, int w, int C, int dtype,
             void* out_feat, void* out_featUP, float* out_conf, void* stream);
int rv_warp3_batched(const void* feat, const void* featUP, const float* conf, const float* flow, int h, int w, int C, int dtype,
                     void* out_feat, void* out_featUP, float* out_conf, int n, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Matching (models/archs/RefVSR_/attention.py:69-91)
 * ------------------------------------------------------------------------------------------------ */
/* 3x3 reflection-padded patches of a 16-channel feature map, L2-normalised (eps 1e-12), written
 * K-major as fp16 rows for the GEMM:   mode 0: [hi]                 (kpad >= 144)
 *                                      mode 1: [hi | lo | hi]       (A side, kpad >= 432)
 *                                      mode 2: [hi | hi | lo]       (B side)
 * values are pre-scaled by 2^6 so the fp16 `lo` part stays normal; rv_match_argmax undoes it.
 * (RefVSR_/utils.py:10-57 same_padding + Unfold; attention.py:83-85 F.normalize) */
int rv_patch_pack(const void* feat, int H, int W, int C, int dtype, int mode, void* out_f16,
                  int kpad, void* stream);
/* conf[l] = max_r <A[l], B[r]>,  idx[l] = argmax_r (lowest r wins ties)  (attention.py:91).
 * A (P,kpad) fp16, B (R,kpad) fp16, outputs conf (P) fp32, idx (P) int32.
 * impl: 0 = CUDA-core fp32 reference kernel, 1 = wgmma (TMA-fed, register accumulators). */
int rv_match_argmax(const void* A, int P, const void* B, int R, int kpad, float out_scale,
                    float* conf, int32_t* idx, int impl, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Reference alignment (attention.py:131-159, alignment.py:39-100)
 * ------------------------------------------------------------------------------------------------ */
/* AlignedAttention gather: out[(ks*i+a, ks*j+b)] = value[(ks*ry+a, ks*rx+b)],
 * (ry,rx) = divmod(idx[i*wq+j], Wv/ks).  value (Hv,Wv,C); out (ks*hq, ks*wq, C). ks=1 -> aa1. */
int rv_gather_blocks(const void* value, int Hv, int Wv, int C, int dtype, const int32_t* idx, int hq,
                     int wq, int ks, void* out, void* stream);
/* AlignedConv2d sampling (alignment.py:45-100,102-178): x (ks*h, ks*w, C), affine (h,w,3) fp32
 * already = clamp(p_conv(..)+1, -3, 3); reflection pad 1; output (ks*h, ks*w, C). */
int rv_aligned_sample(const void* x, int h, int w, int ks, int C, int dtype, const float* affine,
                      void* out, void* stream);
/* bicubic x2 of an image, A=-0.75, align_corners=False, NO clamp (alignment.py:41):
 * src NCHW fp32 (3,H,W) -> out NHWC (2H,2W,out_c) */
int rv_bicubic_up2_image(const float* src_nchw, int H, int W, void* out, int out_c, int out_dtype,
                         void* stream);

/* ------------------------------------------------------------------------------------------------
 * Confidence maps (RefVSR.py:105-106,110,129,140-142,147)
 * ------------------------------------------------------------------------------------------------ */
/* out[(y,x)] = [A(y,x), B(y,x), 0...] (out_c channels); up2: A,B are first bicubic-x2 upsampled and
 * clamped to [0,1].  a,b planar fp32 (h,w). */
int rv_conf_pair(const float* a, const float* b, int h, int w, int up2, void* out, int out_c,
                 int out_dtype, void* stream);
int rv_conf_pair_batched(const float* a, const float* b, int h, int w, int up2, void* out, int out_c,
                         int out_dtype, int n, void* stream);   /* see rv_warp_batched */
int rv_conf_max(const float* a, const float* b, float* out, int n, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Guard of the sliding-window reuse (no reference counterpart: the reference silently ASSUMES that consecutive calls slide
 * the window by one frame when it reuses forward_*_prev, RefVSR.py:256-260; this implementation also reuses per-frame
 * products, so it checks).  Compares n <= 16 (a[i], b[i], nbytes[i]) DEVICE buffer pairs; the pointer / size arrays
 * themselves are HOST arrays.  *flag (device int32, zeroed by the caller) becomes non-zero iff any pair differs.
 * ------------------------------------------------------------------------------------------------ */
int rv_frames_differ(const void* const* a, const void* const* b, const uint64_t* nbytes, int n, int32_t* flag,
                     void* stream);

/* ------------------------------------------------------------------------------------------------
 * Reconstruction tail (RefVSR.py:118,288,297): out = conv_last_out + clamp(bicubic_x4(lr),0,1),
 * optionally clamped to [0,1]; written NCHW fp32 (3, 4h, 4w).  x (4h,4w,xc) is conv_last's output.
 * ------------------------------------------------------------------------------------------------ */
int rv_reconstruct(const void* x, int xc, int x_dtype, const float* lr_nchw, int h, int w, int scale,
                   int clamp01, float* out_nchw, void* stream);
int rv_reconstruct_batched(const void* x, int xc, int x_dtype, const float* lr_nchw, int h, int w, int scale,
                           int clamp01, float* out_nchw, int n, void* stream);   /* see rv_warp_batched */
/* The same reconstruction with 8-bit output: each value the matching rv_reconstruct{,_batched} call writes becomes the byte
 * cv::Mat::convertTo(CV_8U) makes of fl32(v * 255) (csrc/frame_u8.cuh: round half to even, saturated; NaN -> 0), stored
 * as an (scale*h, scale*w) frame of format fmt (RV_FRAME_*; RGB: R, G, B bytes per pixel, BGR: cv2's order, I420 / NV12: the
 * 4:2:0 frame of those RGB bytes), images packed one after the other for n > 1.  The kernel is chosen as rv_reconstruct
 * chooses its own (x4 / x2 fast paths for fp32 x with xc = 4, the generic kernel otherwise), and computes each value with that
 * kernel's expressions.  16-byte stores of 16-pixel row runs (8-byte stores of I420's 8-sample chroma runs) where out is 16-byte
 * aligned and a row is a multiple of 16 pixels (generic kernel: where an image is a multiple of 16 bytes); byte stores
 * elsewhere, to the same bytes.  RV_E_INVALID for a format code outside RV_FRAME_*. */
int rv_reconstruct_u8(const void* x, int xc, int x_dtype, const float* lr_nchw, int h, int w, int scale, int clamp01, int fmt,
                      uint8_t* out, void* stream);
int rv_reconstruct_u8_batched(const void* x, int xc, int x_dtype, const float* lr_nchw, int h, int w, int scale, int clamp01,
                              int fmt, uint8_t* out, int n, void* stream);

/* ------------------------------------------------------------------------------------------------
 * rv_frames_from_u8 - decoded 8-bit video frames into the engine's fp32 frames (data_loader/utils.py::read_frame's
 * np.array(frame) / 255. cast to float32).
 *   src    HOST array of k device pointers, each a contiguous (h, w) uint8 frame of format fmt (RV_FRAME_*), any alignment
 *   dst    HOST array of k device pointers, each a contiguous fp32 (3, h, w) planar RGB frame
 *   1 <= k <= 16, h, w >= 1, h * w <= 2^28; h and w even for I420 / NV12
 * Byte u of the frame's R, G, B bytes (for 4:2:0, the bytes cv2.cvtColor(COLOR_YUV2RGB_I420 / _NV12) gives) becomes
 * fl32(u / 255) with IEEE division (round to nearest).  One launch.  RGB / BGR: 16-byte loads wherever a frame has 16-byte
 * aligned runs of 16 pixels (every frame but at most 30 pixels of it), 16-byte stores where dst allows.  4:2:0: 16-byte loads of
 * the Y rows and each chroma sample read once per 2 x 2 block where src is 16-byte aligned and w a multiple of 16, byte loads
 * otherwise; 16-byte stores where dst is aligned too.
 * RV_E_INVALID for any argument outside the above.
 * ------------------------------------------------------------------------------------------------ */
int rv_frames_from_u8(const uint8_t* const* src, float* const* dst, int k, int h, int w, int fmt, void* stream);

/* ------------------------------------------------------------------------------------------------
 * rv_region_metrics - the per-frame sums behind the FOV evaluation mode: evaluation/metrics.py:18-31 (psnr, psnr_masked,
 * ssim, ssim_masked) as evaluation/eval_quan_FOV.py:153-213 uses them, where every mask is a union or difference of boxes.
 *   a, b        contiguous fp32 (1, 3, H, W) images (output, ground truth), H, W >= 7
 *   boxes_host  HOST array of nbox x (y0, y1, x0, x1), half-open, inside the frame (empty and overlapping boxes allowed),
 *               1 <= nbox <= 8
 *   sums        device fp64 [2 * nbox]:  sums[k]        = sum over box k and the 3 channels of (a - b)^2 (float32 difference
 *                                                         and square, as numpy's float32 arrays compute them)
 *                                        sums[nbox + k] = sum over box k and the 3 channels of the SSIM map S
 *   S is skimage's structural_similarity map for data_range 1: uniform 7x7 window computed in fp64, sample covariance
 *   (49/48), C1 = 1e-4, C2 = 9e-4, over the FULL frame with scipy `reflect` borders (index -1 -> 0, -2 -> 1, -3 -> 2, likewise
 *   at the far edges), i.e. the map ssim_masked multiplies by its mask.
 *   work        device fp64 scratch of RV_REGION_METRICS_WORK(H, W, nbox) doubles.
 * Two launches, no allocation, no atomics: the second reduces the per-CTA partials in a fixed order, so repeated calls are
 * bit-identical.  RV_E_INVALID for any argument outside the above.
 * ------------------------------------------------------------------------------------------------ */
#define RV_REGION_METRICS_WORK(H, W, nbox) ((((H) + 15) / 16) * (((W) + 31) / 32) * 2 * (nbox))
int rv_region_metrics(const float* a, const float* b, int H, int W, const int32_t* boxes_host, int nbox, double* work,
                      double* sums, void* stream);

/* ------------------------------------------------------------------------------------------------
 * rv_conf_map_images - the per-frame image bytes of the confidence-map evaluation mode (evaluation/eval_quan_conf_map.py:
 * 64-165): the colour-mapped confidence maps, the input and the output, each as the uint8 BGR HWC image cv2.imwrite encodes.
 *   conf, prop, prop_b, prop_f   fp32 (h, w) maps: conf_map, conf_map_prop, conf_map_prop_backward, conf_map_prop_forward
 *   normalize    1: the four maps, each min/max-normalised as torch float32 computes it (y = x - min(x); y / max(y))
 *                0: `conf` alone, coloured as it is (the reference's branch for a vis without conf_map_prop; the other three
 *                   pointers are ignored)
 *   inp, out     contiguous fp32 NCHW (1, 3, ih, iw) and (1, 3, oh, ow) RGB frames
 *   lut_rgb      device uint8 [256][3]: the colormap's entries as the 8-bit values cv2.imwrite writes for them
 *   work         device scratch of RV_CONF_MAP_WORK uint32 words
 *   dst          device uint8 of RV_CONF_MAP_BYTES(h, w, ih, iw, oh, ow, normalize) bytes, packed without gaps: the maps
 *                (h, w, 3) in the order above, then the input (ih, iw, 3), then the output (oh, ow, 3), all BGR
 * A map value y (after normalisation, if any) takes matplotlib's Colormap.__call__ index for a float32 array: t = fl32(y * 256),
 * 255 for t == 256, NaN -> black (the "bad" colour), t < 0 -> 0 (under), t >= 256 -> 255 (over), else trunc(t).  A frame value
 * x becomes cv::Mat::convertTo(CV_8U) of fl32(x * 255): round half to even, saturated to [0, 255]; NaN and values outside
 * int32 become 0, as x86 builds of OpenCV convert them.  A constant map normalises to 0 / 0 = NaN and comes out black.
 * At most two launches: per-CTA min / max partials of each map (normalize only), then the image pass, which folds them first.
 * No atomics, no allocation.
 * RV_E_INVALID for any argument outside the above.
 * ------------------------------------------------------------------------------------------------ */
#define RV_CONF_MAP_WORK 512
#define RV_CONF_MAP_BYTES(h, w, ih, iw, oh, ow, normalize) \
  (3ll * ((normalize) ? 4 : 1) * (h) * (w) + 3ll * (ih) * (iw) + 3ll * (oh) * (ow))
int rv_conf_map_images(const float* conf, const float* prop, const float* prop_b, const float* prop_f, int h, int w,
                       int normalize, const float* inp, int ih, int iw, const float* out, int oh, int ow,
                       const uint8_t* lut_rgb, uint32_t* work, uint8_t* dst, void* stream);

/* ------------------------------------------------------------------------------------------------
 * rv_eval_images - the per-frame image bytes of the default evaluation mode (evaluation/eval_qual_quan.py:103-125): the
 * input, the output and the ground truth, each as the uint8 BGR HWC image cv2.imwrite encodes from cv2.cvtColor(x * 255,
 * cv2.COLOR_RGB2BGR).
 *   frames     HOST array of nframes device pointers, each a contiguous fp32 NCHW (1, 3, H, W) RGB frame, 1 <= nframes <= 3
 *   hw_host    HOST array of nframes x (H, W), each H, W >= 1 with H * W <= 2^28
 *   dst        device uint8 of RV_EVAL_IMAGES_BYTES = sum of 3 * H * W bytes, packed without gaps: the frames' (H, W, 3) BGR
 *              images in the order of `frames`
 * A value x becomes cv::Mat::convertTo(CV_8U) of fl32(x * 255), exactly as rv_conf_map_images converts its frames (the same
 * device function): round half to even, saturated to [0, 255]; NaN and values outside int32 become 0.
 * One launch, no allocation.  16-byte loads and stores for a frame whose pointer and place in dst are 16-byte aligned and whose
 * H * W is a multiple of 4; other frames convert pixel by pixel to the same bytes.
 * RV_E_INVALID for any argument outside the above.
 * ------------------------------------------------------------------------------------------------ */
int rv_eval_images(const float* const* frames, const int* hw_host, int nframes, uint8_t* dst, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* REFVSR_B200_H_ */
