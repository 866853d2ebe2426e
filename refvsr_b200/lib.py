"""ctypes binding of the C-ABI library (include/refvsr_b200.h) and the `CudaOps` operator set.

`CudaOps` is the ONLY implementation of the operator interface that ships in the product: every
method launches hand-written sm_90a kernels from `librefvsr_b200.so` on torch's current CUDA stream.
There is no CPU / eager fallback - constructing `CudaOps` without the built library or without a
CUDA device raises.  torch is used for device memory and streams only.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'librefvsr_b200.so')

RV_F32, RV_F16, RV_BF16 = 0, 1, 2
ACT_NONE, ACT_RELU, ACT_LRELU01, ACT_LRELU02, ACT_CLAMP3 = 0, 1, 2, 3, 4
IMPL_SIMT, IMPL_TC = 0, 1
# 8-bit frame formats (RV_FRAME_*): RGB and BGR are HWC bytes (False / True are accepted for them), I420 and NV12 are YUV 4:2:0
FRAME_RGB, FRAME_BGR, FRAME_I420, FRAME_NV12 = 0, 1, 2, 3

DTYPE_CODE = {torch.float32: RV_F32, torch.float16: RV_F16, torch.bfloat16: RV_BF16}


def frame_shape(h, w, fmt):
    """the uint8 shape of one (h, w) frame of format fmt: (h, w, 3) HWC bytes, or the (3h/2, w) array cv2 uses for 4:2:0"""
    if fmt in (FRAME_I420, FRAME_NV12):
        return (3 * h // 2, w)
    assert fmt in (FRAME_RGB, FRAME_BGR), f'unknown frame format {fmt!r}'
    return (h, w, 3)


class rv_conv_desc(C.Structure):
    _fields_ = [
        ('src0', C.c_void_p), ('src1', C.c_void_p), ('c0', C.c_int32), ('c1', C.c_int32),
        ('in_dtype', C.c_int32), ('H', C.c_int32), ('W', C.c_int32),
        ('wpack', C.c_void_p), ('bias', C.c_void_p), ('cout', C.c_int32),
        ('kh', C.c_int32), ('kw', C.c_int32), ('stride', C.c_int32), ('pad', C.c_int32),
        ('act_pre', C.c_int32), ('act_post', C.c_int32),
        ('gate', C.c_void_p), ('gate_cs', C.c_int32),
        ('res', C.c_void_p), ('res_cs', C.c_int32), ('res_dtype', C.c_int32),
        ('out', C.c_void_p), ('out_cs', C.c_int32), ('out_dtype', C.c_int32),
        ('pixel_shuffle', C.c_int32), ('impl', C.c_int32), ('nb', C.c_int32), ('k_real', C.c_int32),
        ('layout', C.c_int32), ('ps_order', C.c_int32),
        ('n', C.c_int32),
        ('bs_src0', C.c_int64), ('bs_src1', C.c_int64), ('bs_gate', C.c_int64), ('bs_res', C.c_int64), ('bs_out', C.c_int64),
    ]


class rv_resblock_desc(C.Structure):
    _fields_ = [
        ('src', C.c_void_p), ('c', C.c_int32), ('dtype', C.c_int32), ('H', C.c_int32), ('W', C.c_int32),
        ('w1', C.c_void_p), ('b1', C.c_void_p), ('w2', C.c_void_p), ('b2', C.c_void_p),
        ('cout', C.c_int32), ('nb', C.c_int32), ('act_mid', C.c_int32), ('act_post', C.c_int32),
        ('out', C.c_void_p), ('out_cs', C.c_int32),
    ]


class rv_chain_layer(C.Structure):
    _fields_ = [('wpack', C.c_void_p), ('bias', C.c_void_p), ('src', C.c_int32), ('res', C.c_int32), ('dst', C.c_int32),
                ('act_pre', C.c_int32), ('act_post', C.c_int32)]


class rv_conv_chain_desc(C.Structure):
    _fields_ = [('buf', C.c_void_p * 6), ('nbuf', C.c_int32), ('H', C.c_int32), ('W', C.c_int32), ('C', C.c_int32),
                ('dtype', C.c_int32), ('nb', C.c_int32), ('layers', C.POINTER(rv_chain_layer)), ('nlayers', C.c_int32),
                ('flags', C.c_void_p), ('max_ctas', C.c_int32)]


CHAIN_MAX_LAYERS, CHAIN_MAX_BUFFERS = 64, 6

# name -> (restype, argtypes); mirrors include/refvsr_b200.h one to one (tests check the export list)
_P, _I, _F = C.c_void_p, C.c_int, C.c_float
SIGNATURES = {
    'rv_last_error': (C.c_char_p, []),
    'rv_version': (_I, []),
    'rv_launch_count': (C.c_uint64, []),
    'rv_conv2d': (_I, [C.POINTER(rv_conv_desc), _P]),
    'rv_set_conv_cta_cap': (_I, [_I]),
    'rv_conv2d_tc_plan': (_I, [C.POINTER(rv_conv_desc), _I, _I, C.POINTER(C.c_int32)]),
    'rv_conv2d_tc_epi_depth': (_I, [C.POINTER(rv_conv_desc), _I, _I, C.POINTER(C.c_int32)]),
    'rv_conv2d_tc_out_store': (_I, [C.POINTER(rv_conv_desc), _I, _I, C.POINTER(C.c_int32)]),
    'rv_set_conv_smem_cap': (_I, [_I]),
    'rv_set_conv_consumers': (_I, [_I]),
    'rv_conv2d_tc_consumers': (_I, [C.POINTER(rv_conv_desc), _I, _I, C.POINTER(C.c_int32)]),
    'rv_resblock': (_I, [C.POINTER(rv_resblock_desc), _P]),
    'rv_conv_chain': (_I, [C.POINTER(rv_conv_chain_desc), _P]),
    'rv_space_to_depth2': (_I, [_P, _I, _I, _I, _I, _P, _P]),
    'rv_prep_image': (_I, [_P, _I, _I, _P, _I, _P, _I, _I, _P]),
    'rv_spynet_resize_norm': (_I, [_P, _I, _I, _P, _I, _I, _P]),
    'rv_avgpool2': (_I, [_P, _I, _I, _I, _P, _P]),
    'rv_maxpool2': (_I, [_P, _I, _I, _I, _I, _P, _P]),
    'rv_resize_planes': (_I, [_P, _I, _I, _I, _F, _I, _I, _I, _I, _P, _P]),
    'rv_spynet_level_input': (_I, [_P, _P, _P, _I, _I, _P, _I, _P, _P]),
    'rv_flow_resize': (_I, [_P, _I, _I, _P, _I, _I, _P]),
    'rv_warp': (_I, [_P, _I, _I, _I, _I, _P, _I, _I, _I, _P, _P]),
    'rv_warp3': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P]),
    'rv_warp_batched': (_I, [_P, _I, _I, _I, _I, _P, _I, _I, _I, _P, _I, _P]),
    'rv_warp3_batched': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _I, _P]),
    'rv_conf_pair_batched': (_I, [_P, _P, _I, _I, _I, _P, _I, _I, _I, _P]),
    'rv_reconstruct_batched': (_I, [_P, _I, _I, _P, _I, _I, _I, _I, _P, _I, _P]),
    'rv_patch_pack': (_I, [_P, _I, _I, _I, _I, _I, _P, _I, _P]),
    'rv_match_argmax': (_I, [_P, _I, _P, _I, _I, _F, _P, _P, _I, _P]),
    'rv_gather_blocks': (_I, [_P, _I, _I, _I, _I, _P, _I, _I, _I, _P, _P]),
    'rv_aligned_sample': (_I, [_P, _I, _I, _I, _I, _I, _P, _P, _P]),
    'rv_bicubic_up2_image': (_I, [_P, _I, _I, _P, _I, _I, _P]),
    'rv_conf_pair': (_I, [_P, _P, _I, _I, _I, _P, _I, _I, _P]),
    'rv_conf_max': (_I, [_P, _P, _P, _I, _P]),
    'rv_frames_differ': (_I, [_P, _P, _P, _I, _P, _P]),
    'rv_reconstruct': (_I, [_P, _I, _I, _P, _I, _I, _I, _I, _P, _P]),
    'rv_region_metrics': (_I, [_P, _P, _I, _I, C.POINTER(C.c_int32), _I, _P, _P, _P]),
    'rv_conf_map_images': (_I, [_P, _P, _P, _P, _I, _I, _I, _P, _I, _I, _P, _I, _I, _P, _P, _P, _P]),
    'rv_eval_images': (_I, [C.POINTER(C.c_void_p), C.POINTER(C.c_int), _I, _P, _P]),
    'rv_reconstruct_u8': (_I, [_P, _I, _I, _P, _I, _I, _I, _I, _I, _P, _P]),
    'rv_reconstruct_u8_batched': (_I, [_P, _I, _I, _P, _I, _I, _I, _I, _I, _P, _I, _P]),
    'rv_frames_from_u8': (_I, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), _I, _I, _I, _I, _P]),
}

CONF_MAP_WORK = 512                 # RV_CONF_MAP_WORK


def conf_map_bytes(h, w, ih, iw, oh, ow, normalize):
    """RV_CONF_MAP_BYTES: size of rv_conf_map_images' packed output"""
    return 3 * (4 if normalize else 1) * h * w + 3 * ih * iw + 3 * oh * ow

_lib = None


def load_library(path=LIB_PATH):
    """dlopen the kernels library and attach prototypes.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(path):
        raise RuntimeError(
            f'{path} not found: build the CUDA extension first (python -c "import __graft_entry__ as g; '
            'g.build()").  refvsr_b200 has no CPU fallback.')
    lib = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def _check(lib, rc, what):
    if rc != 0:
        msg = lib.rv_last_error().decode('utf-8', 'replace')
        if rc == -1:
            raise ValueError(f'{what}: {msg}')
        raise RuntimeError(f'{what}: {msg} (code {rc})')


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _chk_dev(*ts):
    for t in ts:
        if t is not None:
            assert t.is_cuda and t.is_contiguous(), 'operands must be contiguous CUDA tensors'


class CudaOps:
    """Operator set backed by librefvsr_b200.so.  Shapes: activations (H, W, C); images (3, H, W)
    fp32; flows (H, W, 2) fp32; confidence maps (H, W) fp32; index maps (H*W,) int32."""

    name = 'cuda'
    batched = True      # conv2d and the propagation-step operators also take (n, ...) operands (network.py's batched windows)

    def __init__(self, device='cuda'):
        if not torch.cuda.is_available():
            raise RuntimeError('refvsr_b200 requires a CUDA device (no CPU fallback)')
        self.lib = load_library()
        self.device = torch.device(device)

    # -- helpers ---------------------------------------------------------------------------------
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def launch_count(self):
        return int(self.lib.rv_launch_count())

    def set_conv_cta_cap(self, cap):
        """persistent-grid bound of the following tensor-core conv launches (0 = one CTA per SM); returns the previous value"""
        return int(self.lib.rv_set_conv_cta_cap(int(cap)))

    def set_conv_smem_cap(self, nbytes):
        """shared-memory bound the following tensor-core conv launches plan with (0 = the device's limit); returns the previous value"""
        return int(self.lib.rv_set_conv_smem_cap(int(nbytes)))

    def set_conv_consumers(self, n):
        """2: the following tensor-core conv launches run the two-consumer kernel for every conv; 0: the plan's choice (three
        consumers for the single-source 48 -> 48 3x3 convs when they fit); returns the previous value"""
        return int(self.lib.rv_set_conv_consumers(int(n)))

    # -- convolution ------------------------------------------------------------------------------
    def conv2d(self, layer, src0, src1, out, gate=None, res=None, act_pre=ACT_NONE, act_post=ACT_NONE,
               pixel_shuffle=False):
        """`layer` is a packing.PackedConv.  Output geometry is checked by the caller (engine).  Operands are (H, W, C) maps, or
        (n, H, W, C) for a batch of n images through one launch (every operand then has the batch dimension)."""
        _chk_dev(src0, src1, out, gate, res)
        d = rv_conv_desc()
        if src0.dim() == 4:
            ops = (src0, src1, gate, res, out)
            assert all(t is None or (t.dim() == 4 and t.shape[0] == src0.shape[0]) for t in ops), \
                f'{layer.name}: a batched conv needs (n, H, W, C) operands of one n'
            d.n = src0.shape[0]
            d.bs_src0, d.bs_out = src0.stride(0), out.stride(0)
            d.bs_src1 = src1.stride(0) if src1 is not None else 0
            d.bs_gate = gate.stride(0) if gate is not None else 0
            d.bs_res = res.stride(0) if res is not None else 0
        d.src0 = src0.data_ptr()
        d.src1 = src1.data_ptr() if src1 is not None else None
        d.c0 = src0.shape[-1]
        d.c1 = src1.shape[-1] if src1 is not None else 0
        assert (d.c0, d.c1) == (layer.alloc0, layer.alloc1), \
            f'{layer.name}: source channels {(d.c0, d.c1)} != packed layout {(layer.alloc0, layer.alloc1)}'
        d.in_dtype = DTYPE_CODE[src0.dtype]
        d.H, d.W = src0.shape[-3], src0.shape[-2]
        d.wpack = layer.wpack.data_ptr()
        d.bias = layer.bias.data_ptr()
        d.cout = layer.cout
        d.kh, d.kw, d.stride, d.pad = layer.kh, layer.kw, layer.stride, layer.pad
        d.act_pre, d.act_post = act_pre, act_post
        d.gate = gate.data_ptr() if gate is not None else None
        d.gate_cs = gate.shape[-1] if gate is not None else 0
        d.res = res.data_ptr() if res is not None else None
        d.res_cs = res.shape[-1] if res is not None else 0
        d.res_dtype = DTYPE_CODE[res.dtype] if res is not None else 0
        d.out = out.data_ptr()
        d.out_cs = out.shape[-1]
        d.out_dtype = DTYPE_CODE[out.dtype]
        d.pixel_shuffle = 1 if pixel_shuffle else 0
        d.impl = layer.impl
        d.nb = layer.nb
        d.k_real = layer.k_real
        d.layout = getattr(layer, 'layout', 0)
        d.ps_order = getattr(layer, 'ps_order', 0)
        _check(self.lib, self.lib.rv_conv2d(C.byref(d), self._stream()), f'rv_conv2d[{layer.name}]')

    def resblock(self, rb, src, out, act_mid, act_post=ACT_NONE):
        """`rb` is a packing.PackedResBlock; out = act_post(src + conv2(act_mid(conv1(src))))"""
        _chk_dev(src, out)
        assert src.shape[2] == rb.alloc and src.dtype == out.dtype and src.data_ptr() != out.data_ptr()
        d = rv_resblock_desc()
        d.src, d.c, d.dtype = src.data_ptr(), src.shape[2], DTYPE_CODE[src.dtype]
        d.H, d.W = src.shape[0], src.shape[1]
        d.w1, d.b1, d.w2, d.b2 = rb.w1.data_ptr(), rb.b1.data_ptr(), rb.w2.data_ptr(), rb.b2.data_ptr()
        d.cout, d.nb, d.act_mid, d.act_post = rb.cout, rb.nb, act_mid, act_post
        d.out, d.out_cs = out.data_ptr(), out.shape[2]
        _check(self.lib, self.lib.rv_resblock(C.byref(d), self._stream()), f'rv_resblock[{rb.name}]')

    def conv_chain(self, bufs, layers, flags, max_ctas=0):
        """bufs: list of (H, W, C) tensors of one dtype / geometry; layers: [(packing.PackedChainLayer, src, res, dst, act_pre,
        act_post)] with buffer indices (res = -1: none); flags: int32 scratch with >= ceil(H/16)*ceil(W/8) entries.
        Launches ceil(len(layers) / 64) persistent kernels (rv_conv_chain)."""
        _chk_dev(*bufs)
        H, W, Cc = bufs[0].shape
        assert all(tuple(b.shape) == (H, W, Cc) and b.dtype == bufs[0].dtype for b in bufs) and len(bufs) <= CHAIN_MAX_BUFFERS
        assert flags.dtype == torch.int32 and flags.numel() >= ((H + 15) // 16) * ((W + 7) // 8)
        nb = layers[0][0].nb
        for i in range(0, len(layers), CHAIN_MAX_LAYERS):
            part = layers[i:i + CHAIN_MAX_LAYERS]
            arr = (rv_chain_layer * len(part))()
            for j, (pk, src, res, dst, a0, a1) in enumerate(part):
                assert pk.nb == nb
                arr[j].wpack, arr[j].bias = pk.wpack.data_ptr(), pk.bias.data_ptr()
                arr[j].src, arr[j].res, arr[j].dst, arr[j].act_pre, arr[j].act_post = src, res, dst, a0, a1
            d = rv_conv_chain_desc()
            for b, t in enumerate(bufs):
                d.buf[b] = t.data_ptr()
            d.nbuf, d.H, d.W, d.C, d.dtype, d.nb = len(bufs), H, W, Cc, DTYPE_CODE[bufs[0].dtype], nb
            d.layers, d.nlayers, d.flags, d.max_ctas = arr, len(part), flags.data_ptr(), int(max_ctas)
            _check(self.lib, self.lib.rv_conv_chain(C.byref(d), self._stream()), 'rv_conv_chain')

    def space_to_depth2(self, src, out):
        _chk_dev(src, out)
        if src.dim() == 4:     # (n, H, W, C) with H even: the batch is one map of n*H rows
            src, out = src.view(-1, src.shape[2], src.shape[3]), out.view(-1, out.shape[2], out.shape[3])
        _check(self.lib, self.lib.rv_space_to_depth2(_ptr(src), src.shape[0], src.shape[1], src.shape[2],
                                                     DTYPE_CODE[src.dtype], _ptr(out), self._stream()),
               'rv_space_to_depth2')

    # -- image / pyramid prep ---------------------------------------------------------------------
    def prep_image(self, src, out, mat12=None, pool2=False):
        _chk_dev(src, out)
        H, W = src.shape[1], src.shape[2]
        m = None
        if mat12 is not None:
            m = (C.c_float * 12)(*[float(v) for v in mat12])
        _check(self.lib, self.lib.rv_prep_image(_ptr(src), H, W, m, int(pool2), _ptr(out), out.shape[2],
                                                DTYPE_CODE[out.dtype], self._stream()), 'rv_prep_image')

    def spynet_resize_norm(self, src, out):
        _chk_dev(src, out)
        _check(self.lib, self.lib.rv_spynet_resize_norm(_ptr(src), src.shape[1], src.shape[2], _ptr(out),
                                                        out.shape[0], out.shape[1], self._stream()),
               'rv_spynet_resize_norm')

    def avgpool2(self, src, out):
        _chk_dev(src, out)
        _check(self.lib, self.lib.rv_avgpool2(_ptr(src), src.shape[0], src.shape[1], src.shape[2], _ptr(out),
                                              self._stream()), 'rv_avgpool2')

    def maxpool2(self, src, out):
        """NHWC (H,W,C) -> (H/2,W/2,C) 2x2 max (vgg19.features[4], flag_HD_in matching)"""
        _chk_dev(src, out)
        assert src.dtype == out.dtype and tuple(out.shape) == (src.shape[0] // 2, src.shape[1] // 2, src.shape[2])
        _check(self.lib, self.lib.rv_maxpool2(_ptr(src), src.shape[0], src.shape[1], src.shape[2], DTYPE_CODE[src.dtype],
                                              _ptr(out), self._stream()), 'rv_maxpool2')

    def resize_planes(self, src, out, inv_scale, mode='bicubic', clamp01=False):
        """planar fp32 (n,H,W) -> (n,Ho,Wo): F.interpolate(scale_factor=1/inv_scale, mode=bicubic|nearest) [+ clamp(0,1)]"""
        _chk_dev(src, out)
        assert src.dtype == out.dtype == torch.float32 and src.dim() == 3 and out.dim() == 3 and src.shape[0] == out.shape[0]
        _check(self.lib, self.lib.rv_resize_planes(_ptr(src), src.shape[0], src.shape[1], src.shape[2], float(inv_scale),
                                                   out.shape[1], out.shape[2], 0 if mode == 'bicubic' else 1,
                                                   int(clamp01), _ptr(out), self._stream()), 'rv_resize_planes')

    def spynet_level_input(self, ref, supp, flow_prev, out8, flow_up):
        _chk_dev(ref, supp, flow_prev, out8, flow_up)
        _check(self.lib, self.lib.rv_spynet_level_input(_ptr(ref), _ptr(supp), _ptr(flow_prev), ref.shape[0],
                                                        ref.shape[1], _ptr(out8), DTYPE_CODE[out8.dtype],
                                                        _ptr(flow_up), self._stream()), 'rv_spynet_level_input')

    def flow_resize(self, flow, out):
        _chk_dev(flow, out)
        _check(self.lib, self.lib.rv_flow_resize(_ptr(flow), flow.shape[0], flow.shape[1], _ptr(out),
                                                 out.shape[0], out.shape[1], self._stream()), 'rv_flow_resize')

    # -- warp -------------------------------------------------------------------------------------
    def warp(self, src, flow, out, flow_up2=False):
        _chk_dev(src, flow, out)
        if flow.dim() == 3:                        # one image: a batch of 1
            src, flow, out = src[None], flow[None], out[None]
        n = flow.shape[0]                          # a batch of n images: (n, ...) operands, one launch
        Hi, Wi, Cc = (src.shape[1], src.shape[2], 1) if src.dim() == 3 else src.shape[1:]
        assert src.shape[0] == out.shape[0] == n
        _check(self.lib, self.lib.rv_warp_batched(_ptr(src), Hi, Wi, Cc, DTYPE_CODE[src.dtype], _ptr(flow), flow.shape[1],
                                                  flow.shape[2], int(flow_up2), _ptr(out), n, self._stream()), 'rv_warp')

    def warp3(self, feat, featUP, conf, flow, out_feat, out_featUP, out_conf):
        """the three warps of one propagation step in one launch (16-bit features)"""
        _chk_dev(feat, featUP, conf, flow, out_feat, out_featUP, out_conf)
        n = flow.shape[0] if flow.dim() == 4 else 0   # a batch of n images: (n, ...) operands, one launch
        h, w, Cc = feat.shape[-3:]
        lead = (n,) if n else ()
        assert tuple(featUP.shape) == lead + (2 * h, 2 * w, Cc) and tuple(conf.shape) == lead + (h, w)
        assert tuple(flow.shape) == lead + (h, w, 2) and tuple(feat.shape) == lead + (h, w, Cc)
        assert feat.dtype == featUP.dtype == out_feat.dtype == out_featUP.dtype and conf.dtype == torch.float32
        _check(self.lib, self.lib.rv_warp3_batched(_ptr(feat), _ptr(featUP), _ptr(conf), _ptr(flow), h, w, Cc, DTYPE_CODE[feat.dtype],
                                                   _ptr(out_feat), _ptr(out_featUP), _ptr(out_conf), max(n, 1), self._stream()),
               'rv_warp3')

    # -- matching ---------------------------------------------------------------------------------
    def patch_pack(self, feat, out, mode):
        _chk_dev(feat, out)
        _check(self.lib, self.lib.rv_patch_pack(_ptr(feat), feat.shape[0], feat.shape[1], feat.shape[2],
                                                DTYPE_CODE[feat.dtype], mode, _ptr(out), out.shape[1],
                                                self._stream()), 'rv_patch_pack')

    def match_argmax(self, A, B, conf, idx, impl=1):
        _chk_dev(A, B, conf, idx)
        assert A.dtype == torch.float16 and B.dtype == torch.float16 and idx.dtype == torch.int32
        _check(self.lib, self.lib.rv_match_argmax(_ptr(A), A.shape[0], _ptr(B), B.shape[0], A.shape[1],
                                                  1.0 / 4096.0, _ptr(conf), _ptr(idx), impl, self._stream()),
               'rv_match_argmax')

    # -- reference alignment ----------------------------------------------------------------------
    def gather_blocks(self, value, idx, hq, wq, ks, out):
        _chk_dev(value, idx, out)
        _check(self.lib, self.lib.rv_gather_blocks(_ptr(value), value.shape[0], value.shape[1], value.shape[2],
                                                   DTYPE_CODE[value.dtype], _ptr(idx), hq, wq, ks, _ptr(out),
                                                   self._stream()), 'rv_gather_blocks')

    def aligned_sample(self, x, affine, ks, out):
        _chk_dev(x, affine, out)
        h, w = affine.shape[0], affine.shape[1]
        _check(self.lib, self.lib.rv_aligned_sample(_ptr(x), h, w, ks, x.shape[2], DTYPE_CODE[x.dtype],
                                                    _ptr(affine), _ptr(out), self._stream()), 'rv_aligned_sample')

    def bicubic_up2_image(self, src, out):
        _chk_dev(src, out)
        _check(self.lib, self.lib.rv_bicubic_up2_image(_ptr(src), src.shape[1], src.shape[2], _ptr(out),
                                                       out.shape[2], DTYPE_CODE[out.dtype], self._stream()),
               'rv_bicubic_up2_image')

    # -- confidence maps --------------------------------------------------------------------------
    def conf_pair(self, a, b, out, up2=False):
        _chk_dev(a, b, out)
        if out.dim() == 3:                         # one image: a batch of 1
            a, b, out = a[None], b[None], out[None]
        assert a.shape[0] == b.shape[0] == out.shape[0]   # a batch of n images: (n, ...) operands, one launch
        _check(self.lib, self.lib.rv_conf_pair_batched(_ptr(a), _ptr(b), a.shape[1], a.shape[2], int(up2), _ptr(out),
                                                       out.shape[3], DTYPE_CODE[out.dtype], out.shape[0], self._stream()),
               'rv_conf_pair')

    def conf_max(self, a, b, out):
        _chk_dev(a, b, out)
        _check(self.lib, self.lib.rv_conf_max(_ptr(a), _ptr(b), _ptr(out), a.numel(), self._stream()), 'rv_conf_max')

    def frames_differ(self, pairs, flag):
        """pairs: [(a, b)] contiguous same-size CUDA tensors; flag (1,) int32, zeroed here, set non-zero iff any pair differs"""
        n = len(pairs)
        assert 0 < n <= 16
        for a, b in pairs:
            _chk_dev(a, b)
            assert a.numel() * a.element_size() == b.numel() * b.element_size() and a.dtype == b.dtype
        pa = (C.c_void_p * n)(*[a.data_ptr() for a, _ in pairs])
        pb = (C.c_void_p * n)(*[b.data_ptr() for _, b in pairs])
        nb = (C.c_uint64 * n)(*[a.numel() * a.element_size() for a, _ in pairs])
        flag.zero_()
        _check(self.lib, self.lib.rv_frames_differ(pa, pb, nb, n, _ptr(flag), self._stream()), 'rv_frames_differ')

    # -- tail -------------------------------------------------------------------------------------
    def reconstruct(self, x, lr, scale, clamp01, out):
        _chk_dev(x, lr, out)
        if lr.dim() == 3:                          # one image: a batch of 1
            x, lr, out = x[None], lr[None], out[None]
        assert x.shape[0] == out.shape[0] == lr.shape[0]  # a batch of n images: (n, ...) operands, one launch
        _check(self.lib, self.lib.rv_reconstruct_batched(_ptr(x), x.shape[3], DTYPE_CODE[x.dtype], _ptr(lr), lr.shape[2],
                                                         lr.shape[3], scale, int(clamp01), _ptr(out), lr.shape[0],
                                                         self._stream()), 'rv_reconstruct')

    def reconstruct_u8(self, x, lr, scale, clamp01, out, fmt):
        """reconstruct() with 8-bit output: out, one (scale*h, scale*w) frame of format fmt or (n, ...) of them for a batch, gets
        the bytes frame_u8 makes of the values reconstruct() would write (rv_reconstruct_u8).  fmt: False / 0 RGB and True / 1 BGR
        (out (..., H, W, 3)), FRAME_I420 / FRAME_NV12 (out (..., 3H/2, W), the 4:2:0 frame of those RGB bytes)"""
        _chk_dev(x, lr, out)
        H, W = scale * lr.shape[-2], scale * lr.shape[-1]
        assert out.dtype == torch.uint8 and tuple(out.shape[-len(frame_shape(H, W, fmt)):]) == frame_shape(H, W, fmt)
        if lr.dim() == 3:                          # one image: a batch of 1
            x, lr, out = x[None], lr[None], out[None]
        assert x.shape[0] == out.shape[0] == lr.shape[0]  # a batch of n images: (n, ...) operands, one launch
        _check(self.lib, self.lib.rv_reconstruct_u8_batched(_ptr(x), x.shape[3], DTYPE_CODE[x.dtype], _ptr(lr), lr.shape[2],
                                                            lr.shape[3], scale, int(clamp01), int(fmt), _ptr(out),
                                                            lr.shape[0], self._stream()), 'rv_reconstruct_u8')

    # -- 8-bit frames -----------------------------------------------------------------------------
    def frames_from_u8(self, srcs, dsts, fmt):
        """srcs: contiguous uint8 (h, w) frames of format fmt (see reconstruct_u8), dsts: as many contiguous float32 (3, h, w)
        frames, all of one size on one device; dsts[i] = the RGB planes of fl32(u / 255) of srcs[i]'s R, G, B bytes
        (rv_frames_from_u8, 16 frames per launch)"""
        assert len(srcs) == len(dsts)
        if not srcs:
            return
        h, w = dsts[0].shape[1], dsts[0].shape[2]
        for s, d in zip(srcs, dsts):
            _chk_dev(s, d)
            assert s.dtype == torch.uint8 and tuple(s.shape) == frame_shape(h, w, fmt), f'frames_from_u8: source {tuple(s.shape)} {s.dtype}'
            assert d.dtype == torch.float32 and tuple(d.shape) == (3, h, w), f'frames_from_u8: destination {tuple(d.shape)} {d.dtype}'
        for i in range(0, len(srcs), 16):
            ps = [s.data_ptr() for s in srcs[i:i + 16]]
            pd = [d.data_ptr() for d in dsts[i:i + 16]]
            _check(self.lib, self.lib.rv_frames_from_u8((C.c_void_p * len(ps))(*ps), (C.c_void_p * len(pd))(*pd), len(ps), h, w,
                                                        int(fmt), self._stream()), 'rv_frames_from_u8')

    # -- evaluation metrics -----------------------------------------------------------------------
    def region_metrics(self, a, b, boxes):
        """a, b: contiguous fp32 (1, 3, H, W) CUDA images; boxes: up to 8 (y0, y1, x0, x1) half-open boxes inside the frame.
        Returns float64 numpy arrays (sq, s), each [len(boxes)]: per box, the sum of the float32 squared error and the sum of
        skimage's full-frame SSIM map over the box and the 3 channels (rv_region_metrics).  Synchronises the current stream
        with one 8 * 2 * len(boxes) byte device-to-host copy."""
        for name, t in (('a', a), ('b', b)):
            if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
                raise ValueError(f'region_metrics: {name} must be a contiguous float32 CUDA tensor')
            if t.dim() != 4 or t.shape[0] != 1 or t.shape[1] != 3:
                raise ValueError(f'region_metrics: {name} must be (1, 3, H, W), got {tuple(t.shape)}')
        if a.shape != b.shape or a.device != b.device:
            raise ValueError(f'region_metrics: a {tuple(a.shape)} on {a.device} and b {tuple(b.shape)} on {b.device} differ')
        flat = [int(v) for box in boxes for v in box]
        if len(flat) != 4 * len(boxes):
            raise ValueError('region_metrics: every box is (y0, y1, x0, x1)')
        n, H, W = len(boxes), a.shape[2], a.shape[3]
        need = ((H + 15) // 16) * ((W + 31) // 32) * 2 * n          # RV_REGION_METRICS_WORK(H, W, nbox)
        ws = getattr(self, '_region_ws', None)
        if ws is None or ws[0].device != a.device or ws[0].numel() < need:
            ws = (torch.empty(max(need, 1), dtype=torch.float64, device=a.device), torch.empty(16, dtype=torch.float64, device=a.device))
            self._region_ws = ws
        _check(self.lib, self.lib.rv_region_metrics(_ptr(a), _ptr(b), H, W, (C.c_int32 * max(len(flat), 1))(*flat), n, _ptr(ws[0]),
                                                    _ptr(ws[1]), self._stream()), 'rv_region_metrics')
        host = ws[1][:2 * n].cpu().numpy()
        return host[:n], host[n:]

    def mean_ssim(self, a, b):
        """skimage.metrics.structural_similarity(a, b, data_range=1.0, multichannel=True) of two contiguous fp32 (1, 3, H, W) CUDA
        images, H, W >= 7.  skimage averages its full-frame SSIM map over the interior 3 pixels in from every edge and over the
        channels, so this is one region_metrics call with the single box (3, H - 3, 3, W - 3).  Synchronises the current stream."""
        H, W = a.shape[-2], a.shape[-1]
        _, s = self.region_metrics(a, b, [(3, H - 3, 3, W - 3)])
        return float(s[0] / (3 * (H - 6) * (W - 6)))

    def conf_map_images(self, maps, inp, out, lut, normalize):
        """The image bytes of one frame of the confidence-map evaluation mode (rv_conf_map_images).
        maps: [conf_map, conf_map_prop, conf_map_prop_backward, conf_map_prop_forward] with normalize, [conf_map] without;
        each a contiguous float32 (1, 1, h, w) CUDA tensor.  inp, out: contiguous float32 (1, 3, ih, iw) / (1, 3, oh, ow) RGB
        frames.  lut: uint8 (256, 3) RGB CUDA tensor (refvsr_b200.colormap).  Returns a uint8 CUDA tensor of
        conf_map_bytes(...) bytes: the maps', then the input's, then the output's BGR HWC image, packed.  The tensor is a view
        of a buffer this object reuses: the next call on the stream overwrites it."""
        normalize = bool(normalize)
        if len(maps) != (4 if normalize else 1):
            raise ValueError(f'conf_map_images: {4 if normalize else 1} maps expected with normalize={normalize}, got {len(maps)}')
        for name, t, c in [(f'maps[{k}]', m, 1) for k, m in enumerate(maps)] + [('inp', inp, 3), ('out', out, 3)]:
            if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
                raise ValueError(f'conf_map_images: {name} must be a contiguous float32 CUDA tensor')
            if t.dim() != 4 or t.shape[0] != 1 or t.shape[1] != c:
                raise ValueError(f'conf_map_images: {name} must be (1, {c}, H, W), got {tuple(t.shape)}')
            if t.device != inp.device:
                raise ValueError(f'conf_map_images: {name} is on {t.device}, the input on {inp.device}')
        h, w = maps[0].shape[2:]
        if any(m.shape != maps[0].shape for m in maps):
            raise ValueError(f'conf_map_images: the maps differ in shape: {[tuple(m.shape) for m in maps]}')
        if not (isinstance(lut, torch.Tensor) and lut.dtype == torch.uint8 and lut.shape == (256, 3) and lut.is_contiguous()
                and lut.device == inp.device):
            raise ValueError('conf_map_images: lut must be a contiguous uint8 (256, 3) tensor on the frames\' device')
        ih, iw, oh, ow = inp.shape[2], inp.shape[3], out.shape[2], out.shape[3]
        need = conf_map_bytes(h, w, ih, iw, oh, ow, normalize)
        ws = getattr(self, '_conf_ws', None)
        if ws is None or ws[0].device != inp.device or ws[1].numel() < need:
            ws = (torch.empty(CONF_MAP_WORK, dtype=torch.int32, device=inp.device), torch.empty(need, dtype=torch.uint8, device=inp.device))
            self._conf_ws = ws
        m = list(maps) + [None] * (4 - len(maps))
        _check(self.lib, self.lib.rv_conf_map_images(_ptr(m[0]), _ptr(m[1]), _ptr(m[2]), _ptr(m[3]), h, w, int(normalize), _ptr(inp),
                                                     ih, iw, _ptr(out), oh, ow, _ptr(lut), _ptr(ws[0]), _ptr(ws[1]), self._stream()),
               'rv_conf_map_images')
        return ws[1][:need]

    def eval_images(self, frames):
        """The image bytes of one frame of the default evaluation mode (rv_eval_images).  frames: 1 to 3 contiguous float32
        (1, 3, H, W) RGB CUDA tensors on one device (the input, the output, the ground truth; sizes may differ).  Returns a uint8
        CUDA tensor of sum(3 * H * W) bytes: each frame's BGR HWC image as cv2.imwrite stores cv2.cvtColor(x * 255, RGB2BGR),
        packed in the order given.  The tensor is a view of a buffer this object reuses: the next call on the stream overwrites it."""
        if not 1 <= len(frames) <= 3:
            raise ValueError(f'eval_images: 1 to 3 frames, got {len(frames)}')
        for k, t in enumerate(frames):
            if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
                raise ValueError(f'eval_images: frames[{k}] must be a contiguous float32 CUDA tensor')
            if t.dim() != 4 or t.shape[0] != 1 or t.shape[1] != 3:
                raise ValueError(f'eval_images: frames[{k}] must be (1, 3, H, W), got {tuple(t.shape)}')
            if t.device != frames[0].device:
                raise ValueError(f'eval_images: frames[{k}] is on {t.device}, frames[0] on {frames[0].device}')
        hw = [int(v) for t in frames for v in t.shape[2:]]
        need = sum(3 * t.shape[2] * t.shape[3] for t in frames)
        buf = getattr(self, '_eval_images_buf', None)
        if buf is None or buf.device != frames[0].device or buf.numel() < need:
            buf = torch.empty(need, dtype=torch.uint8, device=frames[0].device)
            self._eval_images_buf = buf
        ptrs = (C.c_void_p * len(frames))(*[t.data_ptr() for t in frames])
        _check(self.lib, self.lib.rv_eval_images(ptrs, (C.c_int * len(hw))(*hw), len(frames), _ptr(buf), self._stream()),
               'rv_eval_images')
        return buf[:need]
