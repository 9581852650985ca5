"""ctypes binding of the C-ABI shared library (include/dasr_b200.h).

The library is the product: if it is missing or cannot be loaded every operator raises — there is no
PyTorch/CPU fallback anywhere in this package.  Build it with ``python -c "import __graft_entry__ as g;
g.build()"`` (or ``make -C dasr_b200/csrc``); it lives in-tree at ``dasr_b200/lib/libdasr_b200.so``.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'lib', 'libdasr_b200.so')

_lib = None


class DasrError(RuntimeError):
    pass


class ConvF32Params(C.Structure):
    _fields_ = [
        ('N', C.c_int), ('H', C.c_int), ('W', C.c_int),
        ('cin', C.c_int), ('in_cs', C.c_int), ('in_coff', C.c_int),
        ('OH', C.c_int), ('OW', C.c_int),
        ('cout', C.c_int), ('out_cs', C.c_int), ('out_coff', C.c_int),
        ('kh', C.c_int), ('kw', C.c_int), ('stride', C.c_int), ('pad', C.c_int),
        ('ups', C.c_int), ('mode', C.c_int),
        ('act', C.c_int), ('slope', C.c_float),
        ('alpha', C.c_float),
        ('beta1', C.c_float), ('res1_cs', C.c_int), ('res1_coff', C.c_int),
        ('beta2', C.c_float), ('res2_cs', C.c_int), ('res2_coff', C.c_int),
        ('math', C.c_int),
    ]


class ConvTcParams(C.Structure):
    _fields_ = [
        ('N', C.c_int), ('H', C.c_int), ('W', C.c_int),
        ('cin', C.c_int), ('in_cs', C.c_int), ('in_coff', C.c_int),
        ('cout', C.c_int), ('out_cs', C.c_int), ('out_coff', C.c_int),
        ('nt', C.c_int), ('out_mul', C.c_int), ('nvar', C.c_int), ('ntaps', C.c_int),
        ('tap_dy', (C.c_int8 * 9) * 4), ('tap_dx', (C.c_int8 * 9) * 4),
        ('out_py', C.c_int * 4), ('out_px', C.c_int * 4),
        ('act', C.c_int), ('slope', C.c_float), ('alpha', C.c_float),
        ('beta1', C.c_float), ('res1_cs', C.c_int), ('res1_coff', C.c_int),
        ('beta2', C.c_float), ('res2_cs', C.c_int), ('res2_coff', C.c_int),
        ('mask_cs', C.c_int), ('mask_coff', C.c_int), ('mask_c0', C.c_int), ('mask_c1', C.c_int),
        ('mask_slope', C.c_float),
        ('a_mode', C.c_int), ('epi_mode', C.c_int), ('act_cols', C.c_int),
        ('pre_cs', C.c_int), ('pre_coff', C.c_int), ('out_nc', C.c_int), ('tile_rev', C.c_int),
        ('nchunk_list', C.c_int), ('chunk_off', C.c_int * 8), ('f16', C.c_int),
        ('map_mode', C.c_int), ('map_scale', C.c_float), ('map_stride', C.c_int),
    ]


class PackJob(C.Structure):
    """DasrPackJob (include/dasr_b200.h)"""
    _fields_ = [('src', C.c_void_p), ('dst', C.c_void_p), ('cout', C.c_int), ('cin', C.c_int), ('kind', C.c_int),
                ('ci_lo', C.c_int), ('ci_n', C.c_int), ('cout_rows', C.c_int), ('k_pad', C.c_int), ('dst_rows', C.c_int),
                ('dst_row_off', C.c_int), ('reserved', C.c_int)]


# every symbol include/dasr_b200.h declares: name -> (restype, argtypes)
_vp, _i, _f, _l, _sz = C.c_void_p, C.c_int, C.c_float, C.c_long, C.c_size_t
SYMBOLS = {
    'dasr_last_error': (C.c_char_p, []),
    'dasr_version': (_i, []),
    'dasr_conv2d_f32': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, C.POINTER(ConvF32Params), _vp]),
    'dasr_conv2d_in_lrelu_f32': (_i, [_vp, _vp, _vp, _vp, _vp, C.POINTER(ConvF32Params), _f, _vp]),
    'dasr_conv2d_wgrad_f32_workspace': (_sz, [C.POINTER(ConvF32Params)]),
    'dasr_conv2d_wgrad_f32': (_i, [_vp, _vp, _vp, _vp, C.POINTER(ConvF32Params), _i, _vp, _sz, _vp]),
    'dasr_conv2d_wgrad_bf16': (_i, [_vp, _vp, _vp, _vp, C.POINTER(ConvF32Params), _i, _vp, _sz, _vp]),
    'dasr_conv3x3_wgrad_tc_workspace': (_sz, [_i, _i, _i, _i, _i]),
    'dasr_conv3x3_wgrad_tc': (_i, [_vp, _i, _i, _vp, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _vp, _sz, _vp]),
    'dasr_bias_grad': (_i, [_vp, _vp, _l, _i, _i, _i, _i, _i, _vp, _vp]),
    'dasr_upsample2x_fwd': (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    'dasr_pack_filter_f32': (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp]),
    'dasr_conv_tc': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.POINTER(ConvTcParams), _vp]),
    'dasr_conv_tc2_supported': (_i, [C.POINTER(ConvTcParams)]),
    'dasr_conv_tc2': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, C.POINTER(ConvTcParams), _vp]),
    'dasr_conv_tc_map': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.POINTER(ConvTcParams), _vp]),
    'dasr_conv_tc2_map': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.POINTER(ConvTcParams), _vp]),
    'dasr_conv_tc_setup': (_i, [C.POINTER(ConvTcParams), _i]),
    'dasr_pack_filter_tc_bytes': (_sz, [_i, _i, _i]),
    'dasr_pack_filter_tc': (_i, [_vp, _vp, _i, _i, _i, _vp]),
    'dasr_nchw_to_nhwc': (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    'dasr_nhwc_to_nchw': (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    'dasr_act_bwd': (_i, [_vp, _vp, _l, _i, _i, _i, _i, _i, _f, _i, _vp]),
    'dasr_upsample2x_bwd': (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    'dasr_axpby': (_i, [_vp, _vp, _vp, _l, _i, _i, _i, _i, _i, _i, _i, _f, _f, _i, _vp]),
    'dasr_map_axpby': (_i, [_vp, _vp, _vp, _vp, _l, _i, _i, _i, _i, _i, _i, _i, _f, _f, _vp]),
    'dasr_maxpool2_fwd': (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    'dasr_maxpool2_bwd': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    'dasr_maxpool2_fwd_bf16': (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    'dasr_maxpool2_bwd_bf16': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    'dasr_instnorm_lrelu_fwd': (_i, [_vp, _vp, _i, _i, _i, _f, _f, _vp]),
    'dasr_instnorm_lrelu_bwd': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _f, _vp]),
    'dasr_haar_fwd': (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    'dasr_haar_bwd': (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    'dasr_dwfilter_fwd': (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    'dasr_dwfilter_bwd': (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    'dasr_bilinear_fwd': (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp]),
    'dasr_wl1_loss': (_i, [_vp, _vp, _vp, _vp, _vp, _f, _i, _i, _i, _vp, _vp]),
    'dasr_mse_loss': (_i, [_vp, _vp, _vp, _vp, _f, _l, _vp, _vp]),
    'dasr_bce_logits_loss': (_i, [_vp, _f, _vp, _vp, _f, _l, _vp, _vp]),
    'dasr_mean': (_i, [_vp, _vp, _l, _vp, _vp]),
    'dasr_pack_filter_tc_batch': (_i, [_vp, _i, _i, _vp]),
    'dasr_rdb_wgrad_tc_workspace': (_sz, [_i, _i, _i]),
    'dasr_rdb_wgrad_tc': (_i, [_vp, _i, _vp, _i, _i, _vp, _i, _i, C.POINTER(_vp), _i, _i, _i, _i, _vp, _sz, _vp]),
    'dasr_maxpool_fwd': (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    'dasr_maxpool_bwd': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    'dasr_lpips_layer_fwd': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _i, _vp]),
    'dasr_lpips_layer_bwd': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _i, _vp]),
    'dasr_bn_lrelu_fwd': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _l, _i, _f, _f, _i, _f, _vp]),
    'dasr_bn_lrelu_bwd': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _l, _i, _i, _f, _vp]),
    'dasr_pixel_shuffle': (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    'dasr_ddm': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    'dasr_log_loss': (_i, [_vp, _i, _f, _vp, _vp, _f, _l, _vp, _vp]),
    'dasr_prelu_fwd': (_i, [_vp, _vp, _vp, _l, _vp]),
    'dasr_prelu_bwd': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _l, _vp, _vp]),
    'dasr_prelu_fwd_bf16': (_i, [_vp, _vp, _vp, _l, _vp]),
    'dasr_prelu_bwd_bf16': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _l, _vp, _vp]),
    'dasr_cast_bf16_f32': (_i, [_vp, _vp, _l, _i, _vp]),
    'dasr_sigmoid_fwd': (_i, [_vp, _vp, _l, _vp]),
    'dasr_sigmoid_bwd': (_i, [_vp, _vp, _vp, _l, _vp]),
}


def load():
    """Load the shared library (once).  Raises DasrError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise DasrError('dasr_b200: %s not found — build it first (python -c "import __graft_entry__ as g; g.build()"). '
                        'There is no fallback path.' % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the header and the library disagree
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


LAUNCHES = 0   # kernels launched through the C ABI since import (bench.py reports the delta)


def check(rc, what, kernels=1):
    global LAUNCHES
    LAUNCHES += kernels
    if rc != 0:
        msg = load().dasr_last_error()
        raise DasrError('%s failed (rc=%d): %s' % (what, rc, msg.decode() if msg else ''))
