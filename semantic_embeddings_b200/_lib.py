"""ctypes binding of include/se_b200.h (the C-ABI drop-in boundary).

The product path has no CPU fallback: if `libse_b200.so` is missing or a call fails,
an exception is raised.  PyTorch tensors are only containers -- every entry point gets
raw `data_ptr()`s and the current CUDA stream.
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libse_b200.so')

SE_MODE_F32, SE_MODE_TF32, SE_MODE_TF32X3 = 0, 1, 2
MODE_NAMES = {0: 'f32', 1: 'tf32', 2: 'tf32x3'}
SE_LOSS_INV_CORR, SE_LOSS_UNNORM_CORR, SE_LOSS_MSE, SE_LOSS_SOFTMAX_CORR, SE_LOSS_DEVISE_RANK = 0, 1, 2, 3, 4
SE_PDIST_SQEUCLID, SE_PDIST_NEGDOT = 0, 1
SE_SCALE_ROW_L2, SE_SCALE_COL_MAXABS, SE_SCALE_COL_DIV, SE_SCALE_MUL = 0, 1, 2, 3
SE_ERR_NOT_CONVERGED = -4
SE_ERR_ARG = -1
SE_RESAMPLE_MAX_SIDE, SE_RESAMPLE_MAX_CROP = 4096, 1024
SE_GRAM_SIM, SE_GRAM_SPHERES = 0, 1
SE_COL_SQNORM, SE_COL_CENTER = 0, 1
SE_DEV_SIM, SE_DEV_DIST = 0, 1
# se_bn_bwd_path: bits 0-1 = path (0 reduce + apply, 1 shared-memory slab, 2 register slab), bit 2 = float4 / fixed quad
SE_BN_BWD_SCALAR, SE_BN_BWD_SLAB_ATOMIC, SE_BN_BWD_SLAB_REG, SE_BN_BWD_VEC, SE_BN_BWD_SLAB_QUAD = 0, 1, 2, 4, 5
# se_embed_head_path: bits 0-1 = configuration (one warp per row, class matrix in shared memory, one CTA per row),
# bit 2 = float4 loads
SE_HEAD_WARP, SE_HEAD_SMEM, SE_HEAD_SPLIT, SE_HEAD_VEC = 0, 1, 2, 4

# opcodes of se_run_ops (csrc/opcodes.h)
OP_CONV_FWD, OP_CONV_DGRAD, OP_CONV_WGRAD, OP_BN_STATS, OP_BN_FWD_TRAIN, OP_BN_FWD_INFER, OP_BN_BWD, \
    OP_SHORTCUT_BWD, OP_AVGPOOL_FWD, OP_AVGPOOL_BWD, OP_MAXPOOL_FWD, OP_MAXPOOL_BWD, OP_GAP_FWD, OP_GAP_BWD, \
    OP_ADD_FWD, OP_ADD_BWD, OP_HEAD, OP_XENT, OP_MEMSET, OP_SGD_PREPARE, OP_SGD_APPLY, OP_TRANSPOSE_FILTERS, \
    OP_CONV_BN_FWD, OP_ALLREDUCE, OP_ADAGRAD_APPLY, OP_LABELEMBED, OP_CENTER_LOSS = range(1, 28)


class SeError(RuntimeError):
    def __init__(self, msg, rc=None):
        RuntimeError.__init__(self, msg)
        self.rc = rc


class ConvDesc(ctypes.Structure):
    _fields_ = [(n, c_int32) for n in ('N', 'H', 'W', 'Cin', 'Cout', 'kh', 'kw', 'stride', 'pad_t', 'pad_l', 'Ho', 'Wo')]


class Residual(ctypes.Structure):
    _fields_ = [('ptr', c_void_p), ('C', c_int32), ('pad_lo', c_int32), ('pool', c_int32), ('H', c_int32), ('W', c_int32)]


class ConvAux(ctypes.Structure):
    _fields_ = [('w_t', c_void_p), ('w_t_lo', c_void_p), ('w_lo', c_void_p)]


class L2Segment(ctypes.Structure):
    _fields_ = [('begin', c_int64), ('end', c_int64), ('l2', c_float)]


class ResampleDesc(ctypes.Structure):
    """se_resample_desc: one image of se_resample_crop_batch."""
    _fields_ = [('src_offset', c_int64)] + [(n, c_int32) for n in ('src_h', 'src_w', 'rh', 'rw', 'flip', 'ey', 'ex', 'eh',
                                                                     'ew', 'cy', 'cx', 'noise_id')]


class JpegHuff(ctypes.Structure):
    """se_jpeg_huff: one Huffman table in lookup form."""
    _fields_ = [('lookup', ctypes.c_uint16 * 512), ('maxcode', c_int32 * 18), ('valoffset', c_int32 * 18),
                ('huffval', ctypes.c_uint8 * 256)]


class JpegInfo(ctypes.Structure):
    """se_jpeg_info: what se_jpeg_parse reads from a JPEG file's headers."""
    _fields_ = ([(n, c_int32) for n in ('status', 'width', 'height', 'ncomp')] +
                [(n, c_int32 * 3) for n in ('comp_id', 'h', 'v', 'tq', 'td', 'ta')] +
                [(n, c_int32) for n in ('hmax', 'vmax', 'mcus_x', 'mcus_y', 'restart_interval', 'n_intervals', 'n_subseq',
                                        'saw_jfif', 'saw_adobe', 'adobe_transform', 'qt_mask', 'reserved')] +
                [(n, c_int64) for n in ('scan_begin', 'scan_end', 'data_bytes', 'packed_bytes')] +
                [('qt', (ctypes.c_uint16 * 64) * 4), ('dc', JpegHuff * 4), ('ac', JpegHuff * 4)])


class JpegJob(ctypes.Structure):
    """se_jpeg_job: one image of se_jpeg_decode_batch."""
    _fields_ = [(n, c_int64) for n in ('info_offset', 'packed_offset', 'out_offset', 'ws_offset')]


# se_jpeg_info.status (include/se_b200.h): why a file is not decoded on the device
JPEG_REASONS = ('ok', 'not_jpeg', 'truncated', 'malformed', 'progressive', 'arithmetic', 'other_process', 'precision',
                'components', 'colorspace', 'sampling', 'multiscan', 'size', 'restart')
SE_JPEG_OK, SE_JPEG_DEV_CORRUPT, SE_JPEG_SUBSEQ_BYTES = 0, 1, 128


class Op(ctypes.Structure):
    _fields_ = [('opcode', c_int32), ('i', c_int32 * 15), ('f', c_float * 8), ('p', c_void_p * 16)]


_P = c_void_p
_SIGS = {
    'se_version': (c_char_p, []),
    'se_last_error': (c_char_p, []),
    'se_launch_count': (c_int64, []),
    'se_device_sm_count': (c_int, []),
    'se_init': (c_int, []),
    'se_tc_capabilities': (c_int, []),
    'se_conv2d_fwd': (c_int, [POINTER(ConvDesc), _P, _P, _P, _P, _P, c_int, _P, c_int, _P]),
    'se_conv2d_fwd_ex': (c_int, [POINTER(ConvDesc), _P, _P, _P, _P, _P, _P, c_int, _P, c_int, _P]),
    'se_conv2d_fwd_aux': (c_int, [POINTER(ConvDesc), _P, _P, POINTER(ConvAux), _P, _P, _P, c_int, _P, c_int, _P]),
    'se_conv2d_dgrad_aux': (c_int, [POINTER(ConvDesc), _P, _P, POINTER(ConvAux), _P, c_float, c_int, _P]),
    'se_split_filters': (c_int, [_P, _P, _P, _P, POINTER(c_int64), c_int, _P]),
    'se_hier_precision': (c_int, [_P, c_int, c_int, c_int, c_int, _P, c_int, _P, _P, _P, _P, _P, c_int, c_int, _P, _P]),
    'se_row_topk': (c_int, [_P, c_int64, c_int, c_int, c_int, _P, _P, c_int, _P]),
    'se_conv_bn_fwd': (c_int, [POINTER(ConvDesc), _P, _P, _P, _P, _P, c_int, _P, _P, _P, c_float, c_float, _P, _P, _P, _P, _P,
                               c_int, _P, _P, c_int, _P]),
    'se_transpose_filters': (c_int, [_P, _P, POINTER(c_int64), c_int, _P]),
    'se_conv2d_dgrad': (c_int, [POINTER(ConvDesc), _P, _P, _P, c_float, c_int, _P]),
    'se_conv2d_wgrad': (c_int, [POINTER(ConvDesc), _P, _P, _P, _P, c_int, _P]),
    'se_conv2d_path': (c_int, [POINTER(ConvDesc), c_int, c_int]),
    'se_dense_fwd': (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, _P, c_int, _P]),
    'se_dense_bwd': (c_int, [_P, _P, _P, _P, c_float, _P, _P, c_int, c_int, c_int, c_int, _P]),
    'se_bn_stats': (c_int, [_P, c_int64, c_int, _P, _P]),
    'se_bn_fwd_train': (c_int, [_P, c_int64, c_int, _P, _P, _P, c_float, c_float, _P, _P, _P, _P, POINTER(Residual), c_int, _P, _P]),
    'se_bn_fwd_infer': (c_int, [_P, c_int64, c_int, _P, _P, _P, _P, c_float, POINTER(Residual), c_int, _P, _P]),
    'se_bn_bwd': (c_int, [_P, _P, _P, c_int64, c_int, _P, _P, _P, c_int, c_int, _P, c_float, _P, c_float, _P, _P, _P, _P]),
    'se_bn_bwd_path': (c_int, [c_int64, c_int, c_int]),
    'se_shortcut_bwd': (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, POINTER(Residual), _P, c_float, _P]),
    'se_avgpool2_fwd': (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    'se_avgpool2_bwd': (c_int, [_P, _P, c_float, c_int, c_int, c_int, c_int, _P]),
    'se_maxpool_fwd': (c_int, [_P, _P] + [c_int] * 10 + [_P]),
    'se_maxpool_bwd': (c_int, [_P, _P, _P, _P] + [c_int] * 10 + [_P]),
    'se_gap_fwd': (c_int, [_P, _P, c_int, c_int, c_int, _P]),
    'se_gap_bwd': (c_int, [_P, _P, c_float, c_int, c_int, c_int, _P]),
    'se_add_fwd': (c_int, [_P, _P, _P, c_int64, c_int, _P]),
    'se_add_bwd': (c_int, [_P, _P, c_int, _P, c_float, _P, c_float, c_int64, _P]),
    'se_relu_fwd': (c_int, [_P, _P, c_int64, _P]),
    'se_relu_bwd': (c_int, [_P, _P, _P, c_float, c_int64, _P]),
    'se_embed_head_fwd_bwd': (c_int, [_P, c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float, _P, _P, _P, _P, _P, _P]),
    'se_softmax_xent_fwd_bwd': (c_int, [_P, c_int, _P, c_int, c_int, c_float, _P, _P, _P, _P, _P]),
    'se_softmax_xent_fwd_bwd_ex': (c_int, [_P, c_int, _P, c_int, c_int, c_float, _P, _P, _P, _P, _P, _P]),
    'se_softmax_xent_smooth_fwd_bwd': (c_int, [_P, c_int, _P, c_int, c_int, c_float, c_float, _P, _P, _P, _P, _P, _P]),
    'se_embed_head_fwd_bwd_ex': (c_int, [_P, c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float, _P, _P, _P, _P, _P, _P, _P]),
    'se_devise_rank_fwd_bwd': (c_int, [_P, c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float, _P, _P, _P, _P, _P, _P,
                                       c_float, _P]),
    'se_embed_head_path': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int]),
    'se_labelembed_workspace_bytes': (c_int64, [c_int, c_int]),
    'se_labelembed_fwd_bwd': (c_int, [_P, _P, c_int, _P, _P, c_int, c_int, c_int, c_float, c_float, c_float, c_float, _P, _P,
                                      _P, _P, _P, _P, _P]),
    'se_center_loss_fwd_bwd': (c_int, [_P, c_int, _P, _P, c_int, c_int, c_int, c_int, c_float, _P, _P, _P, _P]),
    'se_linear_svm_workspace_bytes': (c_int64, [c_int, c_int, c_int]),
    'se_linear_svm_fit': (c_int, [_P, c_int64, c_int, c_int, _P, c_int, c_float, c_float, c_int, _P, _P, _P, _P, _P, _P]),
    'se_scale_features': (c_int, [_P, c_int64, c_int, c_int, c_int, _P, c_float, _P, c_int64, _P]),
    'se_sgd_schedule': (c_int, [_P, _P]),
    'se_pairwise_topk_workspace_bytes': (c_int64, [c_int, c_int, c_int]),
    'se_pairwise_topk': (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, c_int, _P, _P, _P]),
    'se_comm_unique_id': (c_int, [_P, c_int]),
    'se_comm_init': (c_int, [c_int, c_int, _P, c_int]),
    'se_comm_world': (c_int, []),
    'se_allreduce_sum': (c_int, [_P, c_int64, _P]),
    'se_comm_destroy': (c_int, []),
    'se_hier_metrics': (c_int, [_P, c_int64, c_int, c_int, c_int, _P, c_int, _P, _P, _P, _P, c_int, c_int, _P, _P, _P, _P]),
    'se_row_argsort_workspace_bytes': (c_int64, [c_int, c_int]),
    'se_row_argsort': (c_int, [_P, c_int64, c_int, c_int, _P, c_int64, _P, _P]),
    'se_class_index': (c_int, [_P, c_int, c_int, _P, _P, _P]),
    'se_relevant_positions': (c_int, [_P, c_int64, c_int, c_int, c_int, _P, c_int, _P, _P, _P, _P, _P]),
    'se_augment_batch': (c_int, [_P, c_int, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    'se_resample_crop_batch': (c_int, [_P, _P, _P, c_int, c_int, c_int, POINTER(c_float), POINTER(c_float), c_int,
                                       ctypes.c_uint64, _P, _P]),
    'se_jpeg_parse': (c_int, [_P, c_int64, POINTER(JpegInfo)]),
    'se_jpeg_pack': (c_int64, [_P, c_int64, POINTER(JpegInfo), _P, c_int64]),
    'se_jpeg_workspace_bytes': (c_int64, [_P, _P, c_int]),
    'se_jpeg_decode_batch': (c_int, [_P, _P, _P, _P, c_int, _P, _P, _P, c_int64, _P]),
    'se_jpeg_layout': (c_int, [POINTER(c_int64), c_int]),
    'se_sgd_step': (c_int, [_P, _P, _P, c_int64, POINTER(L2Segment), c_int, c_float, c_float, c_int, c_float, _P, _P]),
    'se_sgd_prepare': (c_int, [_P, _P, c_int64, POINTER(L2Segment), c_int, _P, _P]),
    'se_sgd_apply': (c_int, [_P, _P, _P, c_int64, c_float, c_float, c_int, c_float, _P, _P]),
    'se_sgd_apply_devlr': (c_int, [_P, _P, _P, c_int64, _P, c_float, c_int, c_float, _P, _P]),
    'se_adagrad_apply_devlr': (c_int, [_P, _P, _P, c_int64, _P, c_float, c_float, _P, _P]),
    'se_pairwise_workspace_bytes': (c_int64, [c_int, c_int, c_int]),
    'se_pairwise_dist': (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, c_int64, _P, c_int, _P]),
    'se_cross_workspace_bytes': (c_int64, [c_int, c_int, c_int, c_int]),
    'se_cross_dist': (c_int, [_P, c_int, c_int, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, c_int64, _P, c_int,
                              _P]),
    'se_cross_topk_workspace_bytes': (c_int64, [c_int, c_int, c_int, c_int]),
    'se_cross_topk': (c_int, [_P, c_int, c_int, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, c_int, _P,
                              _P, _P]),
    'se_hier_metrics_q': (c_int, [_P, c_int64, c_int, c_int, _P, _P, c_int, _P, _P, _P, _P, c_int, c_int, _P, _P, _P, _P]),
    'se_relevant_positions_q': (c_int, [_P, c_int64, c_int, c_int, _P, _P, c_int, _P, _P, _P, _P, _P]),
    'se_lcs_height_table': (c_int, [_P, _P, _P, c_int, c_int, c_int, _P, c_int64, _P]),
    'se_cholesky_f64': (c_int, [_P, c_int64, c_int, _P, _P]),
    'se_class_gram_f64': (c_int, [_P, c_int64, c_int, c_int, _P, c_int64, _P]),
    'se_column_op_f64': (c_int, [_P, c_int64, c_int, c_int, c_int, _P, _P]),
    'se_gather_columns_f64': (c_int, [_P, c_int64, c_int, _P, c_int, _P, c_int64, _P]),
    'se_row_normalize_f64': (c_int, [_P, c_int64, c_int, c_int, _P]),
    'se_jacobi_columns_workspace_bytes': (c_int64, [c_int, c_int]),
    'se_jacobi_columns_f64': (c_int, [_P, c_int64, c_int, c_int, c_int, POINTER(c_int32), _P, _P]),
    'se_embedding_deviation_workspace_bytes': (c_int64, [c_int]),
    'se_embedding_deviation_f64': (c_int, [_P, c_int64, c_int, c_int, _P, c_int64, c_int, _P, _P, _P]),
    'se_run_ops': (c_int, [POINTER(Op), c_int, c_int, _P]),
    'se_run_ops_timed': (c_int, [POINTER(Op), c_int, c_int, _P, POINTER(c_float)]),
}

_lib = None


def exported_symbols():
    """Names include/se_b200.h declares (used by the CPU-side ABI test)."""
    return sorted(_SIGS)


def load():
    """Loads the shared library once; raises SeError when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SeError('%s not found: build it with `python -c "import __graft_entry__ as g; g.build()"` '
                          '(there is no CPU fallback)' % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(rc, what=''):
    if rc != 0:
        msg = load().se_last_error().decode('utf-8', 'replace')
        raise SeError('%s failed (rc=%d): %s' % (what or 'se_b200 call', rc, msg), rc)


def ptr(t):
    """Raw device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def stream_ptr():
    import torch
    return torch.cuda.current_stream().cuda_stream


def call(name, *args):
    fn = getattr(load(), name)
    check(fn(*args), name)


def launch_count():
    return int(load().se_launch_count())
