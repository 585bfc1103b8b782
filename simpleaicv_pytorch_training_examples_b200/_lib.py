"""ctypes binding of libsaicv_b200.so (the C ABI in include/saicv_b200.h).

The library is built in-tree by ``__graft_entry__.build()`` (``make -C csrc``).  There is no
fallback: if the shared object is missing, or a call fails, a RuntimeError is raised.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libsaicv_b200.so')
BN_PARTIAL_ROWS = 264  # SAICV_BN_PARTIAL_ROWS

c_void_p = ctypes.c_void_p
c_int = ctypes.c_int
c_ll = ctypes.c_longlong
c_float = ctypes.c_float


class ConvShape(ctypes.Structure):
    """saicv_conv_shape (include/saicv_b200.h)."""
    _fields_ = [('n', c_int), ('h', c_int), ('w', c_int), ('c', c_int),
                ('k', c_int), ('r', c_int), ('s', c_int), ('stride', c_int),
                ('pad', c_int)]


class AttnArgs(ctypes.Structure):
    """saicv_attn_args (include/saicv_b200.h)."""
    _fields_ = [('q', c_void_p), ('k', c_void_p), ('v', c_void_p), ('out', c_void_p), ('lse', c_void_p),
                ('q_strides', c_ll * 3), ('k_strides', c_ll * 3), ('v_strides', c_ll * 3), ('o_strides', c_ll * 3),
                ('key_mask_bits', c_void_p), ('mask_words', c_int),
                ('b', c_int), ('h', c_int), ('lq', c_int), ('lk', c_int), ('dqk', c_int), ('dv', c_int),
                ('scale', c_float), ('dropout_p', c_float), ('dropout_seed', ctypes.c_ulonglong),
                ('dropout_seed_base', c_void_p)]


class AttnBwdArgs(ctypes.Structure):
    """saicv_attn_bwd_args (include/saicv_b200.h)."""
    _fields_ = [('fwd', AttnArgs), ('dout', c_void_p), ('delta', c_void_p),
                ('dq', c_void_p), ('dk', c_void_p), ('dv', c_void_p),
                ('dq_strides', c_ll * 3), ('dk_strides', c_ll * 3), ('dv_strides', c_ll * 3), ('dk_cols', c_int)]


# name -> argtypes; every symbol declared in include/saicv_b200.h is listed here and
# tests/test_capi_symbols.py checks the header, this table and the .so agree.
SIGNATURES = {
    'saicv_version': [],
    'saicv_sm_count': [],
    'saicv_linear_fwd': [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_gemm_stats_rows': [c_ll, c_int],
    'saicv_linear_dgrad': [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_linear_wgrad': [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_wgrad_splits': [c_int, c_int, c_ll],
    'saicv_wgrad_transposed': [c_int, c_int],
    'saicv_conv_fprop': [c_void_p, c_void_p, c_void_p, c_void_p, ctypes.POINTER(ConvShape), c_int, c_void_p],
    'saicv_conv_dgrad': [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.POINTER(ConvShape), c_void_p],
    'saicv_conv_wgrad': [c_void_p, c_void_p, c_void_p, ctypes.POINTER(ConvShape), c_int, c_void_p],
    'saicv_prep_conv_weight': [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_finish_conv_wgrad': [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_reduce_partials': [c_void_p, c_void_p, c_int, c_ll, c_int, c_void_p],
    'saicv_cast_bf16': [c_void_p, c_void_p, c_ll, c_void_p],
    'saicv_nchw_to_nhwc_bf16': [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_stem_kpad': [c_int, c_int, c_int],
    'saicv_stem_im2col': [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_zero_upsample2': [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_add_strided2': [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_bn_stats': [c_void_p, c_void_p, c_ll, c_int, c_void_p],
    'saicv_bn_finalize': [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_float, c_float, c_void_p],
    'saicv_bn_apply': [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_void_p],
    'saicv_bn_bwd_reduce': [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_void_p],
    'saicv_bn_bwd_apply': [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_void_p],
    'saicv_bn_bwd_reduce2': [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_void_p],
    'saicv_bn_bwd_apply2': [c_void_p] * 15 + [c_ll, c_int, c_int, c_int, c_void_p],
    'saicv_add_bf16': [c_void_p, c_void_p, c_ll, c_void_p],
    'saicv_maxpool3x3s2_fwd': [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_maxpool3x3s2_bwd': [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_maxpool_fwd': [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_maxpool_bwd': [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_avgpool_fwd': [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    'saicv_avgpool_bwd': [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    'saicv_colsum': [c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_void_p],
    'saicv_layernorm_fwd': [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_float, c_void_p],
    'saicv_layernorm_bwd': [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_void_p],
    'saicv_gelu_fwd': [c_void_p, c_void_p, c_ll, c_void_p],
    'saicv_gelu_bwd': [c_void_p, c_void_p, c_void_p, c_ll, c_void_p],
    'saicv_vit_assemble_tokens': [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    'saicv_vit_assemble_tokens_bwd': [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_token_pool_fwd': [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_token_pool_bwd': [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_attention_fwd': [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p],
    'saicv_attention_bwd': [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p],
    'saicv_attn_fwd': [ctypes.POINTER(AttnArgs), c_void_p],
    'saicv_attn_bwd': [ctypes.POINTER(AttnBwdArgs), c_void_p],
    'saicv_window_partition': [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_window_unpartition': [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_add_pos_embed': [c_void_p, c_void_p, c_int, c_ll, c_void_p],
    'saicv_relpos_pack_q': [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_relpos_table': [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_relpos_gather': [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p],
    'saicv_relpos_shift': [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_relpos_dq_combine': [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p],
    'saicv_sam_loss_partial_floats': [c_int, c_int, c_ll],
    'saicv_sam_loss_sums': [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_ll, c_float, c_float, c_float, c_void_p],
    'saicv_sam_loss_bwd': [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_ll, c_float, c_float, c_void_p],
    'saicv_u8_nhwc_to_nchw_norm': [c_void_p, c_void_p, c_int, c_int, c_int, ctypes.POINTER(c_float), ctypes.POINTER(c_float), c_void_p],
    'saicv_token_gather_fwd': [c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    'saicv_token_fill_slabs': [c_ll],
    'saicv_token_gather_bwd': [c_void_p, c_void_p, c_void_p, c_int, c_ll, c_void_p, c_int, c_int, c_int, c_void_p],
    'saicv_opt_chunk': [],
    'saicv_multi_tensor_sgd': [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p],
    'saicv_multi_tensor_adamw': [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p],
    'saicv_multi_tensor_clip_coef': [c_void_p, c_void_p, c_void_p, c_int, c_float, c_void_p, c_void_p, c_void_p],
    'saicv_postln_fwd': [c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_int, c_void_p],
    'saicv_postln_bwd': [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_void_p],
    'saicv_add_pos_cast': [c_void_p, c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_int, c_void_p],
    'saicv_dropout': [c_void_p, c_int, c_void_p, c_void_p, c_ll, c_void_p, c_int, c_ll, c_float, ctypes.c_ulonglong, c_void_p, c_void_p],
    'saicv_heads_pack': [c_void_p, c_int, c_int, c_void_p, c_float, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p],
    'saicv_heads_unpack': [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p],
    'saicv_dwconv_fwd': [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_dwconv_dgrad_masked': [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_avgpool_stream_fwd': [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p],
    'saicv_avgpool_stream_bwd': [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_dwconv_wgrad_blocks': [c_ll],
    'saicv_dwconv_wgrad': [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_mul_bf16': [c_void_p, c_void_p, c_void_p, c_ll, c_void_p],
    'saicv_gate_bwd': [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_void_p],
    'saicv_ls_residual_fwd': [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_ll, c_int, c_void_p],
    'saicv_ls_residual_bwd': [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_void_p],
    'saicv_bn_generic_partial_rows': [c_ll, c_int],
    'saicv_bn_stats_generic': [c_void_p, c_int, c_void_p, c_ll, c_int, c_void_p],
    'saicv_bn_apply_generic': [c_void_p, c_int, c_void_p, c_void_p, c_int, c_ll, c_int, c_void_p],
    'saicv_bn_bwd_generic': [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_ll, c_int, c_int, c_void_p],
    'saicv_im2col_nhwc': [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    'saicv_col2im_nhwc': [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
}

_lib = None


def load():
    """Load the shared library once; raises RuntimeError when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f'{LIB_PATH} not found: build it with `python -c "import __graft_entry__ as g; g.build()"` '
            '(there is no CPU or library fallback for the hot path)')
    lib = ctypes.CDLL(LIB_PATH)
    lib.saicv_last_error.restype = ctypes.c_char_p
    lib.saicv_last_error.argtypes = []
    lib.saicv_launch_count.restype = c_ll
    lib.saicv_launch_count.argtypes = []
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = c_int
    _lib = lib
    return lib


def launch_count():
    """Kernels launched by the library so far in this process."""
    return int(load().saicv_launch_count())


def call(name, *args):
    """Call an int-returning entry point and raise on a non-zero status."""
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise RuntimeError(f'{name} failed ({rc}): {lib.saicv_last_error().decode()}')
    return rc
