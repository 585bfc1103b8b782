"""The C-ABI shared library loads on a CPU-only box and exports every symbol declared in
include/saicv_b200.h; the ctypes table in _lib.py lists the same set; and every compute entry is held to an
independent reference by a named test file (no compute calls here)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'saicv_b200.h')


def _declared():
    src = open(HEADER).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(saicv_[a-z0-9_]+)\s*\(', src)))


def test_library_exports_every_declared_symbol():
    from simpleaicv_pytorch_training_examples_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = _declared()
    assert len(names) >= 30
    for n in names:
        assert hasattr(lib, n), f'{n} declared in the header but not exported'
    assert lib.saicv_version() >= 100


def test_ctypes_table_matches_header():
    from simpleaicv_pytorch_training_examples_b200 import _lib
    declared = set(_declared())
    bound = set(_lib.SIGNATURES) | {'saicv_last_error', 'saicv_launch_count'}
    assert declared == bound, (declared - bound, bound - declared)


# Every compute entry of the header -> the test files that hold it to an independent reference: float64 with a derived
# allowance, an exact formula, or a committed reference fixture / the host pipeline it replaces bit for bit.
# test_ops_gpu.py (fp32 torch at 1e-2) does not count.  A new entry needs a line here, or one in QUERIES.
_GEMM, _NORM, _SYNC = 'test_gemm_conformance_gpu.py', 'test_norm_conformance_gpu.py', 'test_sync_bn_conformance_gpu.py'
_TOKEN, _DW, _OPER = 'test_token_conformance_gpu.py', 'test_dwconv_conformance_gpu.py', 'test_operand_conformance_gpu.py'
_OPTIM = 'test_optim_conformance_gpu.py'
REFERENCE_TESTS = {
    'saicv_linear_fwd': (_GEMM, _OPER), 'saicv_linear_dgrad': (_GEMM,), 'saicv_linear_wgrad': (_GEMM, _OPER),
    'saicv_conv_fprop': (_GEMM,), 'saicv_conv_dgrad': (_GEMM,), 'saicv_conv_wgrad': (_GEMM, _OPER),
    'saicv_ns_gemm': (_OPTIM,),
    'saicv_prep_conv_weight': (_OPER,), 'saicv_finish_conv_wgrad': (_OPER,), 'saicv_reduce_partials': (_OPER, _TOKEN),
    'saicv_cast_bf16': (_OPER,), 'saicv_stem_im2col': (_OPER,), 'saicv_zero_upsample2': (_OPER,),
    'saicv_add_strided2': (_OPER,), 'saicv_add_bf16': (_OPER,),
    'saicv_bn_stats': (_NORM, _SYNC), 'saicv_bn_finalize': (_NORM, _SYNC), 'saicv_bn_apply': (_NORM, _SYNC),
    'saicv_bn_bwd_reduce': (_NORM, _SYNC), 'saicv_bn_bwd_apply': (_NORM, _SYNC), 'saicv_bn_bwd_reduce2': (_NORM, _SYNC),
    'saicv_bn_bwd_apply2': (_NORM, _SYNC), 'saicv_bn_stats_fold': (_SYNC,), 'saicv_bn_finalize_folded': (_SYNC,),
    'saicv_bn_bwd_apply_sync': (_SYNC,), 'saicv_bn_bwd_apply2_sync': (_SYNC,),
    'saicv_bn_stats_generic': (_NORM, _SYNC), 'saicv_bn_apply_generic': (_NORM,), 'saicv_bn_bwd_generic': (_NORM, _SYNC),
    'saicv_bn_bwd_generic_reduce': (_SYNC,), 'saicv_bn_bwd_generic_apply': (_SYNC,),
    'saicv_maxpool3x3s2_fwd': (_NORM,), 'saicv_maxpool3x3s2_bwd': (_NORM,), 'saicv_maxpool_fwd': (_NORM,),
    'saicv_maxpool_bwd': (_NORM,), 'saicv_avgpool_fwd': (_NORM,), 'saicv_avgpool_bwd': (_NORM,),
    'saicv_avgpool_stream_fwd': (_NORM,), 'saicv_avgpool_stream_bwd': (_NORM,), 'saicv_colsum': (_NORM,),
    'saicv_layernorm_fwd': (_NORM,), 'saicv_layernorm_bwd': (_NORM,), 'saicv_postln_fwd': (_NORM,),
    'saicv_postln_bwd': (_NORM,), 'saicv_add_pos_cast': (_NORM,),
    'saicv_gelu_fwd': (_TOKEN,), 'saicv_vit_assemble_tokens': (_TOKEN,), 'saicv_vit_assemble_tokens_bwd': (_TOKEN,),
    'saicv_token_pool_fwd': (_TOKEN,), 'saicv_token_pool_bwd': (_TOKEN,), 'saicv_token_gather_fwd': (_TOKEN,),
    'saicv_token_gather_bwd': (_TOKEN,), 'saicv_window_partition': (_TOKEN,), 'saicv_window_unpartition': (_TOKEN,),
    'saicv_add_pos_embed': (_TOKEN,), 'saicv_relpos_pack_q': (_TOKEN,), 'saicv_relpos_table': (_TOKEN,),
    'saicv_relpos_gather': (_TOKEN,), 'saicv_relpos_shift': (_TOKEN,), 'saicv_relpos_dq_combine': (_TOKEN,),
    'saicv_dropout': (_TOKEN, 'test_attn_conformance_gpu.py'), 'saicv_heads_pack': (_TOKEN,),
    'saicv_heads_unpack': (_TOKEN,),
    'saicv_attn_fwd': ('test_attn_conformance_gpu.py',), 'saicv_attn_bwd': ('test_attn_conformance_gpu.py',),
    'saicv_dwconv_fwd': (_DW,), 'saicv_dwconv_dgrad_masked': (_DW,), 'saicv_dwconv_wgrad': (_DW,),
    'saicv_mul_bf16': (_DW,), 'saicv_gate_bwd': (_DW,), 'saicv_ls_residual_fwd': (_DW,), 'saicv_ls_residual_bwd': (_DW,),
    'saicv_im2col_nhwc': (_DW,), 'saicv_col2im_nhwc': (_DW,), 'saicv_swiglu_fwd': (_DW,), 'saicv_swiglu_bwd': (_DW,),
    'saicv_rope_qk_fwd': ('test_dinov3_gpu.py',), 'saicv_rope_qk_bwd': ('test_dinov3_gpu.py',),
    'saicv_multi_tensor_sgd': (_OPTIM,), 'saicv_multi_tensor_adamw': (_OPTIM,), 'saicv_multi_tensor_clip_coef': (_OPTIM,),
    'saicv_muon_prep': (_OPTIM,), 'saicv_muon_apply': (_OPTIM,),
    'saicv_detr_decode': ('test_detr_decode_gpu.py',),
    'saicv_sam_loss_sums': ('test_sam_loss_gpu.py',), 'saicv_sam_loss_bwd': ('test_sam_loss_gpu.py',),
    'saicv_semantic_softmax_fwd': ('test_semantic_softmax_gpu.py',),
    'saicv_semantic_softmax_bwd': ('test_semantic_softmax_gpu.py',),
    'saicv_semantic_accuracy': ('test_semantic_softmax_gpu.py',),
    'saicv_u8_nhwc_to_nchw_norm': ('test_input_gpu.py',), 'saicv_u8_mix_erase_norm': ('test_mixup_input_gpu.py',),
    'saicv_u8_rand_augment': ('test_randaug_input_gpu.py',), 'saicv_u8_resample': ('test_resample_input_gpu.py',),
    'saicv_u8_resize_pad': ('test_detection_input_gpu.py',),
}
# entries the listed files reach only through a class or method: (wrapper, defining module); ops.py functions that call an
# entry are found by _ops_wrappers
WRAPPERS = {
    'saicv_multi_tensor_sgd': ('FusedSGD', 'optim.py'), 'saicv_multi_tensor_adamw': ('FusedAdamW', 'optim.py'),
    'saicv_multi_tensor_clip_coef': ('clip_grad_norm', 'optim.py'),
    'saicv_muon_prep': ('FusedMuon', 'optim.py'), 'saicv_muon_apply': ('FusedMuon', 'optim.py'),
    'saicv_sam_loss_sums': ('SAMLoss', 'interactive_segmentation/losses.py'),
    'saicv_sam_loss_bwd': ('SAMLoss', 'interactive_segmentation/losses.py'),
    'saicv_u8_nhwc_to_nchw_norm': ('DeviceNormalize', 'classification/common.py'),
}
# size and plan queries: no computation to hold to a reference
QUERIES = {
    'saicv_version', 'saicv_last_error', 'saicv_launch_count', 'saicv_sm_count', 'saicv_gemm_stats_rows',
    'saicv_wgrad_splits', 'saicv_wgrad_transposed', 'saicv_sam_loss_partial_floats', 'saicv_bn_generic_partial_rows',
    'saicv_dwconv_wgrad_blocks', 'saicv_token_fill_slabs', 'saicv_opt_chunk',
}


def _ops_wrappers(cname):
    """ops.py functions whose body calls C entry `cname`."""
    src = open(os.path.join(ROOT, 'simpleaicv_pytorch_training_examples_b200', 'ops.py')).read()
    return {m.group(1) for m in re.finditer(r'^def (\w+)\(.*?(?=^def |\Z)', src, flags=re.S | re.M)
            if re.search(r"'" + cname + r"'", m.group(0))}


def test_every_compute_entry_has_a_reference_test():
    declared = set(_declared())
    assert not QUERIES & set(REFERENCE_TESTS)
    assert not (QUERIES | set(REFERENCE_TESTS)) - declared, 'table entries the header does not declare'
    missing = declared - QUERIES - set(REFERENCE_TESTS)
    assert not missing, f'compute entries without a reference test: {sorted(missing)}'
    pkg = os.path.join(ROOT, 'simpleaicv_pytorch_training_examples_b200')
    for name, files in sorted(REFERENCE_TESTS.items()):
        short = name[len('saicv_'):]
        names = [name] + [f'ops.{w}' for w in _ops_wrappers(name) | {short}] + [f'optim.{short}']
        if name in WRAPPERS:
            wrapper, module = WRAPPERS[name]
            src = open(os.path.join(pkg, module)).read()
            assert re.search(r'^\s*(def|class) ' + wrapper + r'\b', src, flags=re.M), f'{module} defines no {wrapper}'
            assert name in src or any(f'ops.{w}(' in src for w in _ops_wrappers(name)), f'{wrapper} does not reach {name}'
            names.append(wrapper)
        assert files, name
        for f in files:
            assert f != 'test_ops_gpu.py', f'{name}: test_ops_gpu.py compares with fp32 torch at 1e-2, not a reference'
            path = os.path.join(ROOT, 'tests', f)
            assert os.path.exists(path), f'{name}: {f} does not exist'
            text = open(path).read()
            assert any(re.search(re.escape(n) + r'\b', text) for n in names), f'{f} names neither {name} nor {names[1:]}'


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from simpleaicv_pytorch_training_examples_b200 import _lib
    monkeypatch.setattr(_lib, '_lib', None)
    monkeypatch.setattr(_lib, 'LIB_PATH', str(tmp_path / 'nope.so'))
    import pytest
    with pytest.raises(RuntimeError, match='no CPU or library fallback'):
        _lib.load()
