"""CPU: libalm_ocr.so loads and exports every symbol include/alm_ocr.h declares (no compute calls)."""
import ctypes
import os
import re

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(REPO, 'include', 'alm_ocr.h')


@pytest.fixture(scope='module')
def built():
    import __graft_entry__ as g
    g.build()
    from advancedliteratemachinery_b200 import _lib
    return _lib


def declared_symbols():
    src = open(HEADER).read()
    return sorted(set(re.findall(r'ALM_API\s+[\w\s\*]+?\b(alm_[a-z_0-9]+)\s*\(', src)))


def test_header_declares_the_documented_surface():
    syms = declared_symbols()
    for s in ('alm_init', 'alm_free', 'alm_load_weights', 'alm_omni_encode', 'alm_omni_decode', 'alm_mgpstr_forward',
              'alm_last_error', 'alm_op_cross_attention', 'alm_op_self_attention_step', 'alm_op_gemv',
              'alm_op_head_select', 'alm_op_gather_ln', 'alm_op_swin_map', 'alm_op_patch_im2col', 'alm_op_fpn_assemble',
              'alm_op_sine_pos', 'alm_op_softmax_rows', 'alm_op_window_attention_ex', 'alm_op_gemm_planes',
              'alm_op_attention_ex', 'alm_op_row_select', 'alm_op_embed_ln', 'alm_op_gather_ln_joint',
              'alm_op_window_attention_planes'):
        assert s in syms


def test_library_exports_every_declared_symbol(built):
    lib = ctypes.CDLL(built.LIB_PATH)
    for s in declared_symbols():
        assert hasattr(lib, s), f'{s} declared in include/alm_ocr.h but not exported'


def test_python_binding_table_matches_header(built):
    assert sorted(built.SIGNATURES) == declared_symbols()


def test_version_and_no_gpu_error_path(built):
    import torch
    lib = built.load()
    assert b'sm_90a' in lib.alm_version()
    if not torch.cuda.is_available():
        h = ctypes.c_void_p()
        assert lib.alm_init(0, None, ctypes.byref(h)) < 0  # fails loudly, no CPU fallback
        with pytest.raises(built.AlmError):
            built.Context(0)


def test_struct_layouts(built):
    assert ctypes.sizeof(built.DecodeCfg) == 13 * 4
    assert ctypes.sizeof(built.TensorDesc) == 8 + 8 + 4 + 4 + 32
    assert ctypes.sizeof(built.GemmOperand) == 8 + 8 + 4 + 4 + 8 + 4 + 4 + 8 + 8
    # out_f32, out_hi, out_lo, ldo, obs0, obs1, col_group (+4 padding), col_group_stride, bias, bias_mode (+4),
    # bias_bs0, resid, ldr, rbs0, rbs1, out_map, resid_map, act, alpha
    assert ctypes.sizeof(built.GemmEpilogue) == 3 * 8 + 3 * 8 + 8 + 8 + 8 + 8 + 8 + 8 + 3 * 8 + 8 + 8 + 4 + 4


def test_product_never_imports_the_oracle():
    pkg = os.path.join(REPO, 'advancedliteratemachinery_b200')
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.h', '.cuh')):
                src = open(os.path.join(root, f)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle|oracle[./]', src, re.M), f'{f} references the oracle'
