"""ctypes binding of libalm_ocr.so (include/alm_ocr.h).

There is no fallback: if the shared library is missing or cannot be loaded this module raises, and
every adapter built on it fails loudly.  Build it with ``python -c "import __graft_entry__ as g; g.build()"``
or ``make`` at the repo root.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# ALM_OCR_LIB: developer knob for A/B runs of two builds of the same library on one GPU box (never a different backend)
LIB_PATH = os.environ.get('ALM_OCR_LIB') or os.path.join(_HERE, 'libalm_ocr.so')

ALM_OK = 0
MAX_CANDIDATES = 8  # ALM_MAX_CANDIDATES
MAX_BEAMS = 8  # ALM_MAX_BEAMS
MAX_CHARSETS = 65536  # ALM_MAX_CHARSETS
BOX_CROP, BOX_QUAD, BOX_CURVE = 0, 1, 2  # ALM_BOX_*: geometry of alm_mgpstr_forward_boxes
MAX_LINE_WINDOWS = 8  # ALM_MAX_LINE_WINDOWS
MODEL_OMNI_SPOT, MODEL_OMNI_KIE, MODEL_MGPSTR = 1, 2, 3
DT_F32, DT_F16, DT_BF16, DT_I64 = 0, 1, 2, 3


class TensorDesc(C.Structure):
    _fields_ = [('name', C.c_char_p), ('data', C.c_void_p), ('dtype', C.c_int), ('ndim', C.c_int),
                ('shape', C.c_int64 * 4)]


class DecodeCfg(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        'num_bins', 'pt_eos', 'poly_eos', 'rec_eos', 'pt_sos', 'poly_sos', 'rec_sos', 'recog_pad',
        'pt_seq_length', 'rec_length', 'poly_length', 'vie_categories', 'max_instances')]


class GemmOperand(C.Structure):  # alm_gemm_operand
    _fields_ = [('hi', C.c_void_p), ('lo', C.c_void_p), ('rows', C.c_int), ('K', C.c_int), ('ld', C.c_long),
                ('nb0', C.c_int), ('nb1', C.c_int), ('bs0', C.c_long), ('bs1', C.c_long)]


class GemmEpilogue(C.Structure):  # alm_gemm_epilogue
    _fields_ = [('out_f32', C.c_void_p), ('out_hi', C.c_void_p), ('out_lo', C.c_void_p), ('ldo', C.c_long),
                ('obs0', C.c_long), ('obs1', C.c_long), ('col_group', C.c_int), ('col_group_stride', C.c_long),
                ('bias', C.c_void_p), ('bias_mode', C.c_int), ('bias_bs0', C.c_long), ('resid', C.c_void_p),
                ('ldr', C.c_long), ('rbs0', C.c_long), ('rbs1', C.c_long), ('out_map', C.c_void_p),
                ('resid_map', C.c_void_p), ('act', C.c_int), ('alpha', C.c_float)]


class AlmError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f'libalm_ocr error {code}: {msg}')
        self.code = code


_lib = None

# name -> (restype, argtypes); this table is also what tests/test_abi.py checks against include/alm_ocr.h
SIGNATURES = {
    'alm_init': (C.c_int, [C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]),
    'alm_free': (None, [C.c_void_p]),
    'alm_last_error': (C.c_char_p, [C.c_void_p]),
    'alm_version': (C.c_char_p, []),
    'alm_set_option': (C.c_int, [C.c_void_p, C.c_char_p, C.c_long]),
    'alm_launch_count': (C.c_long, [C.c_void_p, C.c_int]),
    'alm_synchronize': (C.c_int, [C.c_void_p]),
    'alm_profile_read': (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_long)]),
    'alm_trace_read': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)]),
    'alm_bench_graph_floor': (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_float)]),
    'alm_bench_gemm_ex': (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.POINTER(C.c_float), C.c_void_p]),
    'alm_bench_gemm': (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float)]),
    'alm_load_weights': (C.c_int, [C.c_void_p, C.c_int, C.POINTER(TensorDesc), C.c_int]),
    'alm_share_weights': (C.c_int, [C.c_void_p, C.c_void_p]),
    'alm_stream_wait': (C.c_int, [C.c_void_p, C.c_void_p]),
    'alm_stream_release': (C.c_int, [C.c_void_p, C.c_void_p]),
    'alm_comm_unique_id': (C.c_int, [C.c_void_p]),
    'alm_comm_init': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    'alm_comm_attach': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    'alm_broadcast_weights': (C.c_int, [C.c_void_p, C.c_int]),
    'alm_gather_sequences': (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'alm_omni_encode': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]),
    'alm_omni_get_feature': (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]),
    'alm_omni_get_memory': (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]),
    'alm_omni_memory_shape': (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    'alm_omni_encode_pages': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    'alm_omni_page_shapes': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    'alm_omni_decode': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(DecodeCfg), C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p]),
    'alm_omni_decode_prompts': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(DecodeCfg), C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    # ctx, prompt, n_prompt, cfg, nx, ny, iou, cap, n_inst, pt, poly, rec, rec_prob, window, grid, saturated
    'alm_omni_decode_dense': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(DecodeCfg), C.c_int, C.c_int,
                                        C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'alm_omni_get_dense_loops': (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'alm_omni_decode_kie': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(DecodeCfg), C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'alm_omni_decode_points': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(DecodeCfg), C.c_void_p, C.c_void_p,
                                         C.c_void_p]),
    # ctx, xy, count, cap, cfg, poly, rec, rec_prob
    'alm_omni_decode_at': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(DecodeCfg), C.c_void_p,
                                     C.c_void_p, C.c_void_p]),
    'alm_omni_set_rec_candidates': (C.c_int, [C.c_void_p, C.c_int]),
    'alm_omni_get_rec_candidates': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    'alm_omni_set_rec_beams': (C.c_int, [C.c_void_p, C.c_int, C.c_float]),
    'alm_omni_get_rec_beams': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    'alm_omni_set_rec_locations': (C.c_int, [C.c_void_p, C.c_int]),
    'alm_omni_set_rec_charset': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t]),
    'alm_omni_get_rec_locations': (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    'alm_omni_decode_logits': (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    'alm_omni_vocab': (C.c_int, [C.c_void_p]),
    'alm_omni_last_timing': (C.c_int, [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    'alm_mgpstr_forward': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p]),
    'alm_mgpstr_topk': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    'alm_mgpstr_forward_boxes': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                           C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p]),
    'alm_mgpstr_forward_oriented': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                              C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_int] + [C.c_void_p] * 7),
    'alm_mgpstr_forward_lines': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                           C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p]),
    'alm_mgpstr_info': (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                  C.POINTER(C.c_int), C.c_void_p]),
    'alm_op_linear': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                C.c_int, C.c_int]),
    # ctx, A, W, M, N, K, batch, w_batch, out_f32, out_hi, out_lo, ldo, obs0, bias, bias_mode, bias_bs0, alpha, act,
    # resid, ldr, rbs0, resid_map, out_map, col_group, col_group_stride
    'alm_op_gemm': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_long, C.c_long, C.c_void_p, C.c_int, C.c_long,
                              C.c_float, C.c_int, C.c_void_p, C.c_long, C.c_long, C.c_void_p, C.c_void_p, C.c_int,
                              C.c_long]),
    'alm_op_gemm_planes': (C.c_int, [C.c_void_p, C.POINTER(GemmOperand), C.POINTER(GemmOperand),
                                     C.POINTER(GemmEpilogue)]),
    'alm_op_attention': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]),
    # ctx, qkv_hi, qkv_lo, ld, B, T, H, out_f32, out_hi, out_lo, ldo
    'alm_op_attention_ex': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_long]),
    # ctx, logits, ld, rows, n, k, ids, probs
    'alm_op_row_select': (C.c_int, [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                    C.c_void_p]),
    'alm_op_layernorm': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_long,
                                   C.c_int]),
    'alm_op_window_attention': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                          C.c_int, C.c_int, C.c_int]),
    # ctx, qkv, bias_table, out_f32, out_hi, out_lo, B, nWh, nWw, C, heads, shift
    'alm_op_window_attention_ex': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    # ctx, qkv_hi, qkv_lo, bias_table, out_f32, out_hi, out_lo, B, nWh, nWw, C, heads, shift
    'alm_op_window_attention_planes': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    # ctx, src, lds, map, nsrc, Cs, rows, gamma, beta, eps, zero_missing, add, ld_add, out_f32, ldo_f32, out_hi, out_lo,
    # ldo_bf, out2_hi, out2_lo, out2_f32
    'alm_op_gather_ln': (C.c_int, [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_int, C.c_int, C.c_long, C.c_void_p,
                                   C.c_void_p, C.c_float, C.c_int, C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_void_p,
                                   C.c_void_p, C.c_long, C.c_void_p, C.c_void_p, C.c_void_p]),
    # alm_op_gather_ln's arguments, then rows_half, gamma2, beta2, add2
    'alm_op_gather_ln_joint': (C.c_int, [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_int, C.c_int, C.c_long,
                                         C.c_void_p, C.c_void_p, C.c_float, C.c_int, C.c_void_p, C.c_long, C.c_void_p,
                                         C.c_long, C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_long, C.c_void_p, C.c_void_p, C.c_void_p]),
    'alm_op_swin_map': (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    'alm_op_patch_im2col': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                      C.c_int, C.c_void_p, C.c_void_p]),
    'alm_op_fpn_assemble': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                      C.c_int, C.c_void_p, C.c_void_p]),
    'alm_op_sine_pos': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                  C.c_void_p]),
    # ctx, s, lds, rows, n, kpm, rows_per_mask, mask_ld, out_f32, out_hi, out_lo, ldo
    'alm_op_softmax_rows': (C.c_int, [C.c_void_p, C.c_void_p, C.c_long, C.c_long, C.c_int, C.c_void_p, C.c_int, C.c_long,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_long]),
    'alm_op_cross_attention': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    'alm_op_cross_attention_ex': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                            C.c_void_p]),
    'alm_op_rec_locations': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_int, C.c_int, C.c_int, C.c_int]),
    # ctx, tokens, tstride, t, S, S_half, tokens2, tstride2, word_emb, V, pos_emb, pos_emb2, gamma, beta, x, qpos, qpos2
    'alm_op_embed_ln': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                  C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p]),
    'alm_op_self_attention_step': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                             C.c_int]),
    'alm_op_self_attention_step_anc': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                                 C.c_int, C.c_int, C.c_void_p]),
    'alm_op_gemv': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                              C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    'alm_op_head_select': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.POINTER(DecodeCfg), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'alm_op_beam_select': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.POINTER(DecodeCfg), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    # test-time image pipeline
    'alm_pre_omni_plan': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int),
                                    C.POINTER(C.c_int)]),
    'alm_pre_coeffs': (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_void_p, C.c_void_p, C.c_size_t]),
    'alm_pre_omni_pages': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                     C.c_void_p]),
    'alm_pre_mgp_crops': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    'alm_pre_quad_crops': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                     C.c_int, C.c_int, C.c_int, C.c_void_p]),
    'alm_pre_quad_plan': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p]),
    'alm_pre_curve_crops': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                      C.c_int, C.c_int, C.c_int, C.c_void_p]),
    'alm_pre_curve_plan': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                     C.c_void_p]),
    'alm_pre_line_windows': (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    'alm_pre_turned_crops': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                       C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]),
    'alm_pre_line_crops': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                     C.c_void_p, C.c_int, C.c_void_p]),
    'alm_pre_omni_tile_plan': (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                         C.c_void_p, C.c_void_p, C.c_int]),
    'alm_pre_omni_tiles': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    # ctx, rgb, heights, widths, n_pages, tile, overlap, index, count, test_min_size, test_max_size, tensors, mask
    'alm_pre_omni_tiles_at': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                        C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    # ctx, heights, widths, n_pages, tile, overlap, n_tiles, tile_page, tile_origin, n_inst, pt, poly, rec, rec_prob,
    # max_inst, rec_length, num_bins, margin, band, iou, page_count, page_offset, pts, polys, rec_out, prob_out, source, cap
    'alm_omni_merge_tiles': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                       C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_long]),
    # ctx, rgb, heights, widths, n_pages, turns, tile, overlap, first, count, test_min_size, test_max_size, tensors, mask
    'alm_pre_omni_tiles_turned': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                            C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                            C.c_void_p]),
    # alm_pre_omni_tiles_at's arguments with turns after n_pages
    'alm_pre_omni_tiles_at_turned': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                               C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                               C.c_void_p]),
    # alm_omni_merge_tiles' arguments with turns after n_pages
    'alm_omni_merge_tiles_turned': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                              C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double,
                                              C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_long]),
    # ctx, n_pages, n_inst, rec, rec_prob, max_inst, rec_length, recog_pad_index, rec_eos_index, turns_out, scores
    'alm_omni_orient_select': (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                         C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    # ctx, n_pages, count, offset, pts, polys, rec, rec_prob, rec_length, recog_pad_index, rec_eos_index, iou,
    # page_count, page_offset, pts_out, polys_out, rec_out, prob_out, source, cap
    'alm_omni_merge_turns': (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_long]),
    'alm_omni_merge_readings': (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_long]),
    # ctx, heights, widths, n_pages, turns, tile, overlap, margin, num_bins, count, offset, pts, polys, rec, rec_prob,
    # source_in, n_inst, pt, poly, whole_rec, whole_prob, cap_in, rec_length, page_count, page_offset, pts_out,
    # polys_out, rec_out, prob_out, source, cap
    # ctx, heights, widths, n_pages, turns, tile, overlap, n_tiles, tile_page, tile_origin, n_tok, tokens, tok_prob,
    # max_tok, n_inst, inst_pos, poly, max_inst, num_bins, class_base, n_classes, margin, band, iou, page_count,
    # page_offset, ent_class, ent_prob, word_offset, word_count, ent_source, cap_ent, word_rect, word_poly, word_source,
    # cap_words
    'alm_omni_merge_kie_tiles': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                           C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                           C.c_int, C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_long,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_long]),
    'alm_omni_merge_whole_page': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                            C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_long]),
    # ctx, heights, widths, n_pages, turns, tile, overlap, margin, num_bins, class_base, n_classes, count, offset,
    # ent_class, ent_prob, word_offset, word_count, ent_source, word_rect, word_poly, word_source, n_tok, tokens,
    # tok_prob, max_tok, n_inst, inst_pos, poly, max_inst, page_count, page_offset, ent_class_out, ent_prob_out,
    # word_offset_out, word_count_out, ent_source_out, cap_ent, word_rect_out, word_poly_out, word_source_out, cap_words
    'alm_omni_merge_kie_whole_page': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                                C.c_int, C.c_double, C.c_int, C.c_int, C.c_int] +
                                      [C.c_void_p] * 13 + [C.c_int] + [C.c_void_p] * 3 + [C.c_int] +
                                      [C.c_void_p] * 7 + [C.c_long] + [C.c_void_p] * 3 + [C.c_long]),
    # ctx, n_words, rec_length, polys, rec, loc, frame_index, n_frames, frames, recog_pad_index, rec_eos_index, n_chars,
    # step, centre, cov, box
    'alm_omni_char_boxes': (C.c_int, [C.c_void_p, C.c_long, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p]),
    # ctx, n_regions, n_cand, frame_index, n_frames, frames, pt, poly, rec, rec_prob, rec_length, num_bins,
    # recog_pad_index, rec_eos_index, kept, scores, pts, polys
    'alm_omni_select_regions': (C.c_int, [C.c_void_p, C.c_long, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    # ctx, n_pages, page_count, page_offset, polys, cos_tol, height_ratio, max_offset, max_overlap, max_gap, n_lines,
    # line_offset, line_first, line_words, order, line_of, rank_of, line_polys, cap
    'alm_omni_group_lines': (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_double,
                                       C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_long]),
    # host-only post-processing (no context, no GPU)
    'alm_post_last_error': (C.c_char_p, []),
    'alm_post_omni_spotting': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.c_int, C.c_char_p, C.c_long, C.c_long, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_size_t]),
    'alm_post_omni_json': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_int, C.c_char_p, C.c_long, C.c_long, C.c_char_p, C.c_void_p, C.c_size_t,
                                     C.POINTER(C.c_size_t)]),
    'alm_post_omni_kie_json': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_int, C.c_int, C.c_int, C.c_char_p, C.POINTER(C.c_char_p), C.c_int, C.c_int,
                                         C.c_long, C.c_long, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    'alm_post_mgp_fuse': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_char_p), C.c_int,
                                    C.POINTER(C.c_char_p), C.c_int, C.POINTER(C.c_char_p), C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_size_t, C.c_void_p, C.c_void_p]),
}


def load():
    """dlopen libalm_ocr.so and bind every symbol of include/alm_ocr.h."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f'{LIB_PATH} not found: build it first (make / __graft_entry__.build()); '
                          'there is no CPU or PyTorch fallback')
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class Context:
    """One alm_ctx: one GPU, one stream, not thread-safe."""

    def __init__(self, device: int = 0, stream: int | None = None):
        self.lib = load()
        h = C.c_void_p()
        rc = self.lib.alm_init(int(device), C.c_void_p(stream) if stream else None, C.byref(h))
        if rc != ALM_OK:
            raise AlmError(rc, 'alm_init failed (no sm_90a CUDA device? this library has no fallback path)')
        self.h = h
        self.device = device
        self.comm_rank, self.comm_world = 0, 1
        # ALM_OCR_OPTIONS="name=value,...": developer knob, applied to every new context (A/B runs of kernel variants
        # through the unchanged tests / bench; the options are the documented alm_set_option ones)
        for kv in filter(None, os.environ.get('ALM_OCR_OPTIONS', '').split(',')):
            k, v = kv.split('=')
            self.set_option(k.strip(), int(v))

    def check(self, rc):
        if rc != ALM_OK:
            raise AlmError(rc, self.lib.alm_last_error(self.h).decode())

    def synchronize(self):
        self.check(self.lib.alm_synchronize(self.h))

    def set_option(self, key: str, value: int):
        self.check(self.lib.alm_set_option(self.h, key.encode(), int(value)))

    def profile_read(self):
        ms, fl, n = C.c_double(), C.c_double(), C.c_long()
        self.check(self.lib.alm_profile_read(self.h, C.byref(ms), C.byref(fl), C.byref(n)))
        return ms.value, fl.value, n.value

    def trace_read(self, max_records=200000):
        import numpy as np
        buf = np.zeros((max_records, 6), dtype=np.uint64)
        n = C.c_int()
        self.check(self.lib.alm_trace_read(self.h, buf.ctypes.data, max_records, C.byref(n)))
        return buf[:n.value]

    def omni_last_timing(self):
        e, p, r = C.c_float(), C.c_float(), C.c_float()
        self.check(self.lib.alm_omni_last_timing(self.h, C.byref(e), C.byref(p), C.byref(r)))
        return {'encode_ms': e.value, 'pt_loop_ms': p.value, 'poly_rec_loops_ms': r.value}

    def bench_gemm_ex(self, M, N, K, batch=1, split_out=0, act=0, iters=10) -> float:
        ms = C.c_float()
        self.check(self.lib.alm_bench_gemm_ex(self.h, M, N, K, batch, split_out, act, iters, C.byref(ms), None))
        return ms.value

    def bench_gemm(self, M, N, K, iters=20) -> float:
        ms = C.c_float()
        self.check(self.lib.alm_bench_gemm(self.h, M, N, K, iters, C.byref(ms)))
        return ms.value

    def launch_count(self, reset=False) -> int:
        return int(self.lib.alm_launch_count(self.h, 1 if reset else 0))

    def load_state_dict(self, kind: int, state_dict):
        """state_dict: name -> torch.Tensor (any device) in the reference checkpoint layout."""
        import torch
        descs = (TensorDesc * len(state_dict))()
        keep = []
        for i, (k, v) in enumerate(state_dict.items()):
            t = v.detach().to('cpu').contiguous()
            if t.dtype == torch.float32:
                dt = DT_F32
            elif t.dtype == torch.float16:
                dt = DT_F16
            elif t.dtype == torch.bfloat16:
                dt = DT_BF16
            elif t.dtype == torch.int64:
                dt = DT_I64
            else:
                t = t.float()
                dt = DT_F32
            keep.append(t)
            assert t.dim() <= 4, k
            descs[i].name = k.encode()
            descs[i].data = t.data_ptr()
            descs[i].dtype = dt
            descs[i].ndim = t.dim()
            for j, s in enumerate(t.shape):
                descs[i].shape[j] = s
        self.check(self.lib.alm_load_weights(self.h, kind, descs, len(state_dict)))

    def load_placeholders(self, kind: int, meta):
        """Shape-only load (data == NULL) of [(name, shape, dtype_code), ...]: lays the weights out exactly like
        `load_state_dict` would; the values arrive through `broadcast_weights` (non-root ranks of a multi-GPU job)."""
        descs = (TensorDesc * len(meta))()
        for i, (k, shape, dt) in enumerate(meta):
            assert len(shape) <= 4, k
            descs[i].name = k.encode()
            descs[i].data = None
            descs[i].dtype = dt
            descs[i].ndim = len(shape)
            for j, s in enumerate(shape):
                descs[i].shape[j] = s
        self.check(self.lib.alm_load_weights(self.h, kind, descs, len(meta)))

    @staticmethod
    def state_dict_meta(state_dict):
        """[(name, shape, dtype_code)] of a reference state dict, as `load_placeholders` takes it."""
        import torch
        code = {torch.float32: DT_F32, torch.float16: DT_F16, torch.bfloat16: DT_BF16, torch.int64: DT_I64}
        return [(k, tuple(v.shape), code.get(v.dtype, DT_F32)) for k, v in state_dict.items()]

    def share_weights(self, owner: 'Context'):
        """Serve the weights resident in `owner` (same GPU) from this context too: no copy (alm_share_weights)."""
        self.check(self.lib.alm_share_weights(self.h, owner.h))
        self._weights_owner = owner  # keeps the Python object alive; the device slabs are ref-counted in the library

    def wait_stream(self, cuda_stream: int):
        """The context's stream waits for everything enqueued so far on `cuda_stream` (device inputs written there)."""
        self.check(self.lib.alm_stream_wait(self.h, C.c_void_p(cuda_stream)))

    def release_stream(self, cuda_stream: int):
        """`cuda_stream` waits for everything this context has enqueued so far (device outputs read there)."""
        self.check(self.lib.alm_stream_release(self.h, C.c_void_p(cuda_stream)))

    def wait_torch(self, *tensors):
        """Order the context's stream after torch's current stream when any argument is a CUDA tensor."""
        import torch
        for t in tensors:
            if t is not None and t.is_cuda:
                self.wait_stream(torch.cuda.current_stream(t.device).cuda_stream)
                return

    # ---- multi-GPU (alm_comm_*): one weight broadcast, one gather per batch
    def comm_unique_id(self) -> bytes:
        buf = C.create_string_buffer(128)
        rc = self.lib.alm_comm_unique_id(buf)
        if rc != ALM_OK:
            raise AlmError(rc, 'alm_comm_unique_id failed (NCCL not loadable?)')
        return buf.raw

    def comm_init(self, uid: bytes, rank: int, world: int):
        assert len(uid) == 128
        self.check(self.lib.alm_comm_init(self.h, C.create_string_buffer(uid, 128), int(rank), int(world)))
        self.comm_rank, self.comm_world = int(rank), int(world)

    def broadcast_weights(self, root: int = 0):
        self.check(self.lib.alm_broadcast_weights(self.h, int(root)))

    def gather(self, send, world: int):
        """All-gather of one equal-size buffer per rank (numpy array in, [world, ...] numpy array out)."""
        import numpy as np
        send = np.ascontiguousarray(send)
        recv = np.empty((world,) + send.shape, dtype=send.dtype)
        self.check(self.lib.alm_gather_sequences(self.h, send.ctypes.data, send.nbytes, recv.ctypes.data))
        return recv

    def close(self):
        if getattr(self, 'h', None):
            self.lib.alm_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
