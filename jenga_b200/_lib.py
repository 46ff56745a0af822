"""ctypes binding of libjenga_b200.so (the C-ABI declared in include/jenga_b200.h).

There is no CPU or PyTorch fallback: if the shared library is missing, importing this module
raises, and every compute entry point returns an error code without a CUDA device.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

LIB_PATH = Path(__file__).resolve().parent / "_C" / "libjenga_b200.so"

JENGA_BF16, JENGA_F16, JENGA_F32 = 0, 1, 2


class JengaError(RuntimeError):
    pass


class JengaAttnArgs(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("out", C.c_void_p),
        ("dtype", C.c_int32), ("batch", C.c_int32), ("heads", C.c_int32), ("head_dim", C.c_int32),
        ("q_rows", C.c_int64), ("kv_rows", C.c_int64),
        ("q_stride_b", C.c_int64), ("q_stride_s", C.c_int64), ("q_stride_h", C.c_int64),
        ("k_stride_b", C.c_int64), ("k_stride_s", C.c_int64), ("k_stride_h", C.c_int64),
        ("v_stride_b", C.c_int64), ("v_stride_s", C.c_int64), ("v_stride_h", C.c_int64),
        ("o_stride_b", C.c_int64), ("o_stride_s", C.c_int64), ("o_stride_h", C.c_int64),
        ("nq_sparse", C.c_int32), ("nq_dense", C.c_int32),
        ("mask_bits", C.c_void_p), ("mask_words", C.c_int32),
        ("sm_scale", C.c_float), ("text_amp", C.c_float), ("text_block_start", C.c_int32),
        ("kv_limit_sparse", C.c_int64), ("q_limit_sparse", C.c_int64),
        ("kv_limit_dense", C.c_int64),
        ("seqlen_dev", C.c_void_p), ("out_dtype", C.c_int32),
        ("err_flag", C.c_void_p),
        ("sp_world", C.c_int32), ("sp_rank", C.c_int32), ("sp_heads_total", C.c_int32),
        ("sp_rows", C.c_int64), ("out_peers_host", C.c_void_p),
        ("sp_head_base", C.c_int32), ("sp_head_base_valid", C.c_int32),
        ("lse_out", C.c_void_p),
        ("v_fp8", C.c_void_p), ("v_fp8_amax", C.c_void_p),
    ]


class JengaQkInt8Args(C.Structure):
    _fields_ = [
        ("q_i8", C.c_void_p), ("q_scale", C.c_void_p), ("k_i8", C.c_void_p), ("k_scale", C.c_void_p),
        ("q_rows_padded", C.c_int64), ("kv_rows_padded", C.c_int64),
    ]


class JengaQkInt8ExArgs(C.Structure):
    _fields_ = [("base", JengaQkInt8Args), ("q_lse_shift", C.c_void_p)]


class JengaAttnSched(C.Structure):
    _fields_ = [("workspace", C.c_void_p), ("workspace_bytes", C.c_int64)]


class JengaUlyssesScatterArgs(C.Structure):
    _fields_ = [
        ("x", C.c_void_p * 3), ("joint", C.c_void_p * 3),
        ("x_stride_s", C.c_int64), ("joint_stride_s", C.c_int64),
        ("world", C.c_int32), ("rank", C.c_int32), ("heads", C.c_int32), ("head_dim", C.c_int32),
        ("n_loc", C.c_int64), ("n_text", C.c_int64), ("peer_qkv_host", C.c_void_p),
        ("head_begin", C.c_int32), ("head_count", C.c_int32),
    ]


class JengaUlyssesScatterBatchArgs(C.Structure):
    _fields_ = [("base", JengaUlyssesScatterArgs), ("batch", C.c_int32),
                ("x_stride_b", C.c_int64), ("joint_stride_b", C.c_int64)]


class JengaSelectArgs(C.Structure):
    _fields_ = [
        ("q_pool", C.c_void_p), ("k_pool", C.c_void_p), ("dtype", C.c_int32),
        ("batch_heads", C.c_int32), ("head_dim", C.c_int32), ("nq", C.c_int32),
        ("nk_pool", C.c_int32), ("n_img", C.c_int32), ("nb", C.c_int32),
        ("mask_words", C.c_int32), ("top_k", C.c_int32), ("p_threshold", C.c_float),
        ("text_blocks", C.c_int32), ("first_frame_blocks", C.c_int32),
        ("nbr_bits", C.c_void_p), ("nbr_rows", C.c_int32), ("nbr_words", C.c_int32),
        ("out_bits", C.c_void_p), ("out_counts", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64),
    ]


class JengaHyPrologueArgs(C.Structure):
    _fields_ = [
        ("img_qkv", C.c_void_p), ("txt_qkv", C.c_void_p), ("dtype", C.c_int32),
        ("batch", C.c_int32), ("heads", C.c_int32), ("head_dim", C.c_int32),
        ("img_tokens", C.c_int64), ("txt_tokens", C.c_int64),
        ("img_stride_b", C.c_int64), ("img_stride_s", C.c_int64), ("img_stride_w", C.c_int64),
        ("img_stride_h", C.c_int64),
        ("txt_stride_b", C.c_int64), ("txt_stride_s", C.c_int64), ("txt_stride_w", C.c_int64),
        ("txt_stride_h", C.c_int64),
        ("w_img_q", C.c_void_p), ("w_img_k", C.c_void_p), ("w_txt_q", C.c_void_p),
        ("w_txt_k", C.c_void_p), ("eps", C.c_float),
        ("rope_cos", C.c_void_p), ("rope_sin", C.c_void_p), ("rope_index", C.c_void_p),
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p),
        ("q_pool", C.c_void_p), ("k_pool", C.c_void_p),
    ]


class JengaWanPrologueArgs(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("w", C.c_void_p), ("x_dtype", C.c_int32), ("w_dtype", C.c_int32),
        ("batch", C.c_int32), ("heads", C.c_int32), ("head_dim", C.c_int32), ("tokens", C.c_int64),
        ("stride_b", C.c_int64), ("stride_s", C.c_int64), ("eps", C.c_float),
        ("freqs", C.c_void_p), ("freq_rows", C.c_int32),
        ("grid_f", C.c_int32), ("grid_h", C.c_int32), ("grid_w", C.c_int32),
        ("freq_remap", C.c_void_p), ("out", C.c_void_p),
    ]


class JengaWanCrossArgs(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("k_img", C.c_void_p), ("v_img", C.c_void_p), ("k_txt", C.c_void_p),
        ("v_txt", C.c_void_p), ("out", C.c_void_p),
        ("dtype", C.c_int32), ("batch", C.c_int32), ("heads", C.c_int32), ("head_dim", C.c_int32),
        ("q_rows", C.c_int64), ("img_rows", C.c_int64), ("txt_rows", C.c_int64),
        ("q_stride_b", C.c_int64), ("q_stride_s", C.c_int64), ("q_stride_h", C.c_int64),
        ("ki_stride_b", C.c_int64), ("ki_stride_s", C.c_int64), ("ki_stride_h", C.c_int64),
        ("vi_stride_b", C.c_int64), ("vi_stride_s", C.c_int64), ("vi_stride_h", C.c_int64),
        ("kt_stride_b", C.c_int64), ("kt_stride_s", C.c_int64), ("kt_stride_h", C.c_int64),
        ("vt_stride_b", C.c_int64), ("vt_stride_s", C.c_int64), ("vt_stride_h", C.c_int64),
        ("o_stride_b", C.c_int64), ("o_stride_s", C.c_int64), ("o_stride_h", C.c_int64),
        ("sm_scale", C.c_float), ("err_flag", C.c_void_p),
    ]


class JengaLinearFp8Args(C.Structure):
    _fields_ = [
        ("a", C.c_void_p), ("a_stride", C.c_int64), ("a_scale", C.c_void_p), ("w", C.c_void_p),
        ("w_scale", C.c_void_p), ("w_scale_stride", C.c_int32), ("bias", C.c_void_p), ("bias_dtype", C.c_int32),
        ("out", C.c_void_p), ("out_stride", C.c_int64), ("m", C.c_int64), ("n", C.c_int32), ("k", C.c_int32),
    ]


class JengaTeaCacheArgs(C.Structure):
    _fields_ = [
        ("cur", C.c_void_p), ("prev", C.c_void_p), ("dtype", C.c_int32), ("n", C.c_int64),
        ("coeff", C.c_double * 8), ("n_coeff", C.c_int32), ("thresh", C.c_double),
        ("force", C.c_int32), ("update_prev", C.c_int32),
        ("state", C.c_void_p), ("flag", C.c_void_p), ("rel_out", C.c_void_p),
    ]


def _load() -> C.CDLL:
    if not LIB_PATH.exists():
        raise JengaError(
            f"{LIB_PATH} is missing: build it with `python -m jenga_b200.build` "
            "(or __graft_entry__.build()); jenga_b200 has no fallback path")
    lib = C.CDLL(str(LIB_PATH))
    lib.jenga_abi_version.restype = C.c_int
    lib.jenga_last_error.restype = C.c_char_p
    lib.jenga_carved_attn_fwd.argtypes = [C.POINTER(JengaAttnArgs), C.c_void_p]
    lib.jenga_carved_attn_fwd.restype = C.c_int
    lib.jenga_mask_onehot_to_bits.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                              C.c_int32, C.c_void_p]
    lib.jenga_mask_onehot_to_bits.restype = C.c_int
    lib.jenga_gather_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                      C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_void_p]
    lib.jenga_gather_rows.restype = C.c_int
    lib.jenga_gilbert_mapping_host.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                               C.c_void_p]
    lib.jenga_gilbert_mapping_host.restype = C.c_int
    lib.jenga_gilbert_block_neighbors_host.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int,
                                                       C.c_int, C.c_void_p]
    lib.jenga_gilbert_block_neighbors_host.restype = C.c_int
    lib.jenga_block_pool.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                     C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_int64,
                                     C.c_int64, C.c_int64, C.c_int32, C.c_void_p]
    lib.jenga_block_pool.restype = C.c_int
    lib.jenga_select_blocks.argtypes = [C.POINTER(JengaSelectArgs), C.c_void_p]
    lib.jenga_select_blocks.restype = C.c_int
    lib.jenga_select_blocks_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    lib.jenga_select_blocks_workspace_bytes.restype = C.c_int64
    lib.jenga_hy_prologue.argtypes = [C.POINTER(JengaHyPrologueArgs), C.c_void_p]
    lib.jenga_hy_prologue.restype = C.c_int
    lib.jenga_wan_prologue.argtypes = [C.POINTER(JengaWanPrologueArgs), C.c_void_p]
    lib.jenga_wan_prologue.restype = C.c_int
    lib.jenga_copy2d_async.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                       C.c_int32, C.c_void_p]
    lib.jenga_copy2d_async.restype = C.c_int
    lib.jenga_ulysses_scatter.argtypes = [C.POINTER(JengaUlyssesScatterArgs), C.c_void_p]
    lib.jenga_ulysses_scatter.restype = C.c_int
    lib.jenga_ulysses_scatter_ragged.argtypes = [C.POINTER(JengaUlyssesScatterArgs), C.c_void_p, C.c_void_p]
    lib.jenga_ulysses_scatter_ragged.restype = C.c_int
    lib.jenga_ulysses_scatter_batched.argtypes = [C.POINTER(JengaUlyssesScatterBatchArgs), C.c_void_p, C.c_void_p]
    lib.jenga_ulysses_scatter_batched.restype = C.c_int
    lib.jenga_block_neighbors_from_mapping_host.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int,
                                                            C.c_void_p, C.c_void_p]
    lib.jenga_block_neighbors_from_mapping_host.restype = C.c_int
    lib.jenga_gilbert_block_neighbors_csr_host.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                                           C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    lib.jenga_gilbert_block_neighbors_csr_host.restype = C.c_int
    lib.jenga_residual_apply.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]
    lib.jenga_residual_apply.restype = C.c_int
    lib.jenga_residual_store.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]
    lib.jenga_residual_store.restype = C.c_int
    lib.jenga_teacache_gate.argtypes = [C.POINTER(JengaTeaCacheArgs), C.c_void_p]
    lib.jenga_teacache_gate.restype = C.c_int
    lib.jenga_ln_modulate.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                      C.c_int64, C.c_int32, C.c_float, C.c_void_p]
    lib.jenga_ln_modulate.restype = C.c_int
    lib.jenga_gate_residual.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                        C.c_int64, C.c_int64, C.c_int32, C.c_void_p]
    lib.jenga_gate_residual.restype = C.c_int
    lib.jenga_ln_modulate_tr.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_float, C.c_void_p]
    lib.jenga_ln_modulate_tr.restype = C.c_int
    lib.jenga_gate_residual_tr.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p]
    lib.jenga_gate_residual_tr.restype = C.c_int
    lib.jenga_gelu_tanh.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p]
    lib.jenga_gelu_tanh.restype = C.c_int
    lib.jenga_wan_ln_modulate.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_int64, C.c_int64, C.c_int32, C.c_float, C.c_void_p]
    lib.jenga_wan_ln_modulate.restype = C.c_int
    lib.jenga_wan_residual_ln.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                          C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                          C.c_int64, C.c_int64, C.c_int32, C.c_float, C.c_void_p]
    lib.jenga_wan_residual_ln.restype = C.c_int
    lib.jenga_wan_gate_residual.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                            C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p]
    lib.jenga_wan_gate_residual.restype = C.c_int
    lib.jenga_prores_switch.argtypes = [C.c_void_p] * 4 + [C.c_int32] * 7 + [C.c_float, C.c_float, C.c_void_p]
    lib.jenga_prores_switch.restype = C.c_int
    lib.jenga_gilbert_mapping_device.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.jenga_gilbert_mapping_device.restype = C.c_int
    lib.jenga_block_neighbor_bits_device.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                                     C.c_int32, C.c_void_p]
    lib.jenga_block_neighbor_bits_device.restype = C.c_int
    lib.jenga_quantize_v_fp8.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_int64, C.c_int64,
                                         C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.jenga_quantize_v_fp8.restype = C.c_int
    lib.jenga_quantize_int8.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_int64, C.c_int64,
                                        C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                        C.c_void_p]
    lib.jenga_quantize_int8.restype = C.c_int
    lib.jenga_carved_attn_fwd_qk_int8.argtypes = [C.POINTER(JengaAttnArgs), C.POINTER(JengaQkInt8Args), C.c_void_p]
    lib.jenga_carved_attn_fwd_qk_int8.restype = C.c_int
    lib.jenga_carved_attn_fwd_sched.argtypes = [C.POINTER(JengaAttnArgs), C.POINTER(JengaQkInt8Args),
                                                C.POINTER(JengaAttnSched), C.c_void_p]
    lib.jenga_carved_attn_fwd_sched.restype = C.c_int
    lib.jenga_carved_attn_fwd_qk_int8_ex.argtypes = [C.POINTER(JengaAttnArgs), C.POINTER(JengaQkInt8ExArgs),
                                                     C.POINTER(JengaAttnSched), C.c_void_p]
    lib.jenga_carved_attn_fwd_qk_int8_ex.restype = C.c_int
    lib.jenga_quantize_q_int8_lse_shift.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_int64,
                                                    C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                                    C.c_void_p, C.c_void_p, C.c_void_p]
    lib.jenga_quantize_q_int8_lse_shift.restype = C.c_int
    lib.jenga_carved_attn_sched_workspace_bytes.argtypes = [C.c_int32] * 4
    lib.jenga_carved_attn_sched_workspace_bytes.restype = C.c_int64
    lib.jenga_wan_i2v_cross_attn.argtypes = [C.POINTER(JengaWanCrossArgs), C.c_void_p]
    lib.jenga_wan_i2v_cross_attn.restype = C.c_int
    lib.jenga_quantize_rows_fp8.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_int64,
                                            C.c_void_p, C.c_void_p]
    lib.jenga_quantize_rows_fp8.restype = C.c_int
    lib.jenga_ln_modulate_fp8.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                          C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_void_p]
    lib.jenga_ln_modulate_fp8.restype = C.c_int
    lib.jenga_ln_modulate_tr_fp8.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32,
                                             C.c_float, C.c_void_p]
    lib.jenga_ln_modulate_tr_fp8.restype = C.c_int
    lib.jenga_linear_fp8.argtypes = [C.POINTER(JengaLinearFp8Args), C.c_void_p]
    lib.jenga_linear_fp8.restype = C.c_int
    lib.jenga_wan_ln_modulate_fp8.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_void_p]
    lib.jenga_wan_ln_modulate_fp8.restype = C.c_int
    lib.jenga_wan_residual_ln_fp8.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                              C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                              C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_void_p]
    lib.jenga_wan_residual_ln_fp8.restype = C.c_int
    lib.jenga_gelu_tanh_fp8.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                        C.c_int32, C.c_void_p]
    lib.jenga_gelu_tanh_fp8.restype = C.c_int
    lib.jenga_gilbert_xyz2d.argtypes = [C.c_int] * 6
    lib.jenga_gilbert_xyz2d.restype = C.c_int64
    if lib.jenga_abi_version() != 3:
        raise JengaError("libjenga_b200.so ABI version mismatch")
    return lib


lib = _load()


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib.jenga_last_error().decode(errors="replace")
        raise JengaError(f"{what} failed (code {rc}): {msg}")
