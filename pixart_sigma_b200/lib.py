"""ctypes binding of libpixart_sm100.so (the C-ABI declared in include/pixart_sm100.h).

PyTorch is used only for device memory and streams: every call passes raw `data_ptr()`s and the current
CUDA stream.  There is no fallback: if the shared library is missing or the device is not sm_90 the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PXA_LIB_PATH") or os.path.join(_HERE, "libpixart_sm100.so")   # override: experiment builds only

EPI_BIAS, EPI_BIAS_GELU, EPI_BIAS_RESIDUAL = 0, 1, 2
EPI_BIAS_GELU_AUX, EPI_MUL_DGELU = 3, 4      # MLP training fusions (include/pixart_sm100.h)
EPI_LN_BIAS, EPI_LN_BIAS_GELU = 5, 6         # fused LayerNorm-modulate consumer epilogues
LN_STAT_PARTS = 8
DTYPE_BF16, DTYPE_F32, DTYPE_F16 = 0, 1, 2    # DTYPE_F16: pxa_iddpm_step only


class PxaError(RuntimeError):
    pass


class GemmArgs(C.Structure):
    _fields_ = [("a", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p), ("out", C.c_void_p),
                ("out_aux_bf16", C.c_void_p), ("residual", C.c_void_p), ("gate", C.c_void_p),
                ("gate_batch_stride", C.c_int64), ("rows_per_batch", C.c_int32),
                ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
                ("lda", C.c_int32), ("ldw", C.c_int32), ("ldo", C.c_int32),
                ("epilogue", C.c_int32), ("out_dtype", C.c_int32), ("block_n", C.c_int32), ("max_ctas", C.c_int32),
                ("operands_mn_major", C.c_int32),
                ("k_splits", C.c_int32), ("aux_is_branch", C.c_int32),
                ("aux_scale", C.c_void_p), ("aux_scale_batch_stride", C.c_int64), ("row_stats_out", C.c_void_p),
                ("ln_stats", C.c_void_p), ("ln_u", C.c_void_p), ("ln_v", C.c_void_p), ("ln_uv_batch_stride", C.c_int64),
                ("ln_dim", C.c_int32), ("ln_eps", C.c_float), ("reverse_tiles", C.c_int32)]


class GemmTail(C.Structure):
    _fields_ = [("tail_a", C.c_void_p), ("tail_w", C.c_void_p), ("tail_k", C.c_int32), ("lda_tail", C.c_int32),
                ("ldw_tail", C.c_int32)]


class DoraNormItem(C.Structure):
    _fields_ = [("w", C.c_void_p), ("a", C.c_void_p), ("b", C.c_void_p), ("m", C.c_void_p), ("wn", C.c_void_p), ("c", C.c_void_p)]


class DoraNormArgs(C.Structure):
    _fields_ = [("items", C.POINTER(DoraNormItem)), ("n_items", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("T", C.c_int32)]


DORA_BWD_ROWS = 128


class DoraBwdArgs(C.Structure):
    _fields_ = [("g", C.c_void_p), ("y", C.c_void_p), ("bias", C.c_void_p), ("c", C.c_void_p), ("m", C.c_void_p),
                ("dz", C.c_void_p), ("dm", C.c_void_p), ("partials", C.c_void_p), ("ldg", C.c_int64), ("ldy", C.c_int64),
                ("ldz", C.c_int64), ("M", C.c_int32), ("N", C.c_int32)]


class LnPrepareArgs(C.Structure):
    _fields_ = [("x", C.c_void_p), ("a_out", C.c_void_p), ("stats_out", C.c_void_p), ("scale", C.c_void_p),
                ("mod_batch_stride", C.c_int64), ("rows_per_batch", C.c_int32), ("M", C.c_int32), ("C", C.c_int32),
                ("ldx", C.c_int32)]


class AdamWArgs(C.Structure):
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p),
                ("shadow_bf16", C.c_void_p), ("n", C.c_int64), ("step", C.c_int32), ("grad_scale", C.c_float), ("lr", C.c_double),
                ("beta1", C.c_double), ("beta2", C.c_double), ("eps", C.c_double), ("weight_decay", C.c_double)]


GRAD_CLIP_PARTS, GRAD_CLIP_MAX_BUCKETS = 1024, 128


class GradBucket(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("n", C.c_int64)]


class GradClipArgs(C.Structure):
    _fields_ = [("buckets", C.POINTER(GradBucket)), ("n_buckets", C.c_int32), ("max_norm", C.c_float), ("grad_scale", C.c_float),
                ("partials", C.c_void_p), ("total_norm", C.c_void_p)]


class CameParam(C.Structure):
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("numel", C.c_int64), ("offset", C.c_int64),
                ("bucket_numel", C.c_int64), ("sq_off", C.c_int64), ("col_off", C.c_int64), ("lead", C.c_int32), ("R", C.c_int32),
                ("C", C.c_int32), ("factored", C.c_int32), ("tile_begin", C.c_int64), ("fin_begin", C.c_int64), ("ws_off", C.c_int64)]


class CameArgs(C.Structure):
    _fields_ = [("table", C.c_void_p), ("exp_avg_sq", C.c_void_p), ("sq_row", C.c_void_p), ("res_row", C.c_void_p),
                ("sq_col", C.c_void_p), ("res_col", C.c_void_p), ("rms", C.c_void_p), ("lr", C.c_void_p), ("workspace", C.c_void_p),
                ("workspace_bytes", C.c_int64), ("n_vec", C.c_int64), ("n_row", C.c_int64), ("n_col", C.c_int64),
                ("n_entries", C.c_int32), ("step", C.c_int32), ("eps1", C.c_double), ("eps2", C.c_double),
                ("clip_threshold", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double), ("beta3", C.c_double),
                ("weight_decay", C.c_double), ("n_tiles", C.c_int64), ("n_fin", C.c_int64), ("ws_floats", C.c_int64)]


class LnModArgs(C.Structure):
    _fields_ = [("x", C.c_void_p), ("out", C.c_void_p), ("shift", C.c_void_p), ("scale", C.c_void_p),
                ("mod_batch_stride", C.c_int64), ("rows_per_batch", C.c_int32),
                ("M", C.c_int32), ("C", C.c_int32), ("ldx", C.c_int32), ("x_dtype", C.c_int32), ("eps", C.c_float),
                ("reverse_rows", C.c_int32), ("max_ctas", C.c_int32)]


class AttnArgs(C.Structure):
    _fields_ = [("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("out", C.c_void_p),
                ("kv_len", C.c_void_p), ("kv_off", C.c_void_p),
                ("q_sn", C.c_int64), ("q_sh", C.c_int64),
                ("k_sn", C.c_int64), ("k_sh", C.c_int64), ("v_sn", C.c_int64), ("v_sh", C.c_int64),
                ("kv_rows", C.c_int64),
                ("B", C.c_int32), ("H", C.c_int32), ("Nq", C.c_int32), ("Nk", C.c_int32),
                ("ldo", C.c_int32), ("scale", C.c_float), ("lse", C.c_void_p),
                ("reverse_batch", C.c_int32), ("p_precision", C.c_int32)]


class T5AttnArgs(C.Structure):
    _fields_ = [("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("out", C.c_void_p), ("bias", C.c_void_p),
                ("key_bias", C.c_void_p), ("q_sn", C.c_int64), ("q_sh", C.c_int64), ("k_sn", C.c_int64), ("k_sh", C.c_int64),
                ("v_sn", C.c_int64), ("v_sh", C.c_int64), ("ldo", C.c_int64), ("B", C.c_int32), ("H", C.c_int32), ("L", C.c_int32),
                ("scale", C.c_float), ("rel_bias", C.c_void_p)]


class KvCompressArgs(C.Structure):
    _fields_ = [("k_in", C.c_void_p), ("v_in", C.c_void_p), ("k_out", C.c_void_p), ("v_out", C.c_void_p),
                ("conv_w", C.c_void_p), ("conv_b", C.c_void_p), ("ln_w", C.c_void_p), ("ln_b", C.c_void_p),
                ("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("C", C.c_int32), ("ld_in", C.c_int32),
                ("eps", C.c_float)]


class Conv3x3Args(C.Structure):
    _fields_ = [("x", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p), ("out", C.c_void_p), ("residual", C.c_void_p),
                ("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("Cin", C.c_int32), ("Cout", C.c_int32)]


class VaeOutArgs(C.Structure):
    _fields_ = [("x", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p), ("out_u8", C.c_void_p), ("out_f32", C.c_void_p),
                ("x_sb", C.c_int64), ("x_sh", C.c_int64), ("x_sw", C.c_int64), ("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
                ("Cin", C.c_int32)]


class DpmStepArgs(C.Structure):
    _fields_ = [("model_out", C.c_void_p), ("x", C.c_void_p), ("x0_prev", C.c_void_p), ("out_batch_stride", C.c_int64),
                ("n", C.c_int32), ("hw", C.c_int32), ("out_dtype", C.c_int32),
                ("cfg_scale", C.c_float), ("sigma_s", C.c_float), ("inv_alpha_s", C.c_float),
                ("a", C.c_float), ("b", C.c_float), ("c", C.c_float)]


class SaStepArgs(C.Structure):
    _fields_ = [("model_out", C.c_void_p), ("x", C.c_void_p), ("x_pred", C.c_void_p), ("m_prev", C.c_void_p),
                ("noise_c", C.c_void_p), ("noise_p", C.c_void_p), ("out_batch_stride", C.c_int64),
                ("n", C.c_int32), ("hw", C.c_int32), ("out_dtype", C.c_int32), ("guided", C.c_int32),
                ("cfg_scale", C.c_float), ("sigma", C.c_float), ("inv_alpha", C.c_float),
                ("c_x", C.c_float), ("c_m0", C.c_float), ("c_m1", C.c_float), ("c_noise", C.c_float),
                ("p_x", C.c_float), ("p_m0", C.c_float), ("p_m1", C.c_float), ("p_noise", C.c_float)]


class IddpmStepArgs(C.Structure):
    _fields_ = [("model_out", C.c_void_p), ("img", C.c_void_p), ("noise", C.c_void_p), ("next_in", C.c_void_p),
                ("out_batch_stride", C.c_int64), ("n", C.c_int32), ("hw", C.c_int32), ("out_dtype", C.c_int32),
                ("guided", C.c_int32), ("clip", C.c_int32), ("cfg_scale", C.c_float), ("sqrt_recip_ac", C.c_float),
                ("sqrt_recipm1_ac", C.c_float), ("post_c1", C.c_float), ("post_c2", C.c_float), ("log_beta", C.c_float),
                ("post_logvar", C.c_float)]


class LcmStepArgs(C.Structure):
    _fields_ = [("model_out", C.c_void_p), ("x", C.c_void_p), ("noise", C.c_void_p), ("denoised", C.c_void_p),
                ("x_next", C.c_void_p), ("out_batch_stride", C.c_int64), ("n", C.c_int32), ("hw", C.c_int32),
                ("out_dtype", C.c_int32), ("sqrt_alpha", C.c_float), ("sqrt_beta", C.c_float), ("c_skip", C.c_float),
                ("c_out", C.c_float), ("c_prev", C.c_float), ("c_noise", C.c_float)]


LCM_MAX_ROWS, LCM_LOSS_PARTS = 1000, 512
LCM_HUBER, LCM_L2 = 0, 1


class LcmRow(C.Structure):
    _fields_ = [("sra_s", C.c_float), ("srm1_s", C.c_float), ("cskip_s", C.c_float), ("cout_s", C.c_float),
                ("sra_t", C.c_float), ("srm1_t", C.c_float), ("cskip_t", C.c_float), ("cout_t", C.c_float),
                ("sqrt_acp", C.c_double), ("sqrt_1macp", C.c_double)]


class LcmTeacherArgs(C.Structure):
    _fields_ = [("teacher_out", C.c_void_p), ("x_t", C.c_void_p), ("index", C.c_void_p), ("table", C.c_void_p),
                ("x_prev", C.c_void_p), ("out_batch_stride", C.c_int64), ("b", C.c_int32), ("hw", C.c_int32),
                ("out_dtype", C.c_int32), ("n_rows", C.c_int32), ("w", C.c_float)]


class LcmLossArgs(C.Structure):
    _fields_ = [("student_out", C.c_void_p), ("ema_out", C.c_void_p), ("x_t", C.c_void_p), ("x_prev", C.c_void_p),
                ("index", C.c_void_p), ("table", C.c_void_p), ("d_student_out", C.c_void_p), ("loss", C.c_void_p),
                ("partials", C.c_void_p), ("student_batch_stride", C.c_int64), ("ema_batch_stride", C.c_int64),
                ("b", C.c_int32), ("hw", C.c_int32), ("ema_dtype", C.c_int32), ("n_rows", C.c_int32),
                ("out_channels", C.c_int32), ("loss_type", C.c_int32), ("huber_c", C.c_float)]


class EmaBucket(C.Structure):
    _fields_ = [("master", C.c_void_p), ("src", C.c_void_p), ("shadow", C.c_void_p), ("n", C.c_int64)]


class EmaArgs(C.Structure):
    _fields_ = [("table", C.c_void_p), ("n_buckets", C.c_int32), ("max_n", C.c_int64), ("rate", C.c_double)]


DMD_PARTS = 64


class DmdLossArgs(C.Structure):
    _fields_ = [("latents", C.c_void_p), ("noisy", C.c_void_p), ("timesteps", C.c_void_p), ("alphas_cumprod", C.c_void_p),
                ("real_out", C.c_void_p), ("fake_out", C.c_void_p), ("d_gen_out", C.c_void_p), ("loss", C.c_void_p),
                ("weight", C.c_void_p), ("partials", C.c_void_p), ("real_batch_stride", C.c_int64),
                ("fake_batch_stride", C.c_int64), ("b", C.c_int32), ("hw", C.c_int32), ("n_timesteps", C.c_int32),
                ("out_channels", C.c_int32), ("real_dtype", C.c_int32), ("fake_dtype", C.c_int32), ("cfg", C.c_float),
                ("gen_sqrt_alpha", C.c_float), ("gen_sqrt_beta", C.c_float)]


class GateResidualArgs(C.Structure):
    _fields_ = [("x", C.c_void_p), ("y", C.c_void_p), ("gate", C.c_void_p), ("out", C.c_void_p), ("dgate", C.c_void_p),
                ("gate_batch_stride", C.c_int64), ("rows_per_batch", C.c_int32), ("M", C.c_int32), ("C", C.c_int32)]


class LnModBwdArgs(C.Structure):
    _fields_ = [("x", C.c_void_p), ("dxn", C.c_void_p), ("scale", C.c_void_p), ("dx", C.c_void_p), ("dshift", C.c_void_p),
                ("dscale", C.c_void_p), ("mod_batch_stride", C.c_int64), ("rows_per_batch", C.c_int32),
                ("M", C.c_int32), ("C", C.c_int32), ("eps", C.c_float), ("add_in", C.c_void_p)]


class KvCompressBwdArgs(C.Structure):
    _fields_ = [("k_in", C.c_void_p), ("v_in", C.c_void_p), ("dk_out", C.c_void_p), ("dv_out", C.c_void_p),
                ("dk_in", C.c_void_p), ("dv_in", C.c_void_p), ("conv_w", C.c_void_p), ("conv_b", C.c_void_p),
                ("ln_w", C.c_void_p), ("d_conv_w", C.c_void_p), ("d_conv_b", C.c_void_p), ("d_ln_w", C.c_void_p),
                ("d_ln_b", C.c_void_p), ("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("C", C.c_int32),
                ("ld_in", C.c_int32), ("ld_din", C.c_int32), ("eps", C.c_float)]


class AttnBwdArgs(C.Structure):
    _fields_ = [("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("o", C.c_void_p), ("d_o", C.c_void_p),
                ("lse", C.c_void_p), ("delta", C.c_void_p), ("dq", C.c_void_p), ("dk", C.c_void_p), ("dv", C.c_void_p),
                ("kv_len", C.c_void_p), ("kv_off", C.c_void_p),
                ("q_sn", C.c_int64), ("q_sh", C.c_int64), ("k_sn", C.c_int64), ("k_sh", C.c_int64),
                ("v_sn", C.c_int64), ("v_sh", C.c_int64),
                ("dq_sn", C.c_int64), ("dq_sh", C.c_int64), ("dk_sn", C.c_int64), ("dk_sh", C.c_int64),
                ("dv_sn", C.c_int64), ("dv_sh", C.c_int64),
                ("ldo", C.c_int64), ("lddo", C.c_int64), ("kv_rows", C.c_int64),
                ("B", C.c_int32), ("H", C.c_int32), ("Nq", C.c_int32), ("Nk", C.c_int32), ("scale", C.c_float)]


EXPORTS = ("pxa_transpose_bf16", "pxa_gelu_tanh_bf16", "pxa_gate_residual_fwd", "pxa_gate_residual_bwd",
           "pxa_ln_modulate_bwd", "pxa_colsum_bf16", "pxa_attn_delta_d72", "pxa_flash_attn_d72_bwd_bf16", "pxa_kv_compress_conv2_ln_bwd",
           "pxa_version", "pxa_last_error", "pxa_launch_count", "pxa_gemm_bf16", "pxa_ln_modulate",
           "pxa_flash_attn_d72_bf16", "pxa_kv_compress_conv2_ln", "pxa_conv3x3_nhwc_bf16", "pxa_dpm_solver_pp_step",
           "pxa_ln_prepare", "pxa_layernorm_affine_bf16", "pxa_groupnorm_silu_nhwc_bf16", "pxa_adamw_flat", "pxa_rmsnorm_bf16",
           "pxa_t5_attn_d64_bf16", "pxa_sa_solver_step", "pxa_iddpm_step",
           "pxa_grad_clip_flat", "pxa_came_workspace_bytes", "pxa_came_flat",
           "pxa_lcm_step", "pxa_lcm_teacher_target", "pxa_lcm_consistency_loss", "pxa_ema_flat",
           "pxa_dmd_loss", "pxa_gemm_lora_bf16", "pxa_vae_out_u8", "pxa_gemm_dora_bf16", "pxa_dora_norm", "pxa_dora_bwd")

_lib = None


def load() -> C.CDLL:
    """Load the C-ABI library (built in-tree by `pixart_sigma_b200.build`). Raises if it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise PxaError(f"{LIB_PATH} not found: run `python -m pixart_sigma_b200.build` (there is no fallback path)")
        lib = C.CDLL(LIB_PATH)
        lib.pxa_version.restype = C.c_int
        lib.pxa_last_error.restype = C.c_char_p
        lib.pxa_launch_count.restype = C.c_uint64
        for name, struct in (("pxa_gemm_bf16", GemmArgs), ("pxa_ln_modulate", LnModArgs),
                             ("pxa_flash_attn_d72_bf16", AttnArgs), ("pxa_kv_compress_conv2_ln", KvCompressArgs),
                             ("pxa_conv3x3_nhwc_bf16", Conv3x3Args), ("pxa_dpm_solver_pp_step", DpmStepArgs),
                             ("pxa_ln_prepare", LnPrepareArgs), ("pxa_adamw_flat", AdamWArgs),
                             ("pxa_t5_attn_d64_bf16", T5AttnArgs),
                             ("pxa_sa_solver_step", SaStepArgs), ("pxa_iddpm_step", IddpmStepArgs),
                             ("pxa_grad_clip_flat", GradClipArgs),
                             ("pxa_came_flat", CameArgs), ("pxa_lcm_step", LcmStepArgs),
                             ("pxa_lcm_teacher_target", LcmTeacherArgs), ("pxa_lcm_consistency_loss", LcmLossArgs),
                             ("pxa_ema_flat", EmaArgs), ("pxa_dmd_loss", DmdLossArgs), ("pxa_vae_out_u8", VaeOutArgs)):
            fn = getattr(lib, name)
            fn.restype = C.c_int
            fn.argtypes = [C.POINTER(struct), C.c_void_p]
        for name, struct in (("pxa_gate_residual_fwd", GateResidualArgs), ("pxa_gate_residual_bwd", GateResidualArgs),
                             ("pxa_ln_modulate_bwd", LnModBwdArgs), ("pxa_flash_attn_d72_bwd_bf16", AttnBwdArgs),
                             ("pxa_kv_compress_conv2_ln_bwd", KvCompressBwdArgs), ("pxa_dora_norm", DoraNormArgs),
                             ("pxa_dora_bwd", DoraBwdArgs)):
            fn = getattr(lib, name)
            fn.restype = C.c_int
            fn.argtypes = [C.POINTER(struct), C.c_void_p]
        lib.pxa_gemm_lora_bf16.restype = C.c_int
        lib.pxa_gemm_lora_bf16.argtypes = [C.POINTER(GemmArgs), C.POINTER(GemmTail), C.c_void_p]
        lib.pxa_gemm_dora_bf16.restype = C.c_int
        lib.pxa_gemm_dora_bf16.argtypes = [C.POINTER(GemmArgs), C.POINTER(GemmTail), C.c_void_p, C.c_void_p]
        lib.pxa_came_workspace_bytes.restype = C.c_int
        lib.pxa_came_workspace_bytes.argtypes = [C.POINTER(CameArgs), C.POINTER(CameParam), C.POINTER(C.c_int64)]
        lib.pxa_layernorm_affine_bf16.restype = C.c_int
        lib.pxa_layernorm_affine_bf16.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_float,
                                                  C.c_void_p]
        lib.pxa_rmsnorm_bf16.restype = C.c_int
        lib.pxa_rmsnorm_bf16.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_int64, C.c_float,
                                         C.c_void_p]
        lib.pxa_groupnorm_silu_nhwc_bf16.restype = C.c_int
        lib.pxa_groupnorm_silu_nhwc_bf16.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                                     C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_void_p]
        lib.pxa_transpose_bf16.restype = C.c_int
        lib.pxa_transpose_bf16.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_int64, C.c_void_p]
        lib.pxa_gelu_tanh_bf16.restype = C.c_int
        lib.pxa_gelu_tanh_bf16.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        lib.pxa_colsum_bf16.restype = C.c_int
        lib.pxa_colsum_bf16.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_void_p]
        lib.pxa_attn_delta_d72.restype = C.c_int
        lib.pxa_attn_delta_d72.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64,
                                           C.c_int64, C.c_void_p]
        _lib = lib
    return _lib


def launch_count() -> int:
    return int(load().pxa_launch_count())


def _check(rc: int, what: str) -> None:
    if rc != 0:
        raise PxaError(f"{what} failed ({rc}): {load().pxa_last_error().decode()}")


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _dt(dtype: torch.dtype) -> int:
    if dtype == torch.bfloat16:
        return DTYPE_BF16
    if dtype == torch.float32:
        return DTYPE_F32
    raise PxaError(f"unsupported dtype {dtype}")


def gemm(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor, *,
         epilogue: int = EPI_BIAS, residual: Optional[torch.Tensor] = None, gate: Optional[torch.Tensor] = None,
         gate_batch_stride: int = 0, rows_per_batch: int = 0, out_aux: Optional[torch.Tensor] = None,
         block_n: int = 0, max_ctas: int = 0, aux_is_branch: bool = False, aux_scale: Optional[torch.Tensor] = None, aux_scale_batch_stride: int = 0,
         row_stats_out: Optional[torch.Tensor] = None, ln_stats: Optional[torch.Tensor] = None,
         ln_u: Optional[torch.Tensor] = None, ln_v: Optional[torch.Tensor] = None, ln_uv_batch_stride: int = 0,
         ln_dim: int = 0, ln_eps: float = 1e-6, reverse_tiles: bool = False, tail_a: Optional[torch.Tensor] = None,
         tail_w: Optional[torch.Tensor] = None, col_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = epilogue(a @ w.T + bias). a (M,K) bf16, w (N,K) bf16 (nn.Linear layout), both K-contiguous.

    K-tail (pxa_gemm_lora_bf16): with tail_a (M, T) and tail_w (N, T), bf16 K-contiguous, T a multiple of 8, the epilogue is
    applied to a @ w.T + tail_a @ tail_w.T -- a LoRA up-projection u (s B)^T added before bias / GELU / gated residual.

    Fused LayerNorm-modulate (include/pixart_sm100.h, PXA_EPI_LN_BIAS): the fp32 residual epilogue can emit the scaled bf16
    copy `out_aux = out * aux_scale[b]` and the per-row partial sums `row_stats_out` (M, 8, 2); the EPI_LN_* epilogues
    consume them (`ln_stats`) together with the per-sample vectors `ln_u`, `ln_v` (fp32 views, row b at b * stride).

    Column scale (pxa_gemm_dora_bf16, a DoRA projection): with col_scale (N,) fp32 the accumulator column n is multiplied by
    col_scale[n] before the epilogue: out = epilogue(col_scale * (a @ w.T [+ tail]) + bias)."""
    assert a.is_cuda and a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16
    assert a.dim() == 2 and w.dim() == 2 and a.stride(1) == 1 and w.stride(1) == 1 and out.dim() == 2 and out.stride(1) == 1
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K and out.shape == (M, N)
    if bias is not None:
        assert bias.dtype == torch.bfloat16 and bias.is_contiguous() and bias.numel() == N
    if residual is not None:
        assert residual.dtype == out.dtype and residual.shape == out.shape and residual.stride() == out.stride()
    if gate is not None:
        assert gate.dtype == torch.float32
    if out_aux is not None:
        assert out_aux.dtype == torch.bfloat16 and out_aux.shape == out.shape and out_aux.stride() == out.stride()
    for tns in (aux_scale, ln_u, ln_v):
        assert tns is None or (tns.dtype == torch.float32 and tns.is_cuda)
    for tns in (row_stats_out, ln_stats):
        assert tns is None or (tns.dtype == torch.float32 and tns.is_contiguous() and tns.numel() == M * LN_STAT_PARTS * 2)
    args = GemmArgs(a=_ptr(a), w=_ptr(w), bias=_ptr(bias), out=_ptr(out), out_aux_bf16=_ptr(out_aux),
                    residual=_ptr(residual), gate=_ptr(gate), gate_batch_stride=gate_batch_stride,
                    rows_per_batch=rows_per_batch or M, M=M, N=N, K=K, lda=a.stride(0), ldw=w.stride(0),
                    ldo=out.stride(0), epilogue=epilogue, out_dtype=_dt(out.dtype), block_n=block_n, max_ctas=max_ctas,
                    operands_mn_major=0, k_splits=0,
                    aux_is_branch=int(aux_is_branch), aux_scale=_ptr(aux_scale), aux_scale_batch_stride=aux_scale_batch_stride,
                    row_stats_out=_ptr(row_stats_out), ln_stats=_ptr(ln_stats), ln_u=_ptr(ln_u), ln_v=_ptr(ln_v),
                    ln_uv_batch_stride=ln_uv_batch_stride, ln_dim=ln_dim, ln_eps=ln_eps, reverse_tiles=int(reverse_tiles))
    if col_scale is not None:
        assert col_scale.dtype == torch.float32 and col_scale.is_cuda and col_scale.is_contiguous() and col_scale.numel() == N
    if tail_a is None and tail_w is None:
        if col_scale is not None:
            _check(load().pxa_gemm_dora_bf16(C.byref(args), None, _ptr(col_scale), _stream()), "pxa_gemm_dora_bf16")
        else:
            _check(load().pxa_gemm_bf16(C.byref(args), _stream()), "pxa_gemm_bf16")
        return out
    assert tail_a is not None and tail_w is not None and tail_a.dtype == tail_w.dtype == torch.bfloat16
    assert tail_a.dim() == 2 and tail_w.dim() == 2 and tail_a.stride(1) == 1 and tail_w.stride(1) == 1
    T = tail_a.shape[1]
    assert tail_a.shape[0] == M and tail_w.shape == (N, T)
    tail = GemmTail(tail_a=_ptr(tail_a), tail_w=_ptr(tail_w), tail_k=T, lda_tail=tail_a.stride(0), ldw_tail=tail_w.stride(0))
    if col_scale is not None:
        _check(load().pxa_gemm_dora_bf16(C.byref(args), C.byref(tail), _ptr(col_scale), _stream()), "pxa_gemm_dora_bf16")
    else:
        _check(load().pxa_gemm_lora_bf16(C.byref(args), C.byref(tail), _stream()), "pxa_gemm_lora_bf16")
    return out


def dora_norm(items, *, N: int, K: int, T: int) -> None:
    """pxa_dora_norm over same-shaped projections.  items: (w, a, b, m, wn, c) per projection -- w bf16 [N, K], a bf16 [T, K],
    b bf16 [N, T] (all contiguous), m fp32 [N] or None, wn / c fp32 [N] outputs or None.  wn = ||w + b a||_2 per row, c = m / wn."""
    arr = (DoraNormItem * max(len(items), 1))()
    for i, (w, a, b, m, wn, c) in enumerate(items):
        assert w.dtype == a.dtype == b.dtype == torch.bfloat16 and w.is_cuda
        assert w.shape == (N, K) and a.shape == (T, K) and b.shape == (N, T)
        assert w.is_contiguous() and a.is_contiguous() and b.is_contiguous()
        for v in (m, wn, c):
            assert v is None or (v.dtype == torch.float32 and v.is_contiguous() and v.numel() == N)
        arr[i] = DoraNormItem(w=_ptr(w), a=_ptr(a), b=_ptr(b), m=_ptr(m), wn=_ptr(wn), c=_ptr(c))
    args = DoraNormArgs(items=arr, n_items=len(items), N=N, K=K, T=T)
    _check(load().pxa_dora_norm(C.byref(args), _stream()), "pxa_dora_norm")


def dora_bwd(g: torch.Tensor, y: torch.Tensor, bias: Optional[torch.Tensor], c: torch.Tensor, m: torch.Tensor,
             dz: torch.Tensor, dm: torch.Tensor) -> torch.Tensor:
    """pxa_dora_bwd: dz = bf16(c * g) (dz may be g) and dm += sum_rows g * (y - bias) / m.  g, y, dz bf16 [M, N] (row stride a
    multiple of 8), bias bf16 [N] or None, c / m / dm fp32 [N].  Returns dz."""
    M, N = g.shape
    assert g.dtype == y.dtype == dz.dtype == torch.bfloat16 and y.shape == dz.shape == (M, N)
    assert g.stride(1) == y.stride(1) == dz.stride(1) == 1
    for v in (c, m, dm):
        assert v.dtype == torch.float32 and v.is_contiguous() and v.numel() == N
    if bias is not None:
        assert bias.dtype == torch.bfloat16 and bias.is_contiguous() and bias.numel() == N
    partials = torch.empty(((M + DORA_BWD_ROWS - 1) // DORA_BWD_ROWS, N), dtype=torch.float32, device=g.device)
    args = DoraBwdArgs(g=_ptr(g), y=_ptr(y), bias=_ptr(bias), c=_ptr(c), m=_ptr(m), dz=_ptr(dz), dm=_ptr(dm),
                       partials=_ptr(partials), ldg=g.stride(0), ldy=y.stride(0), ldz=dz.stride(0), M=M, N=N)
    _check(load().pxa_dora_bwd(C.byref(args), _stream()), "pxa_dora_bwd")
    return dz


def ln_prepare(x: torch.Tensor, mult: torch.Tensor, a_out: torch.Tensor, stats_out: torch.Tensor, *, mod_batch_stride: int,
               rows_per_batch: int) -> None:
    """First link of the fused LayerNorm-modulate chain: a_out = bf16(x * mult[b]) with mult = 1 + scale (the multiplier
    `gemm(aux_scale=...)` takes), stats_out (M, 8, 2) = partial (sum, sum of squares) of each row of x (part 0; the rest
    zero).  x (M, C) fp32, mult an fp32 view (row b at b*stride)."""
    scale = mult
    assert x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1 and scale.dtype == torch.float32
    M, Cc = x.shape
    assert a_out.dtype == torch.bfloat16 and a_out.is_contiguous() and a_out.shape == (M, Cc)
    assert stats_out.dtype == torch.float32 and stats_out.is_contiguous() and stats_out.numel() == M * LN_STAT_PARTS * 2
    args = LnPrepareArgs(x=_ptr(x), a_out=_ptr(a_out), stats_out=_ptr(stats_out), scale=_ptr(scale),
                         mod_batch_stride=mod_batch_stride, rows_per_batch=rows_per_batch, M=M, C=Cc, ldx=x.stride(0))
    _check(load().pxa_ln_prepare(C.byref(args), _stream()), "pxa_ln_prepare")


def ln_modulate(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor, out: torch.Tensor, *,
                mod_batch_stride: int, rows_per_batch: int, eps: float = 1e-6, reverse_rows: bool = False,
                max_ctas: int = 0) -> torch.Tensor:
    """out = LN(x) * (1 + scale[b]) + shift[b]; x (M,C) fp32/bf16, shift/scale fp32 views (row b at b*stride)."""
    assert x.dim() == 2 and x.stride(1) == 1 and out.is_contiguous() and out.dtype == torch.bfloat16
    assert shift.dtype == torch.float32 and scale.dtype == torch.float32
    M, Cc = x.shape
    args = LnModArgs(x=_ptr(x), out=_ptr(out), shift=_ptr(shift), scale=_ptr(scale), mod_batch_stride=mod_batch_stride,
                     rows_per_batch=rows_per_batch, M=M, C=Cc, ldx=x.stride(0), x_dtype=_dt(x.dtype), eps=eps,
                     reverse_rows=int(reverse_rows), max_ctas=max_ctas)
    _check(load().pxa_ln_modulate(C.byref(args), _stream()), "pxa_ln_modulate")
    return out


def layernorm_affine_(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """In-place LayerNorm with affine parameters on the rows of a bf16 (M, 1152) view with unit column stride (qk_norm)."""
    assert x.dtype == weight.dtype == bias.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1
    assert weight.is_contiguous() and bias.is_contiguous() and weight.numel() == bias.numel() == x.shape[1]
    _check(load().pxa_layernorm_affine_bf16(_ptr(x), _ptr(weight), _ptr(bias), x.shape[0], x.shape[1], x.stride(0), eps,
                                            _stream()), "pxa_layernorm_affine_bf16")
    return x


def rmsnorm(x: torch.Tensor, weight: torch.Tensor, out: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    """T5LayerNorm: out (M, C) bf16 = x * rsqrt(mean(x^2) + eps) * weight on the rows of the fp32 stream x (M, C)."""
    assert x.is_cuda and x.dtype == torch.float32 and out.dtype == weight.dtype == torch.bfloat16
    assert x.dim() == 2 and out.shape == x.shape and x.stride(1) == 1 and out.stride(1) == 1
    assert weight.is_contiguous() and weight.numel() == x.shape[1]
    _check(load().pxa_rmsnorm_bf16(_ptr(x), _ptr(weight), _ptr(out), x.shape[0], x.shape[1], x.stride(0), out.stride(0), eps,
                                   _stream()), "pxa_rmsnorm_bf16")
    return out


T5_ATTN_MAX_KEYS = 384


def t5_attn(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, bias: Optional[torch.Tensor],
            key_bias: Optional[torch.Tensor] = None, *, B: int, H: int, L: int, scale: float = 1.0,
            rel_bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """T5 self-attention, head_dim 64, L <= 384: out (B*L, H*64) = softmax(q k^T * scale + bias[h] + key_bias[b]) v.
    q / k / v: bf16 (B*L, H*64) views with unit column stride (e.g. column slices of a fused qkv GEMM output);
    bias fp32 (H, L, L), or rel_bias fp32 (H, 2L-1) with bias[h, i, j] = rel_bias[h, j - i + L - 1]; key_bias fp32 (B, L) or None."""
    for t in (q, k, v, out):
        assert t.is_cuda and t.dtype == torch.bfloat16 and t.dim() == 2 and t.stride(1) == 1 and t.shape == (B * L, H * 64)
    assert (bias is None) != (rel_bias is None), "exactly one of bias / rel_bias"
    assert bias is None or (bias.dtype == torch.float32 and bias.is_contiguous() and bias.shape == (H, L, L))
    assert rel_bias is None or (rel_bias.dtype == torch.float32 and rel_bias.is_contiguous() and rel_bias.shape == (H, 2 * L - 1))
    assert key_bias is None or (key_bias.dtype == torch.float32 and key_bias.is_contiguous() and key_bias.shape == (B, L))
    args = T5AttnArgs(q=_ptr(q), k=_ptr(k), v=_ptr(v), out=_ptr(out), bias=_ptr(bias), key_bias=_ptr(key_bias),
                      q_sn=q.stride(0), q_sh=64, k_sn=k.stride(0), k_sh=64, v_sn=v.stride(0), v_sh=64, ldo=out.stride(0),
                      B=B, H=H, L=L, scale=scale, rel_bias=_ptr(rel_bias))
    _check(load().pxa_t5_attn_d64_bf16(C.byref(args), _stream()), "pxa_t5_attn_d64_bf16")
    return out


def flash_attn(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, *, B: int, H: int, Nq: int,
               Nk: int, kv_rows: int, kv_len: Optional[torch.Tensor] = None, kv_off: Optional[torch.Tensor] = None,
               q_strides=None, k_strides=None, v_strides=None, scale: Optional[float] = None,
               lse: Optional[torch.Tensor] = None, reverse_batch: bool = False, fp32_p: bool = False) -> torch.Tensor:
    """Head-dim-72 attention. q/k/v are bf16 *views*; strides are (row, head) in elements, e.g. slices of the
    (rows, 3, H, 72) qkv GEMM output. out is (B*Nq, H*72) bf16.  fp32_p: `fp32_attention` grade P V (P as bf16 hi + lo)."""
    assert q.dtype == k.dtype == v.dtype == out.dtype == torch.bfloat16
    for tns in (kv_len, kv_off):
        if tns is not None:
            assert tns.dtype == torch.int32 and tns.is_cuda and tns.numel() == B
    args = AttnArgs(q=_ptr(q), k=_ptr(k), v=_ptr(v), out=_ptr(out), kv_len=_ptr(kv_len), kv_off=_ptr(kv_off),
                    q_sn=q_strides[0], q_sh=q_strides[1], k_sn=k_strides[0], k_sh=k_strides[1],
                    v_sn=v_strides[0], v_sh=v_strides[1], kv_rows=kv_rows, B=B, H=H, Nq=Nq, Nk=Nk,
                    ldo=out.stride(0), scale=scale if scale is not None else 72 ** -0.5,
                    lse=_ptr(lse), reverse_batch=int(reverse_batch), p_precision=int(bool(fp32_p)))
    if lse is not None:
        assert lse.dtype == torch.float32 and lse.is_contiguous() and lse.numel() == B * H * Nq
    _check(load().pxa_flash_attn_d72_bf16(C.byref(args), _stream()), "pxa_flash_attn_d72_bf16")
    return out


def kv_compress(k_in: torch.Tensor, v_in: torch.Tensor, k_out: torch.Tensor, v_out: torch.Tensor, conv_w, conv_b,
                ln_w, ln_b, *, B: int, H: int, W: int, ld_in: int, eps: float = 1e-5) -> None:
    args = KvCompressArgs(k_in=_ptr(k_in), v_in=_ptr(v_in), k_out=_ptr(k_out), v_out=_ptr(v_out), conv_w=_ptr(conv_w),
                          conv_b=_ptr(conv_b), ln_w=_ptr(ln_w), ln_b=_ptr(ln_b), B=B, H=H, W=W, C=k_out.shape[-1],
                          ld_in=ld_in, eps=eps)
    _check(load().pxa_kv_compress_conv2_ln(C.byref(args), _stream()), "pxa_kv_compress_conv2_ln")


def conv3x3_nhwc(x: torch.Tensor, w_packed: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor,
                 residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """3x3 / stride 1 / pad 1 convolution on NHWC bf16 tensors. x (B,H,W,Cin), w_packed (Cout,3,3,Cin), out (B,H,W,Cout)."""
    assert x.dtype == w_packed.dtype == out.dtype == torch.bfloat16 and x.is_contiguous() and w_packed.is_contiguous()
    assert out.is_contiguous() and (residual is None or (residual.is_contiguous() and residual.shape == out.shape))
    B, H, W, Cin = x.shape
    Cout = w_packed.shape[0]
    assert w_packed.shape == (Cout, 3, 3, Cin) and out.shape == (B, H, W, Cout)
    args = Conv3x3Args(x=_ptr(x), w=_ptr(w_packed), bias=_ptr(bias), out=_ptr(out), residual=_ptr(residual), B=B, H=H, W=W,
                       Cin=Cin, Cout=Cout)
    _check(load().pxa_conv3x3_nhwc_bf16(C.byref(args), _stream()), "pxa_conv3x3_nhwc_bf16")
    return out


def vae_out_u8(x: torch.Tensor, w_packed: torch.Tensor, bias: torch.Tensor, out_u8: torch.Tensor,
               out_f32: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The VAE decoder's conv_out (3x3, pad 1, Cin -> 3) and save_image's uint8 conversion in one pass (pxa_vae_out_u8).
    x: bf16 (B, H, W, Cin) with unit channel stride and the other strides multiples of 8 (a channels_last tensor or a padded
    view); w_packed: bf16 (3, 3, 3, Cin) contiguous; bias: fp32 (3,); out_u8: uint8 (B, H, W, 3) contiguous; out_f32: the fp32
    convolution output (B, H, W, 3) contiguous, or None."""
    if not (x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 4 and x.stride(3) == 1):
        raise PxaError("vae_out_u8: x must be a bf16 CUDA tensor (B, H, W, Cin) with unit channel stride")
    B, H, W, Cin = x.shape
    if not (w_packed.dtype == torch.bfloat16 and w_packed.is_contiguous() and tuple(w_packed.shape) == (3, 3, 3, Cin)):
        raise PxaError(f"vae_out_u8: w_packed must be contiguous bf16 (3, 3, 3, {Cin})")
    if not (bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == 3):
        raise PxaError("vae_out_u8: bias must be 3 contiguous fp32 values")
    if not (out_u8.dtype == torch.uint8 and out_u8.is_contiguous() and tuple(out_u8.shape) == (B, H, W, 3)):
        raise PxaError(f"vae_out_u8: out_u8 must be contiguous uint8 ({B}, {H}, {W}, 3)")
    if out_f32 is not None and not (out_f32.dtype == torch.float32 and out_f32.is_contiguous() and tuple(out_f32.shape) == (B, H, W, 3)):
        raise PxaError(f"vae_out_u8: out_f32 must be contiguous fp32 ({B}, {H}, {W}, 3)")
    if not all(t.device == x.device for t in (w_packed, bias, out_u8) + ((out_f32,) if out_f32 is not None else ())):
        raise PxaError("vae_out_u8: all tensors must be on the same CUDA device")
    args = VaeOutArgs(x=_ptr(x), w=_ptr(w_packed), bias=_ptr(bias), out_u8=_ptr(out_u8), out_f32=_ptr(out_f32), x_sb=x.stride(0),
                      x_sh=x.stride(1), x_sw=x.stride(2), B=B, H=H, W=W, Cin=Cin)
    _check(load().pxa_vae_out_u8(C.byref(args), _stream()), "pxa_vae_out_u8")
    return out_u8


def adamw_flat(param: torch.Tensor, grad: torch.Tensor, exp_avg: torch.Tensor, exp_avg_sq: torch.Tensor, *, step: int, lr: float,
               betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 1e-2, grad_scale: float = 1.0,
               shadow: Optional[torch.Tensor] = None) -> None:
    """torch.optim.AdamW's update on flat fp32 tensors of equal length (a multiple of 4), in place; `shadow` (bf16, same
    length) receives the bf16 copy of the new parameters."""
    for t in (param, grad, exp_avg, exp_avg_sq):
        assert t.dtype == torch.float32 and t.is_cuda and t.is_contiguous() and t.numel() == param.numel()
    assert shadow is None or (shadow.dtype == torch.bfloat16 and shadow.is_contiguous() and shadow.numel() == param.numel())
    args = AdamWArgs(param=_ptr(param), grad=_ptr(grad), exp_avg=_ptr(exp_avg), exp_avg_sq=_ptr(exp_avg_sq), shadow_bf16=_ptr(shadow),
                     n=param.numel(), step=step, lr=lr, beta1=betas[0], beta2=betas[1], eps=eps, weight_decay=weight_decay,
                     grad_scale=grad_scale)
    _check(load().pxa_adamw_flat(C.byref(args), _stream()), "pxa_adamw_flat")


def grad_clip_flat(grads, partials: torch.Tensor, total_norm: torch.Tensor, *, max_norm: float, grad_scale: float = 1.0,
                   lengths=None) -> torch.Tensor:
    """torch.nn.utils.clip_grad_norm_ over flat fp32 gradient buffers, in place (include/pixart_sm100.h: pxa_grad_clip_flat):
    g *= grad_scale, total = ||g||, g *= min(max_norm / (total + 1e-6), 1).  `lengths[k]`: elements of grads[k] that belong to
    a parameter (default: all).  partials: fp32 [GRAD_CLIP_PARTS] workspace; total_norm (fp32, 1 element) receives the norm on
    the device."""
    grads = list(grads)
    lengths = [g.numel() for g in grads] if lengths is None else list(lengths)
    for g, n in zip(grads, lengths):
        if not (g.is_cuda and g.dtype == torch.float32 and g.is_contiguous() and 0 < n <= g.numel()):
            raise PxaError("grad_clip_flat: gradients must be contiguous fp32 CUDA tensors")
    for t in (partials, total_norm):
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
            raise PxaError("grad_clip_flat: partials / total_norm must be contiguous fp32 CUDA tensors")
    if partials.numel() < GRAD_CLIP_PARTS or total_norm.numel() != 1:
        raise PxaError(f"grad_clip_flat: partials needs {GRAD_CLIP_PARTS} elements, total_norm 1")
    arr = (GradBucket * max(len(grads), 1))(*[GradBucket(ptr=g.data_ptr(), n=n) for g, n in zip(grads, lengths)])
    args = GradClipArgs(buckets=arr, n_buckets=len(grads), max_norm=max_norm, grad_scale=grad_scale, partials=_ptr(partials),
                        total_norm=_ptr(total_norm))
    _check(load().pxa_grad_clip_flat(C.byref(args), _stream()), "pxa_grad_clip_flat")
    return total_norm


def came_plan(args: CameArgs, table) -> int:
    """Validate and plan the host parameter table (a ctypes array of CameParam) in place; fills args.n_tiles / n_fin /
    ws_floats and returns the workspace size in bytes (include/pixart_sm100.h: pxa_came_workspace_bytes)."""
    nbytes = C.c_int64(0)
    args.n_entries = len(table)
    _check(load().pxa_came_workspace_bytes(C.byref(args), table, C.byref(nbytes)), "pxa_came_workspace_bytes")
    return int(nbytes.value)


def came_flat(args: CameArgs) -> None:
    """One CAME step over every parameter of a planned table (include/pixart_sm100.h: pxa_came_flat); `args` holds raw
    device pointers, so the caller keeps the tensors behind them alive."""
    _check(load().pxa_came_flat(C.byref(args), _stream()), "pxa_came_flat")


def groupnorm_silu_nhwc(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, out: torch.Tensor, *, groups: int = 32,
                        eps: float = 1e-6, silu: bool = True, stats_ws: Optional[torch.Tensor] = None) -> torch.Tensor:
    """GroupNorm (+ SiLU) on an NHWC bf16 image x (B, H, W, C) -> out (same shape); statistics in fp32."""
    assert x.dtype == out.dtype == gamma.dtype == beta.dtype == torch.bfloat16 and x.is_contiguous() and out.is_contiguous()
    B, H, W, Cc = x.shape
    assert out.shape == x.shape and gamma.numel() == beta.numel() == Cc and gamma.is_contiguous() and beta.is_contiguous()
    if stats_ws is None:
        stats_ws = torch.empty(B * groups * 2, dtype=torch.float32, device=x.device)
    assert stats_ws.dtype == torch.float32 and stats_ws.numel() >= B * groups * 2
    _check(load().pxa_groupnorm_silu_nhwc_bf16(_ptr(x), _ptr(out), _ptr(gamma), _ptr(beta), _ptr(stats_ws), B, H * W, Cc, groups,
                                               eps, int(silu), _stream()), "pxa_groupnorm_silu_nhwc_bf16")
    return out


def dpm_solver_pp_step(model_out: torch.Tensor, x: torch.Tensor, x0_prev: torch.Tensor, *, cfg_scale: float, sigma_s: float,
                       alpha_s: float, a: float, b: float, c: float) -> torch.Tensor:
    """One DPM-Solver++ (2M) update, in place on x and x0_prev (include/pixart_sm100.h: pxa_dpm_solver_pp_step).
    model_out: denoiser output of the CFG batch [uncond; cond], (2n, C>=4, h, w) fp32 or bf16 -- a channel-sliced view of
    the 8-channel learn-sigma output is fine; x, x0_prev: fp32 (n, 4, h, w) contiguous."""
    assert model_out.is_cuda and x.is_cuda and x0_prev.is_cuda and x.dtype == x0_prev.dtype == torch.float32
    assert x.is_contiguous() and x0_prev.is_contiguous() and x.shape == x0_prev.shape and x.dim() == 4 and x.shape[1] == 4
    n, _, h, w = x.shape
    assert model_out.shape[0] == 2 * n and model_out.shape[1] >= 4 and model_out.shape[2:] == (h, w)
    assert model_out.stride(3) == 1 and model_out.stride(2) == w and model_out.stride(1) == h * w, "model_out: (.., h, w) planes must be dense"
    args = DpmStepArgs(model_out=_ptr(model_out), x=_ptr(x), x0_prev=_ptr(x0_prev), out_batch_stride=model_out.stride(0),
                       n=n, hw=h * w, out_dtype=_dt(model_out.dtype), cfg_scale=cfg_scale, sigma_s=sigma_s,
                       inv_alpha_s=1.0 / alpha_s, a=a, b=b, c=c)
    _check(load().pxa_dpm_solver_pp_step(C.byref(args), _stream()), "pxa_dpm_solver_pp_step")
    return x


def sa_solver_step(model_out: torch.Tensor, x: torch.Tensor, x_pred: torch.Tensor, m_prev: torch.Tensor,
                   noise_c: Optional[torch.Tensor], noise_p: Optional[torch.Tensor], *, guided: bool, cfg_scale: float,
                   sigma: float, alpha: float, c_x: float, c_m0: float, c_m1: float, c_noise: float, p_x: float,
                   p_m0: float, p_m1: float, p_noise: float) -> torch.Tensor:
    """One SA-Solver evaluation step (corrector to x_i, predictor to x~_{i+1}), in place on x, x_pred and m_prev
    (include/pixart_sm100.h: pxa_sa_solver_step); returns x_pred.  model_out: denoiser output at x_pred, (2n, C>=4, h, w)
    [uncond; cond] when guided else (n, C>=4, h, w), fp32 or bf16 -- a channel-sliced view of the 8-channel learn-sigma
    output is fine; x, x_pred, m_prev and the noise tensors: fp32 (n, 4, h, w) contiguous.  A noise tensor may be None
    when its coefficient is 0."""
    state = [x, x_pred, m_prev] + [t for t in (noise_c, noise_p) if t is not None]
    assert model_out.is_cuda and all(t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() for t in state)
    assert x.dim() == 4 and x.shape[1] == 4 and all(t.shape == x.shape for t in state)
    assert (noise_c is not None or c_noise == 0.0) and (noise_p is not None or p_noise == 0.0)
    n, _, h, w = x.shape
    assert model_out.shape[0] == (2 * n if guided else n) and model_out.shape[1] >= 4 and model_out.shape[2:] == (h, w)
    assert model_out.stride(3) == 1 and model_out.stride(2) == w and model_out.stride(1) == h * w, "model_out: (.., h, w) planes must be dense"
    args = SaStepArgs(model_out=_ptr(model_out), x=_ptr(x), x_pred=_ptr(x_pred), m_prev=_ptr(m_prev), noise_c=_ptr(noise_c),
                      noise_p=_ptr(noise_p), out_batch_stride=model_out.stride(0), n=n, hw=h * w,
                      out_dtype=_dt(model_out.dtype), guided=int(bool(guided)), cfg_scale=cfg_scale, sigma=sigma,
                      inv_alpha=1.0 / alpha, c_x=c_x, c_m0=c_m0, c_m1=c_m1, c_noise=c_noise, p_x=p_x, p_m0=p_m0,
                      p_m1=p_m1, p_noise=p_noise)
    _check(load().pxa_sa_solver_step(C.byref(args), _stream()), "pxa_sa_solver_step")
    return x_pred


_IDDPM_DTYPES = {torch.float32: DTYPE_F32, torch.bfloat16: DTYPE_BF16, torch.float16: DTYPE_F16}


def iddpm_step(model_out: torch.Tensor, img: torch.Tensor, noise: Optional[torch.Tensor], next_in: Optional[torch.Tensor], *,
               guided: bool, clip: bool, cfg_scale: float, sqrt_recip_ac: float, sqrt_recipm1_ac: float, post_c1: float,
               post_c2: float, log_beta: float, post_logvar: float) -> torch.Tensor:
    """One IDDPM ancestral step, in place on img (include/pixart_sm100.h: pxa_iddpm_step); returns img.  model_out: the
    learn-sigma output (N, 8, h, w) in fp32, bf16 or fp16 with dense (h, w) planes; guided: N = 2n rows [cond ; uncond], the
    first three eps channels mixed with cfg_scale, and next_in receives [img[:n] ; img[:n]].  img, noise, next_in: fp32
    (N, 4, h, w) contiguous; noise None at t = 0, next_in None when unguided."""
    lat = [t for t in (img, noise, next_in) if t is not None]
    assert model_out.is_cuda and all(t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() for t in lat)
    assert img.dim() == 4 and img.shape[1] == 4 and all(t.shape == img.shape for t in lat)
    assert next_in is not None or not guided
    N, _, h, w = img.shape
    assert not guided or N % 2 == 0, "guided: the batch is CFG pairs [cond ; uncond]"
    assert model_out.dtype in _IDDPM_DTYPES and tuple(model_out.shape) == (N, 8, h, w)
    assert model_out.stride(3) == 1 and model_out.stride(2) == w and model_out.stride(1) == h * w, "model_out: (.., h, w) planes must be dense"
    args = IddpmStepArgs(model_out=_ptr(model_out), img=_ptr(img), noise=_ptr(noise), next_in=_ptr(next_in),
                         out_batch_stride=model_out.stride(0), n=N // 2 if guided else N, hw=h * w,
                         out_dtype=_IDDPM_DTYPES[model_out.dtype], guided=int(bool(guided)), clip=int(bool(clip)),
                         cfg_scale=cfg_scale, sqrt_recip_ac=sqrt_recip_ac, sqrt_recipm1_ac=sqrt_recipm1_ac, post_c1=post_c1,
                         post_c2=post_c2, log_beta=log_beta, post_logvar=post_logvar)
    _check(load().pxa_iddpm_step(C.byref(args), _stream()), "pxa_iddpm_step")
    return img


def _lcm_out(t: torch.Tensor, rows: int, h: int, w: int, what: str) -> None:
    """A denoiser output an LCM kernel reads: CUDA, fp32 / bf16, (rows, >=4, h, w) with dense (h, w) planes."""
    if not (t.is_cuda and t.dtype in (torch.float32, torch.bfloat16) and t.dim() == 4):
        raise PxaError(f"{what}: a 4-D fp32 or bf16 CUDA tensor is required")
    if t.shape[0] != rows or t.shape[1] < 4 or tuple(t.shape[2:]) != (h, w):
        raise PxaError(f"{what}: shape {tuple(t.shape)}, expected ({rows}, >=4, {h}, {w})")
    if not (t.stride(3) == 1 and t.stride(2) == w and t.stride(1) == h * w):
        raise PxaError(f"{what}: (h, w) planes must be dense")


def _lcm_latents(*ts: Optional[torch.Tensor], like: torch.Tensor) -> None:
    for t in ts:
        if t is not None and not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.shape == like.shape):
            raise PxaError(f"latent tensors must be contiguous fp32 CUDA tensors of shape {tuple(like.shape)}")


def lcm_step(model_out: torch.Tensor, x: torch.Tensor, noise: Optional[torch.Tensor], denoised: torch.Tensor,
             x_next: torch.Tensor, *, sqrt_alpha: float, sqrt_beta: float, c_skip: float, c_out: float, c_prev: float,
             c_noise: float) -> None:
    """One LCM sampler step (include/pixart_sm100.h: pxa_lcm_step): denoised and x_next written (x_next may be x).
    model_out: (n, >=4, h, w) fp32 / bf16 (a channel slice is fine); x, noise, denoised, x_next: fp32 (n, 4, h, w)
    contiguous; noise may be None when c_noise is 0."""
    if not (x.dim() == 4 and x.shape[1] == 4):
        raise PxaError("x must be (n, 4, h, w)")
    n, _, h, w = x.shape
    _lcm_out(model_out, n, h, w, "model_out")
    _lcm_latents(x, noise, denoised, x_next, like=x)
    if noise is None and c_noise != 0.0:
        raise PxaError("noise is required when c_noise is non-zero")
    args = LcmStepArgs(model_out=_ptr(model_out), x=_ptr(x), noise=_ptr(noise), denoised=_ptr(denoised), x_next=_ptr(x_next),
                       out_batch_stride=model_out.stride(0), n=n, hw=h * w, out_dtype=_dt(model_out.dtype),
                       sqrt_alpha=sqrt_alpha, sqrt_beta=sqrt_beta, c_skip=c_skip, c_out=c_out, c_prev=c_prev, c_noise=c_noise)
    _check(load().pxa_lcm_step(C.byref(args), _stream()), "pxa_lcm_step")


def _lcm_table(index: torch.Tensor, table: torch.Tensor, b: int, dev) -> int:
    if not (index.is_cuda and index.dtype == torch.int64 and index.is_contiguous() and index.numel() == b and index.device == dev):
        raise PxaError(f"index must be a contiguous int64 CUDA tensor of {b} elements")
    row = C.sizeof(LcmRow)
    if not (table.is_cuda and table.dtype == torch.uint8 and table.numel() % row == 0 and 0 < table.numel() // row <= LCM_MAX_ROWS):
        raise PxaError("table must be the uint8 device copy of 1..LCM_MAX_ROWS LcmRow entries")
    return table.numel() // row


def lcm_teacher_target(teacher_out: torch.Tensor, x_t: torch.Tensor, index: torch.Tensor, table: torch.Tensor,
                       x_prev: torch.Tensor, *, w: float) -> torch.Tensor:
    """Guided DDIM target x_prev (include/pixart_sm100.h: pxa_lcm_teacher_target) from the teacher's output on the batch
    [cond ; uncond] (2b, >=4, h, w) at x_t (b, 4, h, w); `table` is the device copy of the LcmRow table."""
    if not (x_t.dim() == 4 and x_t.shape[1] == 4):
        raise PxaError("x_t must be (b, 4, h, w)")
    b, _, h, w_ = x_t.shape
    _lcm_out(teacher_out, 2 * b, h, w_, "teacher_out")
    _lcm_latents(x_t, x_prev, like=x_t)
    n_rows = _lcm_table(index, table, b, x_t.device)
    args = LcmTeacherArgs(teacher_out=_ptr(teacher_out), x_t=_ptr(x_t), index=_ptr(index), table=_ptr(table), x_prev=_ptr(x_prev),
                          out_batch_stride=teacher_out.stride(0), b=b, hw=h * w_, out_dtype=_dt(teacher_out.dtype),
                          n_rows=n_rows, w=w)
    _check(load().pxa_lcm_teacher_target(C.byref(args), _stream()), "pxa_lcm_teacher_target")
    return x_prev


def lcm_consistency_loss(student_out: torch.Tensor, ema_out: torch.Tensor, x_t: torch.Tensor, x_prev: torch.Tensor,
                         index: torch.Tensor, table: torch.Tensor, d_student_out: torch.Tensor, loss: torch.Tensor,
                         partials: torch.Tensor, *, loss_type: int = LCM_HUBER, huber_c: float = 1e-3) -> torch.Tensor:
    """Consistency loss and its gradient (include/pixart_sm100.h: pxa_lcm_consistency_loss).  student_out: the student's
    fp32 (b, 4 or 8, h, w) output; ema_out: the EMA model's (b, >=4, h, w) output, fp32 or bf16; d_student_out: fp32, the
    shape of student_out, contiguous; loss: fp32 0-d; partials: fp64 [LCM_LOSS_PARTS] workspace."""
    if not (x_t.dim() == 4 and x_t.shape[1] == 4):
        raise PxaError("x_t must be (b, 4, h, w)")
    b, _, h, w = x_t.shape
    _lcm_out(student_out, b, h, w, "student_out")
    _lcm_out(ema_out, b, h, w, "ema_out")
    if student_out.dtype != torch.float32 or student_out.shape[1] not in (4, 8):
        raise PxaError("student_out must be the fp32 (b, 4 or 8, h, w) output of the student")
    _lcm_latents(x_t, x_prev, like=x_t)
    if not (d_student_out.is_cuda and d_student_out.dtype == torch.float32 and d_student_out.is_contiguous()
            and d_student_out.shape == student_out.shape):
        raise PxaError("d_student_out must be a contiguous fp32 CUDA tensor shaped like student_out")
    if not (loss.is_cuda and loss.dtype == torch.float32 and loss.numel() == 1):
        raise PxaError("loss must be a one-element fp32 CUDA tensor")
    if not (partials.is_cuda and partials.dtype == torch.float64 and partials.is_contiguous() and partials.numel() >= LCM_LOSS_PARTS):
        raise PxaError(f"partials must be a contiguous fp64 CUDA tensor of {LCM_LOSS_PARTS} elements")
    n_rows = _lcm_table(index, table, b, x_t.device)
    args = LcmLossArgs(student_out=_ptr(student_out), ema_out=_ptr(ema_out), x_t=_ptr(x_t), x_prev=_ptr(x_prev), index=_ptr(index),
                       table=_ptr(table), d_student_out=_ptr(d_student_out), loss=_ptr(loss), partials=_ptr(partials),
                       student_batch_stride=student_out.stride(0), ema_batch_stride=ema_out.stride(0), b=b, hw=h * w,
                       ema_dtype=_dt(ema_out.dtype), n_rows=n_rows, out_channels=student_out.shape[1], loss_type=loss_type,
                       huber_c=huber_c)
    _check(load().pxa_lcm_consistency_loss(C.byref(args), _stream()), "pxa_lcm_consistency_loss")
    return loss


def ema_flat(table: torch.Tensor, *, n_buckets: int, max_n: int, rate: float) -> None:
    """ema = ema * rate + (1 - rate) * src over every bucket of a device EmaBucket table, with the bf16 shadow written in the
    same pass (include/pixart_sm100.h: pxa_ema_flat).  The caller keeps the tensors behind the table's pointers alive."""
    if not (table.is_cuda and table.dtype == torch.uint8 and table.numel() == n_buckets * C.sizeof(EmaBucket)):
        raise PxaError("table must be the uint8 device copy of n_buckets EmaBucket entries")
    args = EmaArgs(table=_ptr(table), n_buckets=n_buckets, max_n=max_n, rate=rate)
    _check(load().pxa_ema_flat(C.byref(args), _stream()), "pxa_ema_flat")


def dmd_loss(latents: torch.Tensor, noisy: torch.Tensor, timesteps: torch.Tensor, alphas_cumprod: torch.Tensor,
             real_out: torch.Tensor, fake_out: torch.Tensor, d_gen_out: torch.Tensor, loss: torch.Tensor, weight: torch.Tensor,
             partials: torch.Tensor, *, cfg: float, gen_sqrt_alpha: float, gen_sqrt_beta: float) -> torch.Tensor:
    """Distribution-matching loss, its per-sample weight and the gradient with respect to the generator's output
    (include/pixart_sm100.h: pxa_dmd_loss).  latents, noisy: fp32 (b, 4, h, w) contiguous; timesteps: int64 (b,);
    alphas_cumprod: fp32 (T,); real_out: (2b, >=4, h, w) [uncond ; cond], fake_out: (b, >=4, h, w), fp32 or bf16;
    d_gen_out: fp32 (b, 4 or 8, h, w) contiguous; loss: fp32 0-d; weight: fp32 (b,); partials: fp64 [2 b DMD_PARTS]."""
    if not (latents.dim() == 4 and latents.shape[1] == 4):
        raise PxaError("latents must be (b, 4, h, w)")
    b, _, h, w = latents.shape
    _lcm_latents(latents, noisy, like=latents)
    _lcm_out(real_out, 2 * b, h, w, "real_out")
    _lcm_out(fake_out, b, h, w, "fake_out")
    dev = latents.device
    if not (timesteps.is_cuda and timesteps.dtype == torch.int64 and timesteps.is_contiguous() and timesteps.numel() == b
            and timesteps.device == dev):
        raise PxaError(f"timesteps must be a contiguous int64 CUDA tensor of {b} elements")
    if not (alphas_cumprod.is_cuda and alphas_cumprod.dtype == torch.float32 and alphas_cumprod.dim() == 1
            and alphas_cumprod.is_contiguous() and alphas_cumprod.numel() > 0):
        raise PxaError("alphas_cumprod must be a contiguous 1-D fp32 CUDA tensor")
    if not (d_gen_out.is_cuda and d_gen_out.dtype == torch.float32 and d_gen_out.is_contiguous() and d_gen_out.dim() == 4
            and d_gen_out.shape[0] == b and d_gen_out.shape[1] in (4, 8) and tuple(d_gen_out.shape[2:]) == (h, w)):
        raise PxaError(f"d_gen_out must be a contiguous fp32 CUDA tensor of shape ({b}, 4 or 8, {h}, {w})")
    if not (loss.is_cuda and loss.dtype == torch.float32 and loss.numel() == 1):
        raise PxaError("loss must be a one-element fp32 CUDA tensor")
    if not (weight.is_cuda and weight.dtype == torch.float32 and weight.is_contiguous() and weight.numel() == b):
        raise PxaError(f"weight must be a contiguous fp32 CUDA tensor of {b} elements")
    if not (partials.is_cuda and partials.dtype == torch.float64 and partials.is_contiguous()
            and partials.numel() >= 2 * b * DMD_PARTS):
        raise PxaError(f"partials must be a contiguous fp64 CUDA tensor of {2 * b * DMD_PARTS} elements")
    args = DmdLossArgs(latents=_ptr(latents), noisy=_ptr(noisy), timesteps=_ptr(timesteps), alphas_cumprod=_ptr(alphas_cumprod),
                       real_out=_ptr(real_out), fake_out=_ptr(fake_out), d_gen_out=_ptr(d_gen_out), loss=_ptr(loss),
                       weight=_ptr(weight), partials=_ptr(partials), real_batch_stride=real_out.stride(0),
                       fake_batch_stride=fake_out.stride(0), b=b, hw=h * w, n_timesteps=alphas_cumprod.numel(),
                       out_channels=d_gen_out.shape[1], real_dtype=_dt(real_out.dtype), fake_dtype=_dt(fake_out.dtype),
                       cfg=cfg, gen_sqrt_alpha=gen_sqrt_alpha, gen_sqrt_beta=gen_sqrt_beta)
    _check(load().pxa_dmd_loss(C.byref(args), _stream()), "pxa_dmd_loss")
    return loss


# ------------------------------------------------------------------------------------------------- training backward
def transpose(a: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out (C, R) = a (R, C)^T, bf16; a may be a row-strided view (e.g. a column slice)."""
    assert a.dtype == torch.bfloat16 and a.dim() == 2 and a.stride(1) == 1
    R, Cc = a.shape
    if out is None:
        out = torch.empty((Cc, R), dtype=torch.bfloat16, device=a.device)
    assert out.shape == (Cc, R) and out.stride(1) == 1
    _check(load().pxa_transpose_bf16(_ptr(a), _ptr(out), R, Cc, a.stride(0), out.stride(0), _stream()), "pxa_transpose_bf16")
    return out


def gelu_tanh(pre: torch.Tensor, out: Optional[torch.Tensor] = None, dh: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dh None: out = gelu_tanh(pre); else out = dh * gelu_tanh'(pre). Contiguous bf16 tensors."""
    assert pre.dtype == torch.bfloat16 and pre.is_contiguous()
    if out is None:
        out = torch.empty_like(pre)
    assert out.is_contiguous() and out.dtype == torch.bfloat16 and (dh is None or (dh.is_contiguous() and dh.dtype == torch.bfloat16))
    _check(load().pxa_gelu_tanh_bf16(_ptr(pre), _ptr(dh), _ptr(out), pre.numel(), _stream()), "pxa_gelu_tanh_bf16")
    return out


def gate_residual_fwd(x: torch.Tensor, y: torch.Tensor, gate: Optional[torch.Tensor], out: torch.Tensor, *,
                      gate_batch_stride: int = 0, rows_per_batch: int = 0) -> torch.Tensor:
    """out = x + gate[b] * y on the fp32 residual stream (x, out fp32 (M, C); y bf16; gate fp32 view or None)."""
    assert x.dtype == out.dtype == torch.float32 and y.dtype == torch.bfloat16
    assert x.is_contiguous() and y.is_contiguous() and out.is_contiguous() and x.shape == y.shape == out.shape
    M, Cc = x.shape
    args = GateResidualArgs(x=_ptr(x), y=_ptr(y), gate=_ptr(gate), out=_ptr(out), dgate=None,
                            gate_batch_stride=gate_batch_stride, rows_per_batch=rows_per_batch or M, M=M, C=Cc)
    _check(load().pxa_gate_residual_fwd(C.byref(args), _stream()), "pxa_gate_residual_fwd")
    return out


def gate_residual_bwd(dout: torch.Tensor, y: Optional[torch.Tensor], gate: Optional[torch.Tensor], dy: torch.Tensor,
                      dgate: Optional[torch.Tensor], *, gate_batch_stride: int = 0, rows_per_batch: int = 0) -> torch.Tensor:
    """dy = bf16(dout * gate[b]); dgate[b] += sum_rows dout * y (dgate fp32 (B, C) contiguous, pre-zeroed by the caller)."""
    assert dout.dtype == torch.float32 and dout.is_contiguous() and dy.dtype == torch.bfloat16 and dy.is_contiguous()
    assert dgate is None or (dgate.dtype == torch.float32 and dgate.is_contiguous() and y is not None and y.is_contiguous())
    M, Cc = dout.shape
    args = GateResidualArgs(x=_ptr(dout), y=_ptr(y), gate=_ptr(gate), out=_ptr(dy), dgate=_ptr(dgate),
                            gate_batch_stride=gate_batch_stride, rows_per_batch=rows_per_batch or M, M=M, C=Cc)
    _check(load().pxa_gate_residual_bwd(C.byref(args), _stream()), "pxa_gate_residual_bwd")
    return dy


def ln_modulate_bwd(x: torch.Tensor, dxn: torch.Tensor, scale: torch.Tensor, dx: torch.Tensor, dshift: torch.Tensor,
                    dscale: torch.Tensor, *, mod_batch_stride: int, rows_per_batch: int, eps: float = 1e-6,
                    add_in: Optional[torch.Tensor] = None) -> None:
    """Backward of ln_modulate: dx written (= add_in + the gradient through the norm when add_in is given; add_in may be dx
    itself), dshift / dscale (B, C) fp32 accumulated."""
    assert add_in is None or (add_in.dtype == torch.float32 and add_in.is_contiguous() and add_in.shape == x.shape)
    assert x.dtype == dx.dtype == torch.float32 and dxn.dtype == torch.bfloat16
    assert x.is_contiguous() and dxn.is_contiguous() and dx.is_contiguous() and dshift.is_contiguous() and dscale.is_contiguous()
    assert dshift.dtype == dscale.dtype == scale.dtype == torch.float32
    M, Cc = x.shape
    args = LnModBwdArgs(x=_ptr(x), dxn=_ptr(dxn), scale=_ptr(scale), dx=_ptr(dx), dshift=_ptr(dshift), dscale=_ptr(dscale),
                        mod_batch_stride=mod_batch_stride, rows_per_batch=rows_per_batch, M=M, C=Cc, eps=eps,
                        add_in=_ptr(add_in))
    _check(load().pxa_ln_modulate_bwd(C.byref(args), _stream()), "pxa_ln_modulate_bwd")


def colsum(a: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out[c] += sum_r a[r, c]; a bf16 (M, N) row-strided view, out fp32 (N,)."""
    assert a.dtype == torch.bfloat16 and a.dim() == 2 and a.stride(1) == 1 and out.dtype == torch.float32 and out.is_contiguous()
    M, N = a.shape
    assert out.numel() == N
    _check(load().pxa_colsum_bf16(_ptr(a), _ptr(out), M, N, a.stride(0), _stream()), "pxa_colsum_bf16")
    return out


def flash_attn_bwd(q, k, v, o, d_o, lse, dq, dk, dv, *, B: int, H: int, Nq: int, Nk: int, kv_rows: int,
                   kv_len: Optional[torch.Tensor] = None, kv_off: Optional[torch.Tensor] = None, q_strides, k_strides,
                   v_strides, dq_strides, dk_strides, dv_strides, scale: Optional[float] = None,
                   delta: Optional[torch.Tensor] = None) -> None:
    """Backward of flash_attn. q/k/v/dq/dk/dv bf16 views with (row, head) strides; o, d_o (B*Nq, H*72) bf16 row-strided;
    lse (B, H, Nq) fp32 from the forward."""
    for t in (q, k, v, o, d_o, dq, dk, dv):
        assert t.dtype == torch.bfloat16 and t.is_cuda
    assert lse.dtype == torch.float32 and lse.is_contiguous() and lse.numel() == B * H * Nq
    assert o.stride(1) == 1 and d_o.stride(1) == 1
    if delta is None:
        delta = torch.empty(B * H * Nq, dtype=torch.float32, device=q.device)
    args = AttnBwdArgs(q=_ptr(q), k=_ptr(k), v=_ptr(v), o=_ptr(o), d_o=_ptr(d_o), lse=_ptr(lse), delta=_ptr(delta),
                       dq=_ptr(dq), dk=_ptr(dk), dv=_ptr(dv), kv_len=_ptr(kv_len), kv_off=_ptr(kv_off),
                       q_sn=q_strides[0], q_sh=q_strides[1], k_sn=k_strides[0], k_sh=k_strides[1],
                       v_sn=v_strides[0], v_sh=v_strides[1], dq_sn=dq_strides[0], dq_sh=dq_strides[1],
                       dk_sn=dk_strides[0], dk_sh=dk_strides[1], dv_sn=dv_strides[0], dv_sh=dv_strides[1],
                       ldo=o.stride(0), lddo=d_o.stride(0), kv_rows=kv_rows, B=B, H=H, Nq=Nq, Nk=Nk,
                       scale=scale if scale is not None else 72 ** -0.5)
    _check(load().pxa_flash_attn_d72_bwd_bf16(C.byref(args), _stream()), "pxa_flash_attn_d72_bwd_bf16")


def gemm_wgrad(a_t: torch.Tensor, w_t: torch.Tensor, out: torch.Tensor, *, block_n: int = 0, k_splits: int = 0,
               max_ctas: int = 0) -> torch.Tensor:
    """out (M, N) fp32 += a_t^T @ w_t with a_t (K, M) and w_t (K, N) bf16 row-major -- the weight gradient
    dW (N_out, K_in) += dY (rows, N_out)^T @ X (rows, K_in) straight from the activations (MN-major wgmma operands, split-K,
    vector reduce-add into `out`)."""
    assert a_t.dtype == w_t.dtype == torch.bfloat16 and out.dtype == torch.float32
    assert a_t.dim() == 2 and w_t.dim() == 2 and a_t.stride(1) == 1 and w_t.stride(1) == 1 and out.stride(1) == 1
    K, M = a_t.shape
    N = w_t.shape[1]
    assert w_t.shape[0] == K and out.shape == (M, N)
    args = GemmArgs(a=_ptr(a_t), w=_ptr(w_t), bias=None, out=_ptr(out), out_aux_bf16=None, residual=_ptr(out), gate=None,
                    gate_batch_stride=0, rows_per_batch=M, M=M, N=N, K=K, lda=a_t.stride(0), ldw=w_t.stride(0),
                    ldo=out.stride(0), epilogue=EPI_BIAS_RESIDUAL, out_dtype=DTYPE_F32, block_n=block_n, max_ctas=max_ctas,
                    operands_mn_major=1, k_splits=k_splits, aux_is_branch=0)
    _check(load().pxa_gemm_bf16(C.byref(args), _stream()), "pxa_gemm_bf16 (wgrad)")
    return out


def kv_compress_bwd(k_in, v_in, dk_out, dv_out, dk_in, dv_in, conv_w, conv_b, ln_w, d_conv_w, d_conv_b, d_ln_w, d_ln_b, *,
                    B: int, H: int, W: int, ld_in: int, ld_din: int, eps: float = 1e-5) -> None:
    """Backward of kv_compress: dk_in / dv_in (bf16 views, row stride ld_din) written, the four fp32 parameter gradients
    accumulated."""
    for t in (d_conv_w, d_conv_b, d_ln_w, d_ln_b):
        assert t.dtype == torch.float32 and t.is_contiguous()
    assert dk_out.is_contiguous() and dv_out.is_contiguous() and dk_out.dtype == torch.bfloat16
    args = KvCompressBwdArgs(k_in=_ptr(k_in), v_in=_ptr(v_in), dk_out=_ptr(dk_out), dv_out=_ptr(dv_out), dk_in=_ptr(dk_in),
                             dv_in=_ptr(dv_in), conv_w=_ptr(conv_w), conv_b=_ptr(conv_b), ln_w=_ptr(ln_w),
                             d_conv_w=_ptr(d_conv_w), d_conv_b=_ptr(d_conv_b), d_ln_w=_ptr(d_ln_w), d_ln_b=_ptr(d_ln_b),
                             B=B, H=H, W=W, C=dk_out.shape[-1], ld_in=ld_in, ld_din=ld_din, eps=eps)
    _check(load().pxa_kv_compress_conv2_ln_bwd(C.byref(args), _stream()), "pxa_kv_compress_conv2_ln_bwd")
