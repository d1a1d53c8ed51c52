"""ctypes binding of libb200deflicker.so (include/b200_deflicker.h).

The library is the product: there is no Python/PyTorch fallback.  `lib()` raises if the shared
object is missing or a symbol declared in the header is not exported; every wrapper raises
`B200Error` on a non-zero return code.
"""
from __future__ import annotations

import ctypes as C
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libb200deflicker.so")
HOSTCHECK_PATH = os.path.join(HERE, "libb200_hostcheck.so")
HEADER = os.path.join(os.path.dirname(os.path.dirname(HERE)), "include", "b200_deflicker.h")

PREC_FP32 = 0
PREC_TC = 1
LOSS_FLOATS = 8
RECORD_FLOATS = 16
MAX_LAYERS = 16


class B200Error(RuntimeError):
    pass


class MlpDesc(C.Structure):
    _fields_ = [("input_dim", C.c_int32), ("output_dim", C.c_int32), ("hidden_dim", C.c_int32),
                ("num_layers", C.c_int32), ("pe_freqs", C.c_int32), ("skip_mask", C.c_uint32),
                ("use_tanh", C.c_int32), ("reserved", C.c_int32)]


class Video(C.Structure):
    _fields_ = [("records", C.c_void_p), ("mask_fwd_bits", C.c_void_p), ("mask_bwd_bits", C.c_void_p),
                ("H", C.c_int32), ("W", C.c_int32), ("T", C.c_int32),
                ("t_begin", C.c_int32), ("t_end", C.c_int32), ("reserved", C.c_int32)]


class ConvDesc(C.Structure):
    _fields_ = [("N", C.c_int32), ("Cin", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
                ("in_c_total", C.c_int32), ("in_c_off", C.c_int32), ("Cout", C.c_int32), ("KH", C.c_int32),
                ("KW", C.c_int32), ("stride", C.c_int32), ("pad_h", C.c_int32), ("pad_w", C.c_int32),
                ("pad_mode", C.c_int32), ("upsample", C.c_int32), ("out_c_total", C.c_int32),
                ("out_c_off", C.c_int32), ("act", C.c_int32), ("out_scale", C.c_float),
                ("res_c_total", C.c_int32), ("res_c_off", C.c_int32), ("upsample_mode", C.c_int32)]


MAX_RANKS = 16


class DpComm(C.Structure):
    _fields_ = [("world", C.c_int32), ("rank", C.c_int32), ("partials", C.c_void_p * MAX_RANKS),
                ("params", C.c_void_p * MAX_RANKS), ("flags", C.c_void_p * MAX_RANKS)]


class AtlasConfig(C.Structure):
    _fields_ = [("batch", C.c_int32), ("with_global", C.c_int32), ("precision", C.c_int32),
                ("resx", C.c_int32), ("uv_mapping_scale", C.c_float), ("derivative_amount", C.c_float),
                ("global_derivative_amount", C.c_float), ("rgb_coeff", C.c_float),
                ("gradient_coeff", C.c_float), ("rigidity_coeff", C.c_float),
                ("global_rigidity_coeff", C.c_float), ("flow_coeff", C.c_float)]


class SegConfig(C.Structure):
    _fields_ = [("batch", C.c_int32), ("with_global", C.c_int32), ("precision", C.c_int32), ("resx", C.c_int32),
                ("uv_mapping_scale", C.c_float), ("derivative_amount", C.c_float),
                ("global_derivative_amount", C.c_float), ("rgb_coeff", C.c_float), ("gradient_coeff", C.c_float),
                ("rigidity_coeff", C.c_float), ("global_rigidity_coeff_fg", C.c_float),
                ("global_rigidity_coeff_bg", C.c_float), ("flow_coeff", C.c_float), ("alpha_flow_factor", C.c_float),
                ("sparsity_coeff", C.c_float), ("bootstrapping_factor", C.c_float),
                ("mapping1", MlpDesc), ("mapping2", MlpDesc), ("alpha", MlpDesc), ("atlas", MlpDesc)]


class PngPlan(C.Structure):
    _fields_ = [("magic", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("n_blocks", C.c_int32),
                ("n_chunks", C.c_int32), ("prefix_bytes", C.c_int32), ("suffix_bytes", C.c_int32),
                ("max_chunk", C.c_int32), ("raw_bytes", C.c_int64), ("zlib_bytes", C.c_int64),
                ("file_bytes", C.c_int64), ("plan_bytes", C.c_int64), ("block_raw_at", C.c_int64),
                ("chunk_z_at", C.c_int64), ("prefix_at", C.c_int64), ("suffix_at", C.c_int64),
                ("zlib_header", C.c_uint8 * 8)]


SEG_LOSS_FLOATS = 16
SEG_OFFSET_FLOATS = 15

_P = C.c_void_p
_I64 = C.c_int64
_I32 = C.c_int32
_F = C.c_float

# name -> (restype, argtypes); must list every function the header declares
SIGNATURES = {
    "b200_last_error": (C.c_char_p, []),
    "b200_version": (C.c_int, []),
    "b200_device_supports_tc": (C.c_int, []),
    "b200_launch_count": (C.c_longlong, []),
    "b200_debug_wgrad": (C.c_int, [_P, _P, _I32]),
    "b200_set_kernel_timer": (C.c_int, [_P, _P, C.c_int]),
    "b200_mlp_layout": (_I64, [C.POINTER(MlpDesc), C.POINTER(_I64), C.POINTER(_I64)]),
    "b200_mlp_workspace_bytes": (_I64, [C.POINTER(MlpDesc), _I64, C.c_int]),
    "b200_mlp_forward": (C.c_int, [C.POINTER(MlpDesc), _P, _P, _P, _I64, C.c_int, C.c_int, _P, _I64, _P]),
    "b200_mlp_backward": (C.c_int, [C.POINTER(MlpDesc), _P, _P, _P, _P, _P, _I64, C.c_int, _P, _I64, _P]),
    "b200_video_pack": (C.c_int, [_P] * 7 + [_I32] * 5 + [_P, _P, _P, _P]),
    "b200_atlas_param_floats": (_I64, []),
    "b200_atlas_workspace_bytes": (_I64, [C.POINTER(AtlasConfig)]),
    "b200_atlas_workspace_offsets": (C.c_int, [C.POINTER(AtlasConfig), _P, C.POINTER(_I64)]),
    "b200_atlas_loss_grad": (C.c_int, [C.POINTER(AtlasConfig), C.POINTER(Video), _P, _P, _P, _P, _P, _I64, _P]),
    "b200_pretrain_loss_grad": (C.c_int, [C.POINTER(AtlasConfig), _I32, _I32, _I32, _P, _P, _P, _P, _P, _P, _I64, _P]),
    "b200_atlas_param_floats_for": (_I64, [C.POINTER(MlpDesc)]),
    "b200_atlas_workspace_bytes_for": (_I64, [C.POINTER(AtlasConfig), C.POINTER(MlpDesc)]),
    "b200_atlas_workspace_offsets_for": (C.c_int, [C.POINTER(AtlasConfig), C.POINTER(MlpDesc), _P, C.POINTER(_I64)]),
    "b200_mlp_tc_image_offsets": (C.c_int, [C.POINTER(MlpDesc), _I64, _P, C.POINTER(_I64)]),
    "b200_atlas_tc_image_offsets_for": (C.c_int, [C.POINTER(AtlasConfig), C.POINTER(MlpDesc), _P, _I32,
                                                  C.POINTER(_I64)]),
    "b200_atlas_loss_grad_for": (C.c_int, [C.POINTER(AtlasConfig), C.POINTER(MlpDesc), C.POINTER(Video), _P, _P, _P, _P,
                                           _P, _I64, _P]),
    "b200_pretrain_loss_grad_for": (C.c_int, [C.POINTER(AtlasConfig), C.POINTER(MlpDesc), _I32, _I32, _I32, _P, _P, _P,
                                              _P, _P, _P, _I64, _P]),
    "b200_render_workspace_bytes_for": (_I64, [C.POINTER(MlpDesc), _I64]),
    "b200_render_for": (C.c_int, [C.POINTER(MlpDesc), _P, _I32, _I32, _I32, _I32, _I64, _I64, _P, _P, C.c_int, _P, _I64,
                                  _P]),
    "b200_adam_step": (C.c_int, [_P, _P, _P, _P, _I64, C.c_double, C.c_double, C.c_double, C.c_double, _F, _P, _P]),
    "b200_gradient_loss_head": (C.c_int, [_P] * 5 + [_I64] + [_P] * 5),
    "b200_rigidity_loss_head": (C.c_int, [_P, _P, _I64, _F, _F, _F, _P, _P, _P, _P, _P]),
    "b200_flow_loss_head": (C.c_int, [_P, _P, _I64, _F, _F, _P, _P, _P, _P]),
    "b200_flow_loss_head_weighted": (C.c_int, [_P, _P, _P, _I64, _F, _F, _P, _P, _P, _P, _P]),
    "b200_producer_frame": (C.c_int, [_P, _I32, _I32, _P, _P]),
    "b200_producer_scratch_floats": (_I64, [_I32, _I32]),
    "b200_producer_flow_pair": (C.c_int, [_P, _P] + [_I32] * 7 + [_P, _P, _P, _I32, _I32, _P, _P]),
    "b200_stage2_pack_input": (C.c_int, [_P, _I32, _I32, _I32, _P, _I32, _I32, _I32, _P, _I32, _I32, _P]),
    "b200_stage2_emit": (C.c_int, [_P, _I64, _I32, _I32, _P, _I64, _I64, _I32, _I32, _P]),
    "b200_png_plan_bytes": (_I64, [_I32, _I32, _I32, _I32]),
    "b200_png_plan": (C.c_int, [_I32, _I32, _P, _P, _P, _I32, _P, _I32, _P, _I32, _P, _I32, _P, _I64]),
    "b200_png_workspace_bytes": (_I64, [_I32, _I32]),
    "b200_png_encode": (C.c_int, [C.POINTER(PngPlan), _P, _P, _P, _I64, _P, _I64, _P]),
    "b200_dp_adam_step": (C.c_int, [C.POINTER(DpComm), _P, _P, _I64, _I64, C.c_double, C.c_double, C.c_double, C.c_double,
                                    _P, _P, _P]),
    "b200_dp_slice": (C.c_int, [_I32, _I32, _I64, C.POINTER(_I64), C.POINTER(_I64)]),
    "b200_mlp_tc_architecture": (C.c_int, [C.POINTER(MlpDesc)]),
    "b200_seg_param_floats": (_I64, [C.POINTER(SegConfig), C.POINTER(_I64)]),
    "b200_seg_workspace_bytes": (_I64, [C.POINTER(SegConfig)]),
    "b200_seg_loss_grad": (C.c_int, [C.POINTER(SegConfig), C.POINTER(Video), _P, _P, _P, _P, _P, _P, _I64, _P]),
    "b200_seg_workspace_offsets": (C.c_int, [C.POINTER(SegConfig), _P, C.POINTER(_I64)]),
    "b200_seg_tc_image_offsets": (C.c_int, [C.POINTER(SegConfig), _P, _I32, C.POINTER(_I64)]),
    "b200_mlp_pretrain_workspace_bytes": (_I64, [C.POINTER(MlpDesc), _I32]),
    "b200_mlp_pretrain_loss_grad": (C.c_int, [C.POINTER(MlpDesc), _I32, _F, _I32, _I32, _I32, _P, _P, _P, _P, _P, C.c_int,
                                              _P, _I64, _P]),
    "b200_seg_render_workspace_bytes": (_I64, [C.POINTER(SegConfig), _I64]),
    "b200_seg_render": (C.c_int, [C.POINTER(SegConfig), _P, _I32, _I32, _I32, _I32, _I64, _I64, _P, _P, _P, _P, _I64, _P]),
    "b200_eval_maps_workspace_bytes": (_I64, [C.POINTER(MlpDesc), _I64]),
    "b200_eval_maps": (C.c_int, [C.POINTER(MlpDesc), _P, C.POINTER(Video), _I32, _I64, _I64, _F, _F, C.c_int, _P, _P, _P,
                                 _P, _I64, _P]),
    "b200_frame_sse_workspace_bytes": (_I64, [_I32, _I32]),
    "b200_frame_sse": (C.c_int, [C.POINTER(Video), _I32, _P, _P, _P, _I64, _P]),
    "b200_render_workspace_bytes": (_I64, [_I64]),
    "b200_render": (C.c_int, [_P, _I32, _I32, _I32, _I32, _I64, _I64, _P, _P, C.c_int, _P, _I64, _P]),
    "b200_corr_pyramid_floats": (_I64, [_I32, _I32]),
    "b200_corr_build": (C.c_int, [_P, _P, _I32, _I32, _I32, _P, _P]),
    "b200_corr_pool_levels": (C.c_int, [_P, _I32, _I32, _P]),
    "b200_corr_build_tc_workspace_bytes": (C.c_int64, [_I32, _I32, _I32]),
    "b200_corr_build_tc": (C.c_int, [_P, _P, _I32, _I32, _I32, _P, _P, C.c_int64, _P]),
    "b200_corr_lookup": (C.c_int, [_P, _P, _P, _I32, _I32, _I32, _I32, _P]),
    "b200_corr_alt_floats": (_I64, [_I32, _I32, _I32]),
    "b200_corr_alt_build": (C.c_int, [_P, _P, _I32, _I32, _I32, _P, _P]),
    "b200_corr_alt_lookup": (C.c_int, [_P, _P, _P, _I32, _I32, _I32, _I32, _I32, _P]),
    "b200_corr_build_batch": (C.c_int, [_P, _P, _I32, _I32, _I32, _I32, _P, _P]),
    "b200_corr_pool_levels_batch": (C.c_int, [_P, _I32, _I32, _I32, _P]),
    "b200_corr_build_tc_batch_workspace_bytes": (C.c_int64, [_I32, _I32, _I32, _I32]),
    "b200_corr_build_tc_batch": (C.c_int, [_P, _P, _I32, _I32, _I32, _I32, _P, _P, C.c_int64, _P]),
    "b200_corr_lookup_batch": (C.c_int, [_P, _P, _P, _I32, _I32, _I32, _I32, _P]),
    "b200_corr_alt_build_batch": (C.c_int, [_P, _P, _I32, _I32, _I32, _I32, _P, _P]),
    "b200_corr_alt_lookup_batch": (C.c_int, [_P, _P, _P, _I32, _I32, _I32, _I32, _I32, _P]),
    "b200_conv2d": (C.c_int, [C.POINTER(ConvDesc), _P, _P, _P, _P, _P, _P]),
    "b200_conv_tma_workspace_bytes": (C.c_int64, [C.POINTER(ConvDesc)]),
    "b200_conv_tma_weight_image_bytes": (C.c_int64, [C.POINTER(ConvDesc)]),
    "b200_conv_tma_weight_images": (C.c_int, [C.POINTER(ConvDesc), _P, _P, _P]),
    "b200_conv_tma_chainable": (C.c_int, [C.POINTER(ConvDesc)]),
    "b200_conv2d_tma_chain": (C.c_int, [C.POINTER(ConvDesc), _P, _P, _P, _P, _P, _P, _P, C.POINTER(ConvDesc), _I32, _P,
                                        C.c_int64, _P]),
    "b200_conv_tma_pack_chain": (C.c_int, [C.POINTER(ConvDesc), _P, _I32, _P, _I32, _P]),
    "b200_convlstm_tma_weight_images": (C.c_int, [C.POINTER(ConvDesc), _P, _P, _P]),
    "b200_convlstm_tma": (C.c_int, [C.POINTER(ConvDesc), _P, _P, _P, _P, _P, _P, _P, _P, C.c_int64, _P]),
    "b200_maxpool2": (C.c_int, [_P, _P, _I64, _I32, _I32, _P]),
    "b200_upsample_bilinear2": (C.c_int, [_P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "b200_instance_norm": (C.c_int, [_P, _P, _I64, _I64, _F, _I32, _P]),
    "b200_add_relu": (C.c_int, [_P, _P, _P, _I64, _P]),
    "b200_gru_gate": (C.c_int, [_P, _P, _P, _P, _I64, _I64, _I64, _I32, _P]),
    "b200_convlstm_cell": (C.c_int, [_P, _P, _P, _P, _I32, _I32, _I32, _I32, _P]),
    "b200_convlstm_zero_state": (C.c_int, [_P, _P, _P, _I32, _I32, _I32, _I32, _P]),
    "b200_convex_upsample": (C.c_int, [_P, _P, _P, _I32, _I32, _I32, _P]),
}

_lib = None


def header_functions():
    """Names of all functions declared in include/b200_deflicker.h."""
    with open(HEADER) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", text)))


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B200Error(f"{LIB_PATH} is missing — build it with "
                            f"`python all-in-one-deflicker_b200/csrc/build.py` (there is no fallback path)")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)          # AttributeError if not exported
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def last_error() -> str:
    return lib().b200_last_error().decode(errors="replace")


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = lib().b200_last_error().decode(errors="replace")
        raise B200Error(f"{what} failed with code {rc}: {msg}")


def ptr(t):
    """Device (or host) pointer of a torch tensor, None -> NULL."""
    if t is None:
        return None
    return C.c_void_p(t.data_ptr())


def current_stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def hostcheck():
    """CPU build of csrc/loss_math.h for the host-math tests."""
    h = C.CDLL(HOSTCHECK_PATH)
    h.b200_host_sample_loss.argtypes = [_P, _P, _P]
    h.b200_host_seg_sample_loss.argtypes = [_P, _P, _P]
    h.b200_host_norm_coords.argtypes = [_P, _I64, _F, _P]
    h.b200_host_pe_freq.restype = _F
    h.b200_host_pe_freq.argtypes = [C.c_int]
    h.b200_host_pretrain.restype = _F
    h.b200_host_pretrain.argtypes = [_F, _F, _P, _F, _F, _P]
    return h
