"""ctypes binding of libk2b200.so (the C ABI declared in include/k2b200.h).

The library is the only compute path: if it is missing, or no sm_90 device is present, every op
raises -- there is deliberately no PyTorch / CPU fallback (BASELINE.json north_star).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "libk2b200.so")

_lib = None
MISSING = []


class K2Error(RuntimeError):
    pass


class K2ConvSrc(ctypes.Structure):
    _fields_ = [("ptr", ctypes.c_void_p), ("C", ctypes.c_int), ("ld", ctypes.c_int), ("taps", ctypes.c_int)]


_P = ctypes.c_void_p
_I = ctypes.c_int
_F = ctypes.c_float
_LL = ctypes.c_longlong

# name -> (restype, argtypes); kept in one table so tests can check every symbol of k2b200.h is exported
SIGNATURES = {
    "k2_last_error": (ctypes.c_char_p, []),
    "k2_version": (_I, []),
    "k2_launch_count": (_LL, []),
    "k2_reset_launch_count": (None, []),
    "k2_set_tuning": (_I, [_I, _I]),
    "k2_conv_gemm": (_I, [ctypes.POINTER(K2ConvSrc), _I, _I, _I, _I, _P, _I, _I, _I, _I, _P, _P, _I, _P, _I, _I, _P, _LL, _P,
                         ctypes.POINTER(ctypes.c_int), _P]),
    "k2_conv_gemm_cfg": (_I, [ctypes.POINTER(K2ConvSrc), _I, _I, _I, _I, _P, _I, _I, _I, _I, _P, _P, _I, _P, _I, _I, _P, _LL, _P,
                             ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int), _LL, _P]),
    "k2_conv_gemm_wmap": (_I, [ctypes.POINTER(K2ConvSrc), _I, _I, _I, _I, _P, _I, _I, _I, _I, _P, _P, _I, _P, _I, _I, _P, _LL,
                              _P, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int), _LL, _I, _P, _P]),
    "k2_sn_apply": (_I, [_P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _I, _I, _P, _I, _P, _I, _P]),
    "k2_transpose_f16": (_I, [_P, _I, _P, _I, _I, _I, _P]),
    "k2_gn_finalize": (_I, [_P, _I, _I, _P, _I, _I, _I, _I, _I, _F, _P, _P]),
    "k2_upsample2x_nhwc": (_I, [_P, _I, _P, _I, _I, _I, _I, _I, _P]),
    "k2_subsample2_nhwc": (_I, [_P, _I, _P, _I, _I, _I, _I, _I, _I, _I, _P]),
    "k2_softmax_rows": (_I, [_P, _I, _P, _I, _LL, _I, _F, _P]),
    "k2_layernorm_f16": (_I, [_P, _I, _P, _P, _P, _I, _I, _I, _F, _P]),
    "k2_gelu_f16": (_I, [_P, _P, _LL, _P]),
    "k2_quick_gelu_f16": (_I, [_P, _P, _LL, _P]),
    "k2_attention_small": (_I, [_P, _I, _P, _I, _P, _I, _I, _I, _I, _F, _P]),
    "k2_prior_tokens": (_I, [_P, _I, _P, _I, _P, _I, _I, _I, _P]),
    "k2_f16_to_f32": (_I, [_P, _I, _P, _I, _I, _I, _P]),
    "k2_clip_patchify": (_I, [_P, _I, _I, _I, _P, _I, _I, _P]),
    "k2_attention_heads": (_I, [_P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _F, _P, _I, _I, _P]),
    "k2_clip_text_embed": (_I, [_P, _I, _I, _I, _P, _I, _P, _I, _P, _I, _P]),
    "k2_clip_text_pool": (_I, [_P, _I, _I, _I, _I, _P, _I, _I, _P, _I, _P, _P]),
    "k2_xlmr_embed": (_I, [_P, _I, _I, _I, _I, _P, _I, _P, _I, _P, _P, _P, _F, _P, _I, _I, _P]),
    "k2_masked_mean_f16": (_I, [_P, _I, _P, _I, _I, _I, _I, _P, _I, _P]),
    "k2_conv_plan": (_I, [_I, _I, _I, _I, _I, _I, _I, _LL, _I, _P]),
    "k2_gn_scratch_floats": (_LL, [_I, _I, _I]),
    "k2_gn_stats": (_I, [_P, _I, _I, _P, _I, _I, _I, _I, _I, _F, _P, _P, _P]),
    "k2_gn_apply": (_I, [_P, _I, _I, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _I, _I, _I, _P, _I, _P, _I, _P,
                         _I, _I, _P, _P]),
    "k2_gn_apply_fold": (_I, [_P, _I, _I, _P, _I, _I, _I, _I, _I, _I, _P, _I, _P, _I, _F, _P, _P, _P, _I, _I, _I, _P, _I, _P,
                              _I, _P]),
    "k2_attention_d64": (_I, [_P, _I, _I, _I, _I, _I, _P, _I, _I, _I, _I, _I, _I, _I, _I, _F, _P, _I, _P]),
    "k2_attention_d512": (_I, [_P, _I, _I, _I, _I, _I, _I, _F, _P, _I, _P]),
    "k2_linear": (_I, [_P, _I, _P, _I, _P, _P, _I, _P, _I, _I, _I, _I, _I, _I, _P]),
    "k2_layernorm": (_I, [_P, _P, _P, _P, _I, _I, _F, _P]),
    "k2_timestep_embedding": (_I, [_P, _P, _I, _I, _F, _P]),
    "k2_f32_to_f16": (_I, [_P, _P, _LL, _P]),
    "k2_silu_f16": (_I, [_P, _P, _LL, _P]),
    "k2_stem_im2col": (_I, [_P, _I, _P, _I, _P, _I, _I, _I, _I, _I, _P, _I, _P]),
    "k2_sampler_step": (_I, [_P, _P, _P, _P, _I, _I, _I, _F, _I, _F, _I, _P, _P, _P, _P, _P]),
    "k2_step_begin": (_I, [_P, _P, _LL, _P, _I, _P, _P, _P, _P, _P, _P, _P]),
    "k2_step_end": (_I, [_P, _P]),
    "k2_slot_step_begin": (_I, [_P, _P, _I, _LL, _P, _P, _P, _P, _I, _P, _P, _P, _P]),
    "k2_slot_step_end": (_I, [_P, _I, _P]),
    "k2_slot_sampler_step": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _F, _I, _I, _P, _P, _P]),
    "k2_slot_dpm_solver_step": (_I, [_P, _I, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "k2_plms_step": (_I, [_P, _I, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _F, _I, _P]),
    "k2_dpm_solver_step": (_I, [_P, _I, _P, _P, _P, _I, _I, _I, _F, _I, _P, _P, _P, _P]),
    "k2_dpm_solver_sde_step": (_I, [_P, _I, _P, _P, _P, _P, _I, _I, _I, _F, _I, _P, _P, _P, _P]),
    "k2_unipc_step": (_I, [_P, _I, _P, _P, _P, _P, _P, _P, _I, _I, _I, _F, _I, _P, _P, _P, _P]),
    "k2_heun_step": (_I, [_P, _I, _P, _P, _P, _P, _I, _I, _I, _F, _I, _P, _P, _P, _P]),
    "k2_vq_argmin": (_I, [_P, _P, _P, _I, _I, _I, _P]),
    "k2_pointwise_nchw_f32": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "k2_nchw_to_nhwc_f32": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "k2_images_to_u8": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "k2_lora_merge": (_I, [_P, _I, _P, _P, _I, _I, _I, _F, _P, _I, _P]),
    "k2_relu_f16": (_I, [_P, _I, _P, _I, _I, _I, _P]),
    "k2_relu_f32": (_I, [_P, _I, _P, _I, _I, _I, _P]),
    "k2_bilinear_f16": (_I, [_P, _I, _I, _I, _I, _I, _P, _I, _I, _I, _I, _P]),
    "k2_depth_to_space_f16": (_I, [_P, _I, _I, _I, _I, _I, _I, _P, _I, _P]),
    "k2_readout_rows_f16": (_I, [_P, _I, _I, _I, _I, _P, _I, _P]),
    "k2_im2col_f16": (_I, [_P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _I, _I, _P]),
    "k2_maxpool_f16": (_I, [_P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _I, _P]),
    "k2_gn_act_f16": (_I, [_P, _I, _P, _P, _P, _P, _I, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _I, _LL, _P]),
}


def load():
    """Load the shared library (once) and attach prototypes. Raises K2Error if it was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise K2Error(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no fallback path)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            MISSING.append(name)  # tests/test_abi.py asserts this list is empty
            continue
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise K2Error(load().k2_last_error().decode())


def stream_ptr():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL)."""
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())
