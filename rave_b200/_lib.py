"""ctypes binding of the C ABI declared in include/rave_b200.h.

This is the stub a maintainer of the reference would add (INTEGRATION.md): every device
computation of the hot path goes through one of these entry points.  There is NO fallback: if
`librave_b200.so` is missing, or a tensor is not on a CUDA device, the call raises.
"""
import ctypes
import os
from ctypes import c_float, c_int, c_long, c_longlong, c_size_t, c_ulonglong, c_void_p, c_char_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "librave_b200.so")

_P, _I, _F, _L = c_void_p, c_int, c_float, c_long

# name -> (restype, argtypes); must list every symbol of include/rave_b200.h
SIGNATURES = {
    "rave_b200_version": (c_int, []),
    "rave_b200_last_error": (c_char_p, []),
    "rave_b200_launch_count": (c_ulonglong, []),
    "rave_pqmf_analysis_fwd": (c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "rave_pqmf_synthesis_fwd": (c_int, [_P, _P, _P, _I, _I, _I, _I, _F, _I, _P]),
    "rave_pqmf_analysis_fast": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "rave_pqmf_synthesis_fast": (c_int, [_P, _P, _P, _P, _I, _I, _I, _F, _I, _P]),
    "rave_conv1d_gather_f32": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _L, _L,
                                       _I, _F, _P, _I, _F, _P, _P, _P]),
    "rave_conv1d_scatter_f32": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _L, _L,
                                        _I, _F, _P, _I, _F, _P, _P, _P]),
    "rave_conv1d_wgrad_workspace_bytes": (c_size_t, [_I, _I, _I, _I, _I]),
    "rave_conv1d_wgrad_f32": (c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _L, _L, _I, _I,
                                      _F, _P, _P, _P]),
    "rave_weight_norm_fwd": (c_int, [_P, _P, _P, _P, _I, _I, _P]),
    "rave_weight_norm_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _I, _I, _P]),
    "rave_act_fwd": (c_int, [_P, _P, _I, _I, _I, _I, _F, _P, _P]),
    "rave_act_bwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _F, _P, _P]),
    "rave_am_tanh_fwd": (c_int, [_P, _P, _I, _I, _I, _P]),
    "rave_am_tanh_bwd": (c_int, [_P, _P, _P, _I, _I, _I, _P]),
    "rave_reparam_fwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _P]),
    "rave_mmd_fwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _P]),
    "rave_mmd_bwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _P]),
    "rave_sphere_norm_fwd": (c_int, [_P, _P, _P, _I, _I, _I, _P]),
    "rave_sphere_norm_bwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _P]),
    "rave_latent_moments": (c_int, [_P, _I, _I, _I, _I, _P, _P, _P]),
    "rave_latent_moments_workspace_bytes": (c_long, [_I, _I, _I]),
    "rave_conv1d_tc_supported": (c_int, [_I, _I, _I, _I, _I]),
    "rave_dilated_unit_tc_supported": (c_int, [_I, _I]),
    "rave_dilated_unit_tc_fwd": (c_int, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _F, _I, _F, _P]),
    "rave_conv1d_tc_plan": (c_int, [_I, _I, _I, _I, _I]),
    "rave_conv1d_tc_pp_stages": (c_int, [_I, _I, _I, _I, _I, _I, _I]),
    "rave_conv1d_tc_pp_fwd_stages": (c_int, [_I, _I, _I, _I, _I]),
    "rave_conv1d_tc_wide_stages": (c_int, [_I, _I, _I, _I, _I]),
    "rave_conv1d_tc_fwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, _F, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I,
                                   _F, _I, _I, _I, _P, _I, _P]),
    "rave_conv1d_tc_fwd_x3": (c_int, [_P, _P, _P, _P, _P, _F, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _F, _I,
                                      _I, _I, _I, _P]),
    "rave_weight_prep_tc_multi_x3": (c_int, [_I, _P, _P]),
    "rave_ncl_to_cl_x3": (c_int, [_P, _P, _I, _I, _I, _P]),
    "rave_conv1d_tc_wgrad": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "rave_tapmajor_to_weight_f32": (c_int, [_P, _P, _I, _I, _I, _I, _I, _P]),
    "rave_conv1d_tc_wgrad_splits": (c_int, [_I, _I, _I, _I, _I]),
    "rave_conv1d_tc_wgrad_plan": (c_int, [_I, _I, _I, _I, _I]),
    "rave_time_stack_cl": (c_int, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "rave_time_stack_cl_bwd": (c_int, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "rave_time_stack_nhwc": (c_int, [_P, _P, _I, _I, _I, _I, ctypes.c_long, ctypes.c_long, _I, _I, _I, _I, _P]),
    "rave_time_stack_nhwc_bwd": (c_int, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "rave_time_stack_nhwc_dil": (c_int, [_P, _P, _I, _I, _I, _I, ctypes.c_long, ctypes.c_long, _I, _I, _I, _I, _I, _P]),
    "rave_time_stack_nhwc_dil_bwd": (c_int, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "rave_l1_stats_f32": (c_int, [_P, _P, _P, ctypes.c_long, _P]),
    "rave_leaky_fm_fwd": (c_int, [_P, _P, _P, ctypes.c_long, ctypes.c_float, _P]),
    "rave_leaky_fm_bwd": (c_int, [_P, _P, _P, _P, ctypes.c_long, ctypes.c_float, _P]),
    "rave_leaky_fm_stack_fwd": (c_int, [_P, _P, _P, _P, ctypes.c_long, _I, _I, _I, _I, ctypes.c_float, _P]),
    "rave_leaky_fm_stack_bwd": (c_int, [_P, _P, _P, _P, _P, ctypes.c_long, _I, _I, _I, _I, ctypes.c_float, _P]),
    "rave_leaky_fm_stack_dil_fwd": (c_int, [_P, _P, _P, _P, ctypes.c_long, _I, _I, _I, _I, _I, ctypes.c_float, _P]),
    "rave_leaky_fm_stack_dil_bwd": (c_int, [_P, _P, _P, _P, _P, ctypes.c_long, _I, _I, _I, _I, _I, ctypes.c_float, _P]),
    "rave_l1_grad_f32": (c_int, [_P, _P, _P, _P, _P, ctypes.c_long, _P]),
    "rave_snake_cl_fwd": (c_int, [_P, _P, _P, ctypes.c_long, _I, _P]),
    "rave_snake_cl_bwd": (c_int, [_P, _P, _P, _P, _P, _P, ctypes.c_long, _I, _P]),
    "rave_adain_cl_stats": (c_int, [_P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _P, _P]),
    "rave_adain_snake_cl_fwd": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "rave_weight_prep_tc": (c_int, [_P, _P, _P, _P, _P, _I, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "rave_weight_norm_bwd_tapmajor": (c_int, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "rave_conv1d_c1_fwd": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _F, _P]),
    "rave_conv1d_c1_wgrad_splits": (c_int, [_I, _I]),
    "rave_conv1d_c1_wgrad": (c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "rave_conv1d_c1_dgrad": (c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "rave_colsum_bf16": (c_int, [_P, _P, _I, _I, _I, _I, _I, _P]),
    "rave_im2col_c1": (c_int, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "rave_gather_c1": (c_int, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "rave_im2col_cin": (c_int, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "rave_gather_cin": (c_int, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "rave_fm_stats": (c_int, [_P, _P, _I, _I, _I, _I, _F, _P]),
    "rave_fm_grad": (c_int, [_P, _P, _P, _I, _I, _I, _I, _F, _P]),
    "rave_score_stats": (c_int, [_P, _P, _I, _I, _I, _I, _P]),
    "rave_score_grad": (c_int, [_P, _P, _P, _I, _I, _I, _I, _P]),
    "rave_spectral_stats": (c_int, [_P, _P, _P, _L, _F, _P]),
    "rave_spectral_grad": (c_int, [_P, _P, _P, _P, _P, _L, _F, _P]),
    "rave_stft_frames": (c_int, [_P, _P, _P, _I, _I, _I, _I, _P]),
    "rave_stft_frames_bwd": (c_int, [_P, _P, _P, _I, _I, _I, _I, _P]),
    "rave_stft_frames_valid": (c_int, [_P, _P, _P, _I, _I, _I, _I, _F, _P]),
    "rave_stft_frames_valid_bwd": (c_int, [_P, _P, _P, _I, _I, _I, _I, _F, _P]),
    "rave_rfft_bwd_scale": (c_int, [_P, _P, _L, _I, _I, _L, _L, _L, _P]),
    "rave_mel_log1p_fwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _F, _P]),
    "rave_mel_log1p_bwd": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _F, _P]),
    "rave_gru_fwd": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "rave_gru_bwd": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "rave_gemm_f32_splits": (c_int, [_I, _I, _I]),
    "rave_gemm_f32": (c_int, [_P, _L, _L, _P, _L, _L, _P, _P, _L, _P, _I, _I, _I, _P, _I, _P]),
    "rave_noise_fir_fwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "rave_noise_fir_bwd": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "rave_adam_multi": (c_int, [_I, _P, _P, _P, _P, _P, _P, _P, _F, _F, _F, _P]),
    "rave_weight_prep_tc_multi": (c_int, [_I, _P, _P]),
    "rave_weight_norm_bwd_multi": (c_int, [_I, _P, _P]),
    "rave_ncl_to_cl": (c_int, [_P, _P, _P, _I, _I, _I, _I, _F, _P, _P]),
    "rave_cl_to_ncl": (c_int, [_P, _P, _I, _I, _I, _P]),
    "rave_act_to_bf16": (c_int, [_P, _P, _I, _I, _I, _I, _F, _P, _P]),
    "rave_weight_to_tapmajor_bf16": (c_int, [_P, _P, _I, _I, _I, _I, _I, _P]),
    "rave_prior_latent_classes": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "rave_prior_embed_fwd": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _F, _P]),
    "rave_prior_embed_wgrad": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _F, _P]),
    "rave_gate_fwd": (c_int, [_P, _P, _I, _I, _I, _I, _P]),
    "rave_gate_bwd": (c_int, [_P, _P, _P, _I, _I, _I, _I, _P]),
    "rave_prior_head_ce_fwd": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _P]),
    "rave_prior_head_ce_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _P]),
    "rave_prior_sample_workspace_bytes": (c_long, [_I, _I, _I, _I, _I, _I, _I]),
    "rave_prior_sample": (c_int, [_P, _I, _I, _I, _I, _I, _I, _I, _P, _I, _P, _I, _I, _I, _P, _P, _P, _L, _P]),
    "rave_prior_classes_to_latent": (c_int, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "rave_prior_stream_workspace_bytes": (c_long, [_I, _I, _I, _I, _I, _I, _I]),
    "rave_prior_stream_create": (c_int, [_P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _L, _P]),
    "rave_prior_stream_reset": (c_int, [_P, _P]),
    "rave_prior_stream": (c_int, [_P, _P, _P, _P, _P, _I, _P]),
    "rave_prior_stream_destroy": (c_int, [_P]),
    "rave_augment": (c_int, [_P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _I, _I, _P]),
    "rave_ema_chunk_elems": (c_longlong, []),
    "rave_ema_update": (c_int, [_P, _I, c_longlong, _P, _F, _F, _P]),
    "rave_ema_swap": (c_int, [_P, _I, c_longlong, _P]),
    "rave_latent_project": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "rave_latent_unproject": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "rave_rvq_encode": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "rave_rvq_decode": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "rave_sphere_to_angles": (c_int, [_P, _P, _I, _I, _I, _P]),
    "rave_angles_to_sphere": (c_int, [_P, _P, _I, _I, _I, _P]),
    "rave_resample": (c_int, [_P, _P, _P, c_longlong, _I, _I, _I, _I, _I, _I, _P]),
}



class WPrepLayer(ctypes.Structure):
    """struct rave_wprep_layer of include/rave_b200.h"""
    _fields_ = [("v", c_void_p), ("g", c_void_p), ("norm", c_void_p), ("outA", c_void_p), ("outB", c_void_p),
                ("dwt", c_void_p), ("dv", c_void_p), ("dg", c_void_p),
                ("C0", c_int), ("C1", c_int), ("K", c_int), ("C0p", c_int), ("C1p", c_int), ("nA", c_int),
                ("nB", c_int), ("splits", c_int), ("tapsA", c_int * 32), ("tapsB", c_int * 32)]


_lib = None


class RaveB200Error(RuntimeError):
    pass


def load():
    """Load librave_b200.so (once). Raises if it has not been built: there is no CPU path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise RaveB200Error(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(rave_b200 has no CPU or PyTorch fallback)")
    import torch  # noqa: F401  (makes libcudart.so.12 resident before our library asks for it)
    lib = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error() -> str:
    return load().rave_b200_last_error().decode()


def launch_count() -> int:
    return int(load().rave_b200_launch_count())


PROFILE = None      # set to a list: every call is timed alone (sync + CUDA events) and logged as
                    # (entry point, integer arguments, milliseconds)


def call(name: str, *args):
    """Invoke an int-returning entry point; non-zero -> RuntimeError with the library's message."""
    lib = load()
    if PROFILE is not None:
        import torch
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        rc = getattr(lib, name)(*args)
        e1.record()
        torch.cuda.synchronize()
        ints = tuple(a for a in args if isinstance(a, int) and not isinstance(a, bool) and abs(a) < (1 << 24))
        ptrs = "".join("-" if a is None else "P" for a in args
                       if a is None or (isinstance(a, int) and abs(a) >= (1 << 24)))
        PROFILE.append((name, ints, ptrs, e0.elapsed_time(e1)))
    else:
        rc = getattr(lib, name)(*args)
    if rc != 0:
        raise RaveB200Error(f"{name} failed (rc={rc}): {last_error()}")


def ptr(t):
    """Device pointer of a tensor (None -> NULL).  Refuses host tensors: no CPU fallback."""
    if t is None:
        return None
    if not t.is_cuda:
        raise RaveB200Error("rave_b200 ops need CUDA tensors (there is no CPU path)")
    if not t.is_contiguous():
        raise RaveB200Error("rave_b200 ops need contiguous tensors")
    return t.data_ptr()


def stream_ptr():
    import torch
    return torch.cuda.current_stream().cuda_stream
