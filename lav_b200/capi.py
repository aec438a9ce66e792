"""ctypes binding of include/lav_b200.h — the only way Python reaches the CUDA kernels.

There is no CPU fallback: if the shared library is missing or a call fails, this raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_lib", "liblavb200.so")

F32, BF16, F16 = 0, 1, 2


class LavbError(RuntimeError):
    pass


class ConvDesc(C.Structure):
    """mirror of lavb_conv_desc"""
    _fields_ = [
        ("inp", C.c_void_p), ("in_dtype", C.c_int), ("n", C.c_int), ("hin", C.c_int), ("win", C.c_int), ("cin", C.c_int),
        ("in_cstride", C.c_int), ("in_coff", C.c_int),
        ("out", C.c_void_p), ("out_dtype", C.c_int), ("hout", C.c_int), ("wout", C.c_int), ("cout", C.c_int),
        ("out_cstride", C.c_int), ("out_coff", C.c_int),
        ("hog", C.c_int), ("wog", C.c_int),
        ("in_sy", C.c_int), ("in_sx", C.c_int), ("out_sy", C.c_int), ("out_sx", C.c_int), ("out_oy", C.c_int), ("out_ox", C.c_int),
        ("ntaps", C.c_int), ("dy", C.c_int * 16), ("dx", C.c_int * 16),
        ("w", C.c_void_p), ("bias", C.c_void_p), ("scale", C.c_void_p), ("shift", C.c_void_p),
        ("res", C.c_void_p), ("res_dtype", C.c_int), ("res_cstride", C.c_int), ("res_coff", C.c_int),
        ("pre_relu", C.c_int), ("post_relu", C.c_int), ("sigmoid", C.c_int), ("d2s_nout", C.c_int),
    ]


class ConvPairDesc(C.Structure):
    """mirror of lavb_conv_pair_desc"""
    _fields_ = [
        ("inp", C.c_void_p), ("out", C.c_void_p), ("res", C.c_void_p),
        ("n", C.c_int), ("h", C.c_int), ("w", C.c_int), ("c", C.c_int), ("dil", C.c_int), ("post_relu", C.c_int),
        ("w1", C.c_void_p), ("bias1", C.c_void_p),
        ("w2", C.c_void_p), ("shift2", C.c_void_p),
    ]


class ControlConfig(C.Structure):
    """mirror of lavb_control_config"""
    _fields_ = [
        ("aim_point", C.c_int * 8), ("speed_ratio", C.c_double * 8),
        ("turn_kp", C.c_double), ("turn_ki", C.c_double), ("turn_kd", C.c_double),
        ("speed_kp", C.c_double), ("speed_ki", C.c_double), ("speed_kd", C.c_double),
        ("turn_n", C.c_int), ("speed_n", C.c_int),
        ("brake_speed", C.c_double), ("clip_delta", C.c_double), ("max_throttle", C.c_double), ("max_speed", C.c_double),
        ("cmd_thresh", C.c_double), ("pixels_per_meter", C.c_double),
    ]


class ViewConfig(C.Structure):
    """mirror of lavb_view_config"""
    _fields_ = [("pixels_per_meter", C.c_double), ("cmd_thresh", C.c_double), ("jet", C.c_ubyte * (259 * 3))]


_SIGS = {
    "lavb_abi_version": (C.c_int, []),
    "lavb_last_error": (C.c_char_p, []),
    "lavb_device_cc": (C.c_int, []),
    "lavb_h16_dtype": (C.c_int, []),
    "lavb_paint": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                             C.c_longlong, C.c_longlong, C.c_longlong, C.c_longlong, C.c_void_p, C.c_int,
                             C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "lavb_paint_batched": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_longlong, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_longlong, C.c_longlong, C.c_longlong, C.c_longlong, C.c_longlong, C.c_void_p, C.c_int,
                                     C.c_void_p, C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_void_p]),
    "lavb_paint_deconv_batched": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_longlong, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                            C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_longlong, C.c_int, C.c_int,
                                            C.c_void_p]),
    "lavb_seg_confusion": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_void_p, C.c_void_p]),
    "lavb_paint_confusion_ints": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "lavb_paint_confusion": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float,
                                       C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    "lavb_stack_jobs": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "lavb_bev_targets": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "lavb_png_decode_gray8": (C.c_int, [C.c_void_p, C.c_longlong, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                        C.c_void_p, C.c_void_p]),
    "lavb_lidar_batch": (C.c_int, [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p, C.c_longlong, C.c_void_p, C.c_int, C.c_void_p,
                                   C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "lavb_lidar_batch_paint": (C.c_int, [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                         C.c_int, C.c_void_p, C.c_void_p]),
    "lavb_det_heatmaps": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float,
                                    C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "lavb_eval_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                  C.c_void_p, C.c_int, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float, C.c_double,
                                  C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p]),
    "lavb_forecast_eval": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                     C.c_void_p, C.c_void_p]),
    "lavb_det_forecast_match": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float,
                                          C.c_float, C.c_float, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p]),
    "lavb_det_box_eval": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_float, C.c_float,
                                    C.c_float, C.c_float, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p]),
    "lavb_plan_safety": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_longlong, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_void_p,
                                   C.c_void_p]),
    "lavb_driving_score": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float,
                                     C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]),
    "lavb_agent_control_state_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "lavb_agent_control": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(ControlConfig), C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p]),
    "lavb_agent_control_dcmd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(ControlConfig), C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p]),
    "lavb_agent_nav_state_bytes": (C.c_size_t, []),
    "lavb_agent_nav_front": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "lavb_agent_nav_update": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "lavb_stack_job_poses": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p,
                                       C.c_void_p]),
    "lavb_agent_view_scratch_bytes": (C.c_size_t, [C.c_int]),
    "lavb_agent_view": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_longlong, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                  C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(ViewConfig), C.c_void_p,
                                  C.c_size_t, C.c_void_p, C.c_void_p]),
    "lavb_roof_filter": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_longlong, C.c_void_p, C.c_longlong, C.c_void_p, C.c_int,
                                   C.c_void_p]),
    "lavb_stack_sweep": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_float, C.c_float, C.c_int, C.c_int, C.c_int,
                                   C.c_void_p, C.c_void_p]),
    "lavb_pillar_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "lavb_pillar_forward": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                      C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_int,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                      C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "lavb_pillar_sorted_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_longlong]),
    "lavb_pillar_forward_sorted": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                             C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_int,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                             C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "lavb_pillar_decorate": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                       C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_int,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "lavb_pillar_scatter_max": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p,
                                          C.c_void_p]),
    "lavb_pillar_scatter_max_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "lavb_conv_taps": (C.c_int, [C.POINTER(ConvDesc), C.c_void_p]),
    "lavb_pool2_affine_relu": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "lavb_rgb_normalize": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]),
    "lavb_convert": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_longlong, C.c_void_p]),
    "lavb_stem7x7s2_u8": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p]),
    "lavb_erf_stem": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "lavb_erf_down16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "lavb_erf_nb16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "lavb_conv_pair_umma": (C.c_int, [C.c_void_p, C.c_void_p]),
    "lavb_maxpool3x3s2_nhwc": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "lavb_det_peaks_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "lavb_det_peaks": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int,
                                 C.c_void_p, C.c_void_p, C.c_void_p]),
    "lavb_crop_bilinear": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                     C.c_int, C.c_void_p, C.c_void_p]),
    "lavb_crop_bilinear_u8": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                        C.c_void_p, C.c_void_p]),
    "lavb_cast_gru": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                C.c_int, C.c_void_p, C.c_void_p]),
    "lavb_conv_pair_set_trace": (C.c_int, [C.c_void_p, C.c_int]),
    "lavb_crop_bilinear_bwd": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                         C.c_void_p, C.c_void_p]),
    "lavb_deconv3x3s2_small": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "lavb_conv_umma": (C.c_int, [C.POINTER(ConvDesc), C.c_void_p]),
    "lavb_conv7x7s2_umma": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p]),
    "lavb_conv3x3_umma": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
}

_lib = None


def exported_symbols():
    """names include/lav_b200.h declares (used by the ABI test)."""
    return sorted(_SIGS)


def lib():
    """Load liblavb200.so once; raise loudly when it is not built (no fallback path exists)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise LavbError(f"{LIB_PATH} is missing — run `python -m lav_b200.build` (or __graft_entry__.build()); "
                            "lav_b200 has no CPU fallback")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(handle, name)          # AttributeError here == header/library drift
            fn.restype = res
            fn.argtypes = args
        if handle.lavb_abi_version() != 3:
            raise LavbError("liblavb200.so ABI version mismatch")
        _lib = handle
    return _lib


def h16_code():
    """element-type code of the 16-bit storage type the library was built with (LAVB_F16 unless -DLAVB_H16_BF16)."""
    return lib().lavb_h16_dtype()


def check(code, what):
    if code != 0:
        raise LavbError(f"{what} failed ({code}): {lib().lavb_last_error().decode()}")
