"""ctypes binding of libsgb200.so (the C ABI declared in include/sgb200.h).

The product path has no CPU fallback: if the shared library is missing or a call fails, this raises.
PyTorch is used only for device memory and streams; every pointer handed to the library is a raw
``tensor.data_ptr()`` on the current CUDA stream.
"""
import ctypes
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SGB_LIB") or os.path.join(_HERE, "lib", "libsgb200.so")   # SGB_LIB: A/B builds of the same ABI

c_int = ctypes.c_int32
c_i64 = ctypes.c_int64
c_f = ctypes.c_float
c_d = ctypes.c_double
c_p = ctypes.c_void_p


class ConvDesc(ctypes.Structure):
    """Mirror of ``sgb_conv_desc`` (include/sgb200.h)."""
    _fields_ = [
        ("B", c_int), ("H", c_int), ("W", c_int),
        ("Cin", c_int), ("Cout", c_int),
        ("KH", c_int), ("KW", c_int), ("pad_h", c_int), ("pad_w", c_int),
        ("x", c_p), ("x_cstride", c_i64),
        ("w", c_p), ("w_mode", c_int),
        ("alpha", c_f), ("alpha_ptr", c_p),
        ("bias", c_p),
        ("residual", c_p), ("res_cstride", c_i64), ("res_up2", c_int), ("res_after_mask", c_int),
        ("mask", c_p), ("mask_cstride", c_i64),
        ("relu", c_int),
        ("y", c_p), ("y_cstride", c_i64), ("y_fp32", c_int),
        ("Hin", c_int), ("Win", c_int), ("out_sub", c_int),
        ("res_scale", c_f),
        ("mask_bits", c_p), ("relu_bits", c_p),
        ("sm_mode", c_int), ("sm_stats", c_p), ("sm_delta", c_p), ("sm_p", c_p), ("sm_p_cstride", c_i64),
    ]


class WgradDesc(ctypes.Structure):
    """Mirror of ``sgb_wgrad_desc`` (include/sgb200.h)."""
    _fields_ = [
        ("B", c_int), ("H", c_int), ("W", c_int),
        ("Cin", c_int), ("Cout", c_int),
        ("KH", c_int), ("KW", c_int), ("pad_h", c_int), ("pad_w", c_int),
        ("x", c_p), ("x_cstride", c_i64),
        ("dy", c_p), ("dy_cstride", c_i64),
        ("dw", c_p), ("accumulate", c_int), ("per_image", c_int),
        ("dbias", c_p),
    ]


# name -> (restype, argtypes); every symbol declared in include/sgb200.h must appear here (tests check both ways).
SIGNATURES = {
    "sgb_abi_version": (c_int, []),
    "sgb_device_check": (c_int, []),
    "sgb_bind_device": (c_int, [c_int]),
    "sgb_conv_fprop": (c_int, [ctypes.POINTER(ConvDesc), c_p]),
    "sgb_conv_wgrad_fuses_dbias": (c_int, [ctypes.POINTER(WgradDesc)]),
    "sgb_conv_wgrad": (c_int, [ctypes.POINTER(WgradDesc), c_p]),
    "sgb_sn_workspace_floats": (c_i64, [c_int, c_int]),
    "sgb_sn_power_iter": (c_int, [c_p, c_p, c_p, c_p, c_p, c_int, c_int, c_f, c_int, c_p]),
    "sgb_weight_pack": (c_int, [c_p, c_p, c_p, c_p, c_int, c_int, c_int, c_int, c_int, c_int, c_p]),
    "sgb_sn_batch": (c_int, [c_p, c_int, c_p, c_p, c_p, c_f, c_int, c_int, c_int, c_int, c_p]),
    "sgb_sn_backward": (c_int, [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_int, c_int, c_int, c_int, c_int, c_int, c_p]),
    "sgb_sn_backward_batch": (c_int, [c_p, c_int, c_p, c_p, c_p, c_p, c_p, c_int, c_p]),
    "sgb_bn_stats": (c_int, [c_p, c_i64, c_int, c_i64, c_p, c_p, c_p]),
    "sgb_bn_finalize": (c_int, [c_p, c_p, c_f, c_p, c_p, c_f, c_f, c_int, c_int, c_int, c_p, c_p, c_int, c_int,
                                c_p, c_p, c_p, c_p, c_i64, c_p]),
    "sgb_scale_shift_act": (c_int, [c_p, c_int, c_int, c_int, c_int, c_i64, c_p, c_p, c_int, c_int, c_int, c_p, c_i64, c_p]),
    "sgb_bn_bwd_reduce": (c_int, [c_p, c_i64, c_p, c_i64, c_int, c_int, c_int, c_int, c_p, c_p, c_int, c_p, c_p, c_int,
                                  c_int, c_p, c_p, c_p, c_p, c_p]),
    "sgb_bn_bwd_apply": (c_int, [c_p, c_i64, c_p, c_i64, c_int, c_int, c_int, c_int, c_p, c_p, c_int, c_p, c_p, c_p, c_p,
                                 c_f, c_int, c_int, c_int, c_p, c_i64, c_p]),
    "sgb_axpby": (c_int, [c_p, c_i64, c_p, c_i64, c_p, c_i64, c_p, c_i64, c_i64, c_int, c_f, c_p, c_f, c_int, c_p]),
    "sgb_pool2_fwd": (c_int, [c_p, c_i64, c_p, c_i64, c_int, c_int, c_int, c_int, c_int, c_p]),
    "sgb_relu_pool2": (c_int, [c_p, c_i64, c_p, c_i64, c_p, c_i64, c_int, c_int, c_int, c_int, c_p]),
    "sgb_pool2_bwd": (c_int, [c_p, c_i64, c_p, c_i64, c_p, c_i64, c_p, c_i64, c_p, c_i64, c_int, c_int, c_int, c_int,
                              c_int, c_p]),
    "sgb_softmax_rows": (c_int, [c_p, c_p, c_i64, c_int, c_p]),
    "sgb_dhead_fwd": (c_int, [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_int, c_int, c_p, c_p]),
    "sgb_dhead_bwd": (c_int, [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_int, c_int, c_p, c_p, c_p, c_p, c_p]),
    "sgb_rowdot": (c_int, [c_p, c_i64, c_p, c_i64, c_i64, c_int, c_p, c_p]),
    "sgb_conv_softmax_parts": (c_int, [ctypes.POINTER(ConvDesc)]),
    "sgb_softmax_bwd_rows": (c_int, [c_p, c_p, c_p, c_i64, c_int, c_p]),
    "sgb_dot": (c_int, [c_p, c_p, c_i64, c_p, c_p]),
    "sgb_sum_hw": (c_int, [c_p, c_i64, c_int, c_int, c_int, c_int, c_p, c_p]),
    "sgb_sum_hw_bwd": (c_int, [c_p, c_p, c_i64, c_p, c_i64, c_int, c_int, c_int, c_int, c_p]),
    "sgb_img_to_nhwc": (c_int, [c_p, c_p, c_int, c_int, c_int, c_int, c_p]),
    "sgb_nhwc_to_img": (c_int, [c_p, c_int, c_i64, c_p, c_int, c_int, c_int, c_int, c_p]),
    "sgb_img_grad_to_nhwc": (c_int, [c_p, c_p, c_p, c_int, c_int, c_int, c_int, c_p]),
    "sgb_col27": (c_int, [c_p, c_int, c_i64, c_p, c_int, c_int, c_int, c_p]),
    "sgb_col27_bwd": (c_int, [c_p, c_p, c_int, c_int, c_int, c_p]),
    "sgb_pool3x3": (c_int, [c_p, c_i64, c_p, c_i64, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_p]),
    "sgb_zero_stuff2": (c_int, [c_p, c_i64, c_p, c_i64, c_int, c_int, c_int, c_int, c_p]),
    "sgb_quantize_u8": (c_int, [c_p, c_p, c_i64, c_p]),
    "sgb_quantize_resize_normalize": (c_int, [c_p, c_int, c_int, c_int, c_int, c_int, c_p, c_p, c_int, c_p]),
    "sgb_u8_to_img": (c_int, [c_p, c_p, c_p, c_int, c_int, c_int, c_p]),
    "sgb_cast_f32_to_bf16": (c_int, [c_p, c_p, c_i64, c_f, c_p]),
    "sgb_cast_bf16_to_f32": (c_int, [c_p, c_p, c_i64, c_p]),
    "sgb_adam_ema_step": (c_int, [c_p, c_p, c_p, c_p, c_i64, c_f, c_f, c_f, c_f, c_int, c_p, c_p, c_f, c_f, c_p]),
    "sgb_ema_lerp": (c_int, [c_p, c_p, c_i64, c_f, c_p]),
    "sgb_gp_interpolate": (c_int, [c_p, c_p, c_p, c_p, c_int, c_i64, c_p]),
    "sgb_gp_sumsq": (c_int, [c_p, c_p, c_int, c_i64, c_p]),
    "sgb_gp_seed": (c_int, [c_p, c_p, c_p, c_int, c_i64, c_p]),
    "sgb_gp_seed_max": (c_int, [c_p, c_p, c_p, c_p, c_int, c_i64, c_p]),
    "sgb_dra_std": (c_int, [c_p, c_i64, c_p, c_p, c_p]),
    "sgb_dra_perturb": (c_int, [c_p, c_p, c_p, c_p, c_p, c_int, c_i64, c_p]),
    "sgb_clamp": (c_int, [c_p, c_i64, c_f, c_p]),
    "sgb_sample_mean": (c_int, [c_p, c_int, c_i64, c_p, c_p]),
    "sgb_diffaug_fwd": (c_int, [c_p, c_p, c_p, c_p, c_int, c_int, c_int, c_int, c_int, c_int, c_p]),
    "sgb_diffaug_bwd": (c_int, [c_p, c_p, c_p, c_p, c_int, c_int, c_int, c_int, c_int, c_int, c_p]),
    "sgb_cr_aug": (c_int, [c_p, c_p, c_p, c_p, c_p, c_int, c_int, c_int, c_int, c_p]),
    "sgb_feat_moments_accumulate": (c_int, [c_p, c_int, c_int, c_p, c_p, c_p]),
    "sgb_feat_moments_finalize": (c_int, [c_p, c_p, c_d, c_int, c_p, c_p, c_p]),
    "sgb_prdc_radii": (c_int, [c_p, c_int, c_int, c_int, c_p, c_p, c_p]),
    "sgb_prdc_cross": (c_int, [c_p, c_p, c_p, c_p, c_p, c_p, c_int, c_int, c_int, c_p, c_p, c_p, c_p]),
    "sgb_bn_tangent_bwd_reduce": (c_int, [c_p, c_i64, c_p, c_i64, c_p, c_i64, c_i64, c_int, c_p, c_p, c_p, c_p]),
    "sgb_bn_tangent_bwd_apply": (c_int, [c_p, c_i64, c_p, c_i64, c_p, c_i64, c_i64, c_int, c_p, c_p, c_p, c_p, c_f, c_int,
                                         c_p, c_i64, c_p, c_i64, c_p]),
}

_ERR = {1: "SGB_ERR_ARG (invalid argument)", 2: "SGB_ERR_CUDA (CUDA failure)", 3: "SGB_ERR_UNSUPPORTED"}

_lib = None


def load():
    """Load libsgb200.so and bind every entry point. Raises if the library is absent (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "libsgb200.so not found at %s: build it with `python pytorch-studiogan_b200/build.py` "
            "(the sgb200 product path has no CPU / PyTorch fallback)" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def stream_ptr():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def check(rc, what):
    if rc != 0:
        raise RuntimeError("libsgb200: %s failed with %s" % (what, _ERR.get(rc, rc)))


def ptr(t):
    """Raw device pointer of a tensor (or NULL for None)."""
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())


LAUNCHES = [0]  # number of library entry-point calls (each launches >= 1 kernel); bench.py reports the delta per step


_tls = threading.local()


# Optional per-call accounting (bench.py's roofline block / profiles): when PROFILE["enabled"], every library call is
# bracketed by CUDA events on the launching stream and logged as (tag, algorithmic FLOPs, start, stop).
PROFILE = {"enabled": False, "events": []}


def call(name, *args, tag=None, flops=0.0, nbytes=0.0):
    lib = load()
    if getattr(_tls, "device", None) is None:
        # first library call on this host thread (e.g. an autograd worker): bind the thread to torch's current device
        dev = torch.cuda.current_device()
        check(lib.sgb_bind_device(dev), "sgb_bind_device")
        _tls.device = dev
    if PROFILE["enabled"]:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = getattr(lib, name)(*args)
        e1.record()
        PROFILE["events"].append((tag or name, flops, e0, e1, nbytes))
    else:
        rc = getattr(lib, name)(*args)
    LAUNCHES[0] += 1
    check(rc, name)
