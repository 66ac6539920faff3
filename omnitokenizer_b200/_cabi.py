"""ctypes binding of libomnitok_b200.so (the C ABI in include/omnitok_b200.h).

There is no fallback: if the shared library is missing or a call fails, a RuntimeError is
raised.  Tensors are passed as raw device pointers; every call runs on torch's current stream.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int64, c_void_p, POINTER

import torch

_LIB_NAME = "libomnitok_b200.so"
_lib = None

EPI_NONE, EPI_GEGLU, EPI_QKV, EPI_QKV_PLANES = 0, 1, 2, 3
MATH_FP32, MATH_3XTF32, MATH_F16X1, MATH_F16X3 = 0, 1, 2, 3
ABI_VERSION = 2


class LinearHArgs(ctypes.Structure):
    """omt_linear_h_args (include/omnitok_b200.h), field for field."""
    _fields_ = [("a_hi", c_void_p), ("a_lo", c_void_p), ("a_rs", c_void_p), ("a2_rs", c_void_p), ("w_scale", c_float),
                ("a2_hi", c_void_p), ("a2_lo", c_void_p), ("n_split", c_int),
                ("lda", c_int), ("a_seg", c_int), ("a_seg_stride", c_int), ("a_seg_off", c_int),
                ("w_hi", c_void_p), ("w_lo", c_void_p),
                ("c", c_void_p), ("ldc", c_int), ("c_seg", c_int), ("c_seg_stride", c_int), ("c_seg_off", c_int),
                ("u_hi", c_void_p), ("u_lo", c_void_p), ("ldu", c_int),
                ("M", c_int), ("N", c_int), ("K", c_int),
                ("bias", c_void_p), ("residual", c_void_p), ("ldr", c_int),
                ("epilogue", c_int),
                ("q_scale", c_void_p), ("k_scale", c_void_p), ("rope_cos", c_void_p), ("rope_sin", c_void_p),
                ("qk_cols", c_int), ("tokens", c_int),
                ("q_plane_scale", c_float), ("k_plane_scale", c_float), ("vinv", c_void_p),
                ("a_rs_uniform", c_float), ("u_scale", c_float)]


class LpipsTap(ctypes.Structure):
    """omt_lpips_tap (include/omnitok_b200.h): one tap map of omt_lpips_upsample_mean."""
    _fields_ = [("map", c_void_p), ("h", c_int), ("w", c_int)]


def lpips_taps(maps):
    """A host omt_lpips_tap array of (map [P][h][w] tensor or address, h, w) entries, for omt_lpips_upsample_mean.
    The caller keeps the maps alive."""
    return (LpipsTap * len(maps))(*[LpipsTap(_ptr(m), h, w) for m, h, w in maps])


# name -> (restype, argtypes); mirrors include/omnitok_b200.h one to one
SIGNATURES = {
    "omt_abi_version": (c_int, []),
    "omt_last_error": (c_char_p, []),
    "omt_device_info": (c_int, [POINTER(c_int)] * 3),
    "omt_set_option": (c_int, [c_char_p, c_int]),
    "omt_linear": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                           c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "omt_linear2": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                            c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "omt_linear_h": (c_int, [POINTER(LinearHArgs), c_void_p]),
    "omt_linear_h1": (c_int, [POINTER(LinearHArgs), c_void_p]),
    "omt_layernorm": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_float, c_int, c_int,
                              c_int, c_void_p]),
    "omt_layernorm_h": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_int, c_void_p, c_void_p, c_int, c_int, c_float, c_int, c_int, c_int, c_void_p]),
    "omt_patchify_ln": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 8 + [c_float, c_void_p]),
    "omt_patchify_ln_u8": (c_int, [c_void_p] * 9 + [c_int] * 8 + [c_float, c_void_p]),
    "omt_u8_norm_select": (c_int, [c_void_p, c_int, c_int64, c_void_p, c_void_p]),
    "omt_resample_u8": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int,
                                c_void_p, c_void_p]),
    "omt_resample_clips": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_int,
                                   c_int, c_int, c_int, c_void_p, c_void_p]),
    "omt_fvd_preprocess": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p,
                                   c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "omt_fvd_suite_preprocess": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                         c_int64, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "omt_is_preprocess": (c_int, [c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int,
                                  c_int, c_int, c_int, c_void_p, c_void_p]),
    "omt_eval_downsample": (c_int, [c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p,
                                    c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "omt_conv3d": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p]
                   + [c_int] * 13 + [c_void_p, c_int, c_int, c_void_p]),
    "omt_maxpool3d": (c_int, [c_void_p] + [c_int] * 17 + [c_void_p, c_void_p]),
    "omt_i3d_head": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "omt_fid_preprocess": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p,
                                   c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "omt_pool2d": (c_int, [c_void_p] + [c_int] * 13 + [c_void_p, c_int, c_int, c_void_p]),
    "omt_psnr_ssim": (c_int, [c_void_p] * 6 + [c_int] * 4 + [c_void_p] * 4),
    "omt_lpips_input": (c_int, [c_void_p] * 4 + [c_int] * 4 + [c_void_p, c_void_p]),
    "omt_lpips_head": (c_int, [c_void_p] + [c_int] * 5 + [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "omt_lpips_map": (c_int, [c_void_p] + [c_int] * 5 + [c_void_p, c_void_p, c_void_p]),
    "omt_lpips_upsample_mean": (c_int, [c_void_p] + [c_int] * 4 + [c_void_p, c_void_p, c_void_p]),
    "omt_softmax_rows": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "omt_inception_score": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "omt_jpeg_roundtrip_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "omt_unpatchify": (c_int, [c_void_p, c_void_p] + [c_int] * 8 + [c_void_p]),
    "omt_unpatchify_u8": (c_int, [c_void_p, c_void_p] + [c_int] * 8 + [c_float] * 5 + [c_void_p]),
    "omt_peg": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "omt_peg_volume": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 7 + [c_void_p]),
    "omt_peg_volume_varlen": (c_int, [c_void_p] * 6 + [c_int] * 7 + [c_void_p]),
    "omt_qk_prep": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                            c_int, c_void_p]),
    "omt_attn_spatial": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                 c_int, c_int, c_int, c_float, c_void_p]),
    "omt_attn_spatial_h": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                   c_float, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "omt_attn_spatial_h1": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_float, c_void_p, c_void_p,
                                    c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "omt_attn_window": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "omt_attn_temporal": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                  c_int, c_int, c_int, c_int, c_float, c_int, c_void_p]),
    "omt_attn_temporal_varlen": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                         c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_int, c_void_p]),
    "omt_pre_vq": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "omt_vq_search": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "omt_vq_fused": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int,
                             c_void_p, c_void_p, c_void_p]),
    "omt_post_vq": (c_int, [c_void_p] * 8 + [c_int, c_int, c_int, c_void_p]),
}


def lib_path() -> str:
    # OMT_LIB: developer override to A/B-test another build of the same ABI
    return os.environ.get("OMT_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), _LIB_NAME)


def load():
    """Load the shared library (once).  Raises if it has not been built (see __graft_entry__.build)."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise RuntimeError(
            f"{path} not found: the CUDA extension is not built. Run `python -c 'import __graft_entry__ as g; "
            f"g.build()'` (or `make -C omnitokenizer_b200/csrc`). There is no CPU fallback.")
    lib = ctypes.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)     # AttributeError if a declared symbol is missing
        fn.restype = res
        fn.argtypes = args
    if lib.omt_abi_version() != ABI_VERSION:
        raise RuntimeError("libomnitok_b200.so ABI version mismatch")
    _lib = lib
    return lib


def _ptr(t):
    if t is None:
        return None
    if isinstance(t, int):
        return t
    return t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


# kernels launched per entry point (for bench.py's gpu_launches accounting)
KERNELS_PER_CALL = {"omt_u8_norm_select": 2, "omt_jpeg_roundtrip_u8": 2}
launch_count = 0


def call(name: str, *args):
    """Invoke an entry point on torch's current CUDA stream; tensors are converted to pointers."""
    global launch_count
    lib = load()
    conv = [_ptr(a) if (a is None or isinstance(a, torch.Tensor)) else a for a in args]
    rc = getattr(lib, name)(*conv, _stream())
    if rc != 0:                     # a refused call launched nothing
        raise RuntimeError(f"{name} failed ({rc}): {lib.omt_last_error().decode()}")
    launch_count += KERNELS_PER_CALL.get(name, 1)


def linear_h(name="omt_linear_h", **kw):
    """omt_linear_h (or, with name="omt_linear_h1", its single-product form) with keyword fields of omt_linear_h_args
    (tensors -> device pointers; missing fields = 0 / NULL)."""
    global launch_count
    lib = load()
    a = LinearHArgs()
    for k, v in kw.items():
        setattr(a, k, _ptr(v) if (v is None or isinstance(v, torch.Tensor)) else v)
    launch_count += 1
    rc = getattr(lib, name)(ctypes.byref(a), _stream())
    if rc != 0:
        raise RuntimeError(f"{name} failed ({rc}): {lib.omt_last_error().decode()}")


# process-wide kernel selectors and their library defaults (omt_set_option); tests restore these after flipping them
DEFAULT_OPTIONS = {"attn_kernel": 3, "peg_kernel": 4, "f16_bn": 0, "attn_f16_ctas": 2}


def set_option(name: str, value: int):
    lib = load()
    rc = lib.omt_set_option(name.encode(), int(value))
    if rc != 0:
        raise RuntimeError(f"omt_set_option({name}) failed: {lib.omt_last_error().decode()}")


def device_info():
    lib = load()
    a, b, c = c_int(), c_int(), c_int()
    rc = lib.omt_device_info(ctypes.byref(a), ctypes.byref(b), ctypes.byref(c))
    if rc != 0:
        raise RuntimeError(lib.omt_last_error().decode())
    return a.value, b.value, c.value
