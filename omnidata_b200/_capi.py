"""ctypes binding of include/omnidata_b200.h (the C-ABI shared library).

There is deliberately no fallback: if the library is missing or a call fails, this raises.
Only plain pointers and integers cross the boundary; torch is used by callers for device memory
and streams, never passed through.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

LIB_PATH = Path(__file__).resolve().parent / "lib" / "libomnidata_b200.so"

ODB_MAX_VIEWS = 4
ODB_MAX_TAPS = 9
ACT_NONE, ACT_RELU, ACT_GELU = 0, 1, 2
DTYPE_BF16, DTYPE_F32 = 0, 1


class OdbError(RuntimeError):
    pass


class View(C.Structure):
    _fields_ = [
        ("ptr", C.c_void_p),
        ("c", C.c_int32), ("w", C.c_int32), ("h", C.c_int32), ("b", C.c_int32),
        ("sx", C.c_int64), ("sy", C.c_int64), ("sb", C.c_int64),
    ]


class ConvGemmDesc(C.Structure):
    _fields_ = [
        ("num_views", C.c_int32),
        ("views", View * ODB_MAX_VIEWS),
        ("num_taps", C.c_int32),
        ("tap_view", C.c_int8 * ODB_MAX_TAPS),
        ("tap_dx", C.c_int8 * ODB_MAX_TAPS),
        ("tap_dy", C.c_int8 * ODB_MAX_TAPS),
        ("weight", C.c_void_p),
        ("n", C.c_int32),
        ("out", View),
        ("out2", View),
        ("bias", C.c_void_p),
        ("bias_sb", C.c_int64),
        ("residual", View),
        ("act", C.c_int32),
        ("tile_w", C.c_int32), ("tile_h", C.c_int32),
        ("block_n", C.c_int32),
        ("cta_pair", C.c_int32),
        ("halo", C.c_int32),
        ("head_w", C.c_void_p),
        ("head_b", C.c_void_p),
        ("head_c", C.c_int32),
        ("head_relu", C.c_int32),
        ("head_out", C.c_void_p),
        ("gn_partial", C.c_void_p),
        ("gn_groups", C.c_int32),
        ("epilogue", C.c_int32),
        ("in_dtype", C.c_int32),
        ("out_dtype", C.c_int32),
        ("out2_act", C.c_int32),
    ]


class PackItem(C.Structure):
    _fields_ = [("w", C.c_void_p), ("fwd", C.c_void_p), ("bwd", C.c_void_p), ("n", C.c_int32), ("c", C.c_int32),
                ("taps", C.c_int32), ("n_pad", C.c_int32), ("c_pad", C.c_int32), ("standardize", C.c_int32),
                ("first_block", C.c_int32), ("first_tile", C.c_int32)]


class UnpackItem(C.Structure):
    _fields_ = [("gp", C.c_void_p), ("w", C.c_void_p), ("dw", C.c_void_p), ("n", C.c_int32), ("c", C.c_int32),
                ("taps", C.c_int32), ("c_pad", C.c_int32), ("standardize", C.c_int32), ("first_block", C.c_int32),
                ("pad0", C.c_int32), ("pad1", C.c_int32)]


class WgradDesc(C.Structure):
    _fields_ = [
        ("num_views", C.c_int32),
        ("views", View * ODB_MAX_VIEWS),
        ("num_taps", C.c_int32),
        ("tap_view", C.c_int8 * ODB_MAX_TAPS),
        ("tap_dx", C.c_int8 * ODB_MAX_TAPS),
        ("tap_dy", C.c_int8 * ODB_MAX_TAPS),
        ("dy", View),
        ("n", C.c_int32),
        ("out", C.c_void_p),
        ("workspace", C.c_void_p),
        ("workspace_bytes", C.c_int64),
        ("accumulate", C.c_int32),
        ("dtype", C.c_int32),
    ]


_SIGNATURES = {
    "odb_conv_gemm": (C.c_int, [C.POINTER(ConvGemmDesc), C.c_void_p]),
    "odb_conv_gemm_plan": (C.c_int, [C.POINTER(ConvGemmDesc), C.POINTER(C.c_int32)]),
    "odb_groupnorm_finalize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_double,
                                         C.c_float, C.c_void_p]),
    "odb_layernorm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                C.c_float, C.c_int32, C.c_int32, C.c_void_p]),
    "odb_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                C.c_void_p]),
    "odb_attention_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                    C.c_void_p]),
    "odb_head_tail_f32": (C.c_int, [C.c_void_p] * 5 + [C.c_int32] * 5 + [C.c_void_p]),
    "odb_groupnorm_scratch_bytes": (C.c_int64, [C.c_int32] * 4),
    "odb_groupnorm_stats": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_void_p]),
    "odb_groupnorm_apply": (C.c_int, [C.c_void_p] * 9 + [C.c_int32] * 6 + [C.c_void_p]),
    "odb_stem_gn_relu_maxpool": (C.c_int, [C.c_void_p] * 5 + [C.c_int32] * 6 + [C.c_void_p]),
    "odb_stem_im2col": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                  C.c_void_p]),
    "odb_patchify": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                               C.c_void_p]),
    "odb_upsample2x_add": (C.c_int, [C.c_void_p] * 4 + [C.c_int32] * 5 + [C.c_void_p]),
    "odb_write_cls_row": (C.c_int, [C.c_void_p] * 3 + [C.c_int32] * 4 + [C.c_void_p]),
    "odb_readout_cls_bias": (C.c_int, [C.c_void_p] * 4 + [C.c_int32] * 4 + [C.c_void_p]),
    "odb_cast_f32_bf16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "odb_conv_wgrad_workspace_bytes": (C.c_int64, [C.POINTER(WgradDesc)]),
    "odb_conv_wgrad": (C.c_int, [C.POINTER(WgradDesc), C.c_void_p]),
    "odb_attention_bwd_workspace_bytes": (C.c_int64, [C.c_int32] * 4),
    "odb_attention_bwd": (C.c_int, [C.c_void_p] * 6 + [C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_int32,
                                                       C.c_void_p]),
    "odb_mask_add": (C.c_int, [C.c_void_p] * 4 + [C.c_int64, C.c_int32, C.c_void_p]),
    "odb_gelu_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]),
    "odb_gelu_bwd": (C.c_int, [C.c_void_p] * 3 + [C.c_int64, C.c_int32, C.c_void_p]),
    "odb_colsum_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int64, C.c_int32]),
    "odb_colsum": (C.c_int, [C.c_void_p] * 3 + [C.c_int32, C.c_int64, C.c_int32, C.c_int64, C.c_int64, C.c_int32, C.c_int32,
                                                C.c_void_p]),
    "odb_reduce_partials": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_void_p]),
    "odb_layernorm_bwd_workspace_bytes": (C.c_int64, [C.c_int32]),
    "odb_layernorm_bwd": (C.c_int, [C.c_void_p] * 10 + [C.c_int64, C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_void_p]),
    "odb_groupnorm_bwd_workspace_bytes": (C.c_int64, [C.c_int32] * 4),
    "odb_groupnorm_bwd": (C.c_int, [C.c_void_p] * 9 + [C.c_int32] * 6 + [C.c_void_p]),
    "odb_upsample2x_bwd": (C.c_int, [C.c_void_p, C.c_void_p] + [C.c_int32] * 5 + [C.c_void_p]),
    "odb_stem_pool_bwd": (C.c_int, [C.c_void_p] * 6 + [C.c_int32] * 6 + [C.c_void_p]),
    "odb_stem_input_grad": (C.c_int, [C.c_void_p] * 3 + [C.c_int32] * 5 + [C.c_void_p]),
    "odb_patch_input_grad": (C.c_int, [C.c_void_p] * 2 + [C.c_int32] * 5 + [C.c_void_p]),
    "odb_pos_embed_resize_bwd": (C.c_int, [C.c_void_p] * 2 + [C.c_int32] * 3 + [C.c_void_p]),
    "odb_head_tail_fwd": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_int32] * 6 + [C.c_void_p]),
    "odb_head_tail_bwd_workspace_bytes": (C.c_int64, [C.c_int32]),
    "odb_head_tail_bwd": (C.c_int, [C.c_void_p] * 3 + [C.c_int32] + [C.c_void_p] * 5 + [C.c_int32] * 7 + [C.c_void_p]),
    "odb_add_cast": (C.c_int, [C.c_void_p] * 4 + [C.c_int64, C.c_int32, C.c_void_p]),
    "odb_clamp01": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "odb_clamp01_bwd": (C.c_int, [C.c_void_p] * 4 + [C.c_int64, C.c_void_p]),
    "odb_pack_weight": (C.c_int, [C.c_void_p] * 3 + [C.c_int32] * 6 + [C.c_float, C.c_int32, C.c_void_p]),
    "odb_pack_weights_multi": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_void_p]),
    "odb_unpack_wgrads_multi": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_void_p]),
    "odb_unpack_wgrad": (C.c_int, [C.c_void_p] * 3 + [C.c_int32] * 5 + [C.c_float, C.c_void_p]),
    "odb_make_valid_mask": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "odb_midas_loss_workspace_bytes": (C.c_int64, [C.c_int32]),
    "odb_midas_loss_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                     C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "odb_vnl_loss_fwd": (C.c_int, [C.c_void_p] * 5 + [C.c_int32] * 4 + [C.c_float] * 3 + [C.c_int32, C.c_void_p,
                                                                                        C.c_void_p, C.c_void_p]),
    "odb_midas_loss_bwd_workspace_bytes": (C.c_int64, [C.c_int32]),
    "odb_midas_loss_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                     C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "odb_vnl_loss_bwd": (C.c_int, [C.c_void_p] * 5 + [C.c_int32] * 4 + [C.c_float] * 2 + [C.c_int32, C.c_void_p, C.c_float,
                                                                                   C.c_void_p, C.c_void_p, C.c_void_p,
                                                                                   C.c_void_p]),
    "odb_normal_loss_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_void_p, C.c_void_p, C.c_void_p]),
    "odb_grad_norm_workspace_bytes": (C.c_int64, []),
    "odb_clip_grad_norm": (C.c_int, [C.c_void_p, C.c_int64, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "odb_adam_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_float,
                                C.c_float, C.c_float, C.c_float, C.c_int64, C.c_void_p, C.c_void_p]),
    "odb_adam_step_scalars": (C.c_int, [C.c_float, C.c_float, C.c_float, C.c_int64, C.c_void_p]),
    "odb_clip_grad_norm_segments": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_void_p,
                                              C.c_void_p, C.c_void_p]),
    "odb_adam_step_segments": (C.c_int, [C.c_void_p] * 5 + [C.c_int32, C.c_int64, C.c_void_p] + [C.c_float] * 4 +
                               [C.c_int64, C.c_void_p, C.c_void_p]),
    "odb_refocus_quantiles": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_void_p,
                                        C.c_void_p]),
    "odb_refocus_compose": (C.c_int, [C.c_void_p] * 4 + [C.c_int32] * 4 + [C.c_void_p] * 5),
    "odb_normal_loss_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "odb_fill_zero": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p]),
    "odb_pil_resize_crop_to_tensor": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_void_p,
                                                C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                                C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float,
                                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "odb_bicubic_resize_f32": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                         C.c_void_p, C.c_void_p]),
    "odb_f32_chw_to_u8_hwc": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "odb_abi_version": (C.c_int, []),
    "odb_last_error": (C.c_char_p, []),
    "odb_launch_count": (C.c_int64, []),
    "odb_debug_conv_trace": (C.c_int, [C.c_void_p]),
}

ABI_VERSION = 4        # include/omnidata_b200.h: ODB_ABI_VERSION (descriptor layouts this module mirrors)

_lib = None


def exported_symbols():
    return sorted(_SIGNATURES)


def lib():
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise OdbError(
                f"{LIB_PATH} is missing: build it with `python -m omnidata_b200.build` "
                "(there is no CPU / eager fallback)")
        _lib = C.CDLL(str(LIB_PATH))
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(_lib, name)  # raises AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        if _lib.odb_abi_version() != ABI_VERSION:
            raise OdbError(f"{LIB_PATH} has ABI version {_lib.odb_abi_version()}, this package expects {ABI_VERSION}: "
                           "rebuild with `python -m omnidata_b200.build`")
    return _lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = lib().odb_last_error().decode(errors="replace")
        raise OdbError(f"{what or 'omnidata_b200'} failed (status {rc}): {msg}")


def on_tensor_device(fn):
    """Decorator for host entry points that enqueue C-ABI work with `torch.cuda.current_stream()`: makes the device of
    the first CUDA tensor argument (or of an object argument with a CUDA `.device`) current for the duration of the
    call, so that kernels, kernel attributes and streams all belong to the device the data lives on."""
    import functools

    @functools.wraps(fn)
    def wrapper(*args, **kw):
        import torch
        dev = None
        for a in list(args) + list(kw.values()):
            if isinstance(a, torch.Tensor):
                if a.is_cuda:
                    dev = a.device
                    break
                continue
            d = getattr(a, "device", None)
            if isinstance(d, torch.device) and d.type == "cuda":
                dev = d
                break
        if dev is None or dev.index is None or dev.index == torch.cuda.current_device():
            return fn(*args, **kw)
        with torch.cuda.device(dev):
            return fn(*args, **kw)
    return wrapper


def launch_count() -> int:
    return int(lib().odb_launch_count())
