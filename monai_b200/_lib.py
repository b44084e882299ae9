"""ctypes binding of the C ABI declared in include/monai_b200.h.

The CUDA library is the product: there is no CPU or PyTorch fallback behind these calls.  If the shared object is
missing (or fails to load) every kernel entry point raises `RuntimeError` -- loudly, by design.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import torch

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "lib" / "libmonai_b200.so"

ABI_VERSION = 2
DT_F32, DT_F16 = 0, 1
_DT = {torch.float32: DT_F32, torch.float16: DT_F16}

ACT_NONE, ACT_LEAKY, ACT_PRELU, ACT_RELU, ACT_GELU = 0, 1, 2, 3, 4
PAD_ZEROS, PAD_BORDER, PAD_REFLECTION = 0, 1, 2
INTERP_NEAREST, INTERP_LINEAR = 0, 1

i32, i64, f32, vp = C.c_int, C.c_longlong, C.c_float, C.c_void_p


class BlendDesc(C.Structure):
    _fields_ = [
        ("preds", vp), ("pred_dtype", i32), ("pred_stride", i64 * 5), ("win_begin", i32), ("win_end", i32),
        ("B", i32), ("C", i32), ("D", i32), ("H", i32), ("W", i32), ("rd", i32), ("rh", i32), ("rw", i32),
        ("starts_d", vp), ("nd", i32), ("starts_h", vp), ("nh", i32), ("starts_w", vp), ("nw", i32),
        ("gd", vp), ("gh", vp), ("gw", vp), ("clamp_min", f32), ("wmap", vp),
        ("out", vp), ("out_dtype", i32), ("acc", vp), ("box", i32 * 4), ("starts_w_align", i32),
        ("max_cover", i32), ("slot_map", vp), ("n_slots", i32), ("resample", C.POINTER(C.c_double)),
        ("out_D", i32), ("out_H", i32), ("out_W", i32), ("resample_interp", i32), ("resample_pad", i32),
    ]


class ConvDesc(C.Structure):
    _fields_ = [
        ("N", i32), ("Cin", i32), ("Cout", i32), ("Di", i32), ("Hi", i32), ("Wi", i32), ("Do", i32), ("Ho", i32),
        ("Wo", i32), ("kd", i32), ("kh", i32), ("kw", i32), ("sd", i32), ("sh", i32), ("sw", i32), ("pd", i32),
        ("ph", i32), ("pw", i32), ("transposed", i32), ("in_dtype", i32), ("out_dtype", i32),
        ("in_stride_n", i64), ("out_stride_n", i64),
    ]


class ConvTcDesc(C.Structure):
    _fields_ = [
        ("N", i32), ("Cin", i32), ("Cout", i32), ("D", i32), ("H", i32), ("W", i32),
        ("in_ctot", i32), ("in_coff", i32), ("out_ctot", i32), ("out_coff", i32),
        ("in_stats", vp), ("in_eps", f32), ("in_act", i32), ("in_slope", f32),
        ("res_w", vp), ("res_y", vp), ("res_ctot", i32), ("res_coff", i32), ("res_stats", vp),
    ]


class ConvGatherDesc(C.Structure):
    _fields_ = [(n, i32) for n in (
        "N", "Cin", "Cout", "Di", "Hi", "Wi", "Do", "Ho", "Wo", "k", "stride", "pad", "transposed", "in_ctot", "in_coff",
        "out_ctot", "out_coff", "out_layout", "out_dtype")]


class GemmTcDesc(C.Structure):
    _fields_ = [
        ("Nb", i32), ("S", i32), ("K", i32), ("N", i32), ("in_ctot", i32), ("in_coff", i32), ("out_ctot", i32),
        ("out_coff", i32), ("res_ctot", i32), ("res_coff", i32), ("S_out", i64), ("mode", i32), ("act", i32),
        ("D", i32), ("H", i32), ("W", i32),
    ]


# name -> (restype, argtypes); must list every symbol include/monai_b200.h declares (tests check this).
SIGNATURES = {
    "b200_abi_version": (i32, []),
    "b200_last_error": (C.c_char_p, []),
    "b200_launch_count": (i64, []),
    "b200_sw_gather": (i32, [vp, i32, vp, i32, vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, vp]),
    "b200_sw_blend": (i32, [C.POINTER(BlendDesc), i32, vp]),
    "b200_conv3d_direct": (i32, [C.POINTER(ConvDesc), vp, vp, vp, vp, vp]),
    "b200_instnorm_stats_workspace_bytes": (i64, [i32, i32, i64]),
    "b200_instnorm_stats": (i32, [vp, i32, i32, i32, i64, i64, vp, vp, vp]),
    "b200_norm_act": (i32, [vp, i32, i32, i32, i64, i64, vp, f32, vp, vp, vp, i64, vp, i32, f32, vp, i32, vp, i64, vp]),
    "b200_maxpool3d_2": (i32, [vp, i32, i32, i32, i32, i32, vp, vp]),
    "b200_copy_channels": (i32, [vp, i32, i32, i32, i32, i32, i32, vp, i32, i32, i32, i32, i32, vp]),
    "b200_resample_affine": (i32, [vp, i32, i32, i32, i32, i32, vp, i32, i32, i32, i32, C.POINTER(C.c_double), i32, i32, i32, vp]),
    "b200_grid_pull": (i32, [vp, i32, i32, i32, i32, i32, i32, vp, i32, i64, i64, i64, i32, i32, i32, C.POINTER(C.c_double), C.POINTER(C.c_double),
                       C.POINTER(C.c_int), C.POINTER(C.c_int), i32, i32, vp, i32, vp]),
    "b200_grid_push": (i32, [vp, i32, i32, i32, i32, i32, i32, vp, i32, i64, i64, i64, i32, i32, i32, C.POINTER(C.c_double), C.POINTER(C.c_double),
                       C.POINTER(C.c_int), C.POINTER(C.c_int), i32, vp, vp]),
    "b200_grid_grad": (i32, [vp, i32, i32, i32, i32, i32, i32, vp, i32, i64, i64, i64, i32, i32, i32, C.POINTER(C.c_double), C.POINTER(C.c_double),
                       C.POINTER(C.c_int), C.POINTER(C.c_int), i32, vp, i32, vp]),
    "b200_separable_filter3d": (i32, [vp, i32, i32, i32, i32, i32, vp, i32, vp, i32, vp, i32, vp, vp, vp]),
    "b200_pack_nc8": (i32, [vp, i32, i32, i32, i64, vp, i32, i32, vp]),
    "b200_unpack_nc8": (i32, [vp, i32, i32, i32, i32, i64, vp, i32, vp]),
    "b200_conv3x3x3_tc_weight_bytes": (i64, [i32, i32]),
    "b200_conv3x3x3_tc_pack_weight": (i32, [vp, i32, i32, vp, vp]),
    "b200_conv3x3x3_tc_workspace_bytes": (i64, [C.POINTER(ConvTcDesc)]),
    "b200_conv3x3x3_tc": (i32, [C.POINTER(ConvTcDesc), vp, vp, vp, vp, vp, vp, vp]),
    "b200_conv3x3x3_tc_affine": (i32, [C.POINTER(ConvTcDesc), vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "b200_conv_gather_tc_weight_bytes": (i64, [C.POINTER(ConvGatherDesc)]),
    "b200_conv_gather_tc_pack_weight": (i32, [C.POINTER(ConvGatherDesc), vp, vp, vp]),
    "b200_conv_gather_tc_workspace_bytes": (i64, [C.POINTER(ConvGatherDesc)]),
    "b200_conv_gather_tc": (i32, [C.POINTER(ConvGatherDesc), vp, vp, vp, vp, vp, vp, vp]),
    "b200_convt3s2_head_nc8": (i32, [vp, i32, i32, i32, i32, i32, i32, i32, vp, vp, i32, vp, i32, vp]),
    "b200_gemm_tc_weight_bytes": (i64, [i32, i32]),
    "b200_gemm_tc_pack_weight": (i32, [vp, i32, i32, i64, i64, vp, vp]),
    "b200_gemm_tc_workspace_bytes": (i64, [C.POINTER(GemmTcDesc)]),
    "b200_gemm_tc": (i32, [C.POINTER(GemmTcDesc), vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "b200_mlp_fused_tc": (i32, [vp, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, f32, vp, i32, vp]),
    "b200_layernorm_cf": (i32, [vp, i32, i32, i32, i64, vp, vp, f32, vp, vp]),
    "b200_patchify": (i32, [vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, vp, vp]),
    "b200_mhsa_cf": (i32, [vp, i32, i32, i32, i32, i64, f32, i32, vp, vp, vp, vp]),
    "b200_gather_cf": (i32, [vp, i32, i32, i32, i64, vp, i64, vp, vp]),
    "b200_layernorm_nc8": (i32, [vp, i32, i32, i64, vp, i64, vp, vp, f32, vp, vp]),
    "b200_patch_merge_ln_nc8": (i32, [vp, i32, i32, i32, i32, i32, vp, vp, f32, i32, vp, vp]),
    "b200_window_attention_nc8": (i32, [vp, i32, i32, i32, i32, i32, f32, vp, i32, i32, i32, vp, vp, vp]),
    "b200_conv_cin1_nc8_workspace_bytes": (i64, [i32] * 8),
    "b200_conv_cin1_nc8": (i32, [vp, i32, i32, i32, i32, i32, vp, vp, i32, i32, i32, i32, vp, i32, i32, vp, vp, vp]),
    "b200_conv_cin1_tc_workspace_bytes": (i64, [i32] * 8),
    "b200_conv_cin1_tc": (i32, [vp, i32, i32, i32, i32, i32, vp, vp, i32, i32, i32, i32, vp, i32, i32, vp, vp, vp]),
    "b200_window_attention_tc_bias_bytes": (i64, [i32, i32, i32]),
    "b200_window_attention_tc_pack_bias": (i32, [vp, i32, i32, i32, i32, i32, vp, i32, vp, vp]),
    "b200_window_attention_tc": (i32, [vp, i32, i32, i32, i32, i32, vp, vp, i32, vp, vp]),
    "b200_mhsa_tc": (i32, [vp, i32, i32, i32, i64, vp, vp]),
    "b200_patch_accumulate": (i32, [vp, i32, i64, i32, i32, i32, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp]),
    "b200_add_f32": (i32, [vp, vp, i64, vp]),
    "b200_patch_finalize": (i32, [vp, vp, i32, i64, vp]),
    "b200_channel_post": (i32, [vp, i32, i32, i64, i32, f32, i32, vp, i32, vp]),
    "b200_head_conv_nc8": (i32, [vp, i32, i32, i64, vp, vp, i32, vp, i32, vp]),
    "b200_head_conv_norm_nc8": (i32, [vp, i32, i32, i64, vp, f32, vp, i32, i32, vp, f32, vp, vp, i32, vp, i32, vp]),
    "b200_head_conv_norm_affine_nc8": (i32, [vp, i32, i32, i64, vp, f32, vp, i32, i32, vp, f32, vp, vp, i32, vp, i32, vp, vp, vp]),
    "b200_norm_act_nc8": (i32, [vp, i32, i32, i32, i32, i64, vp, f32, vp, i32, i32, vp, i32, f32, vp, i32, i32, vp]),
    "b200_norm_act_affine_nc8": (i32, [vp, i32, i32, i32, i32, i64, vp, f32, vp, i32, i32, vp, i32, f32, vp, i32, i32, vp, vp, vp, vp, vp]),
    "b200_norm_act_cin1res_nc8": (i32, [vp, i32, i32, i32, i32, i64, vp, f32, vp, vp, vp, i32, f32, vp, i32, i32, vp]),
}

_lib = None
_load_error: str | None = None


def load(required: bool = True):
    """Load libmonai_b200.so (once).  With required=True a missing library is a hard error."""
    global _lib, _load_error
    if _lib is None and _load_error is None:
        try:
            lib = C.CDLL(str(LIB_PATH))
            for name, (res, args) in SIGNATURES.items():
                fn = getattr(lib, name)
                fn.restype, fn.argtypes = res, args
            if lib.b200_abi_version() != ABI_VERSION:
                raise OSError(f"ABI version mismatch: {lib.b200_abi_version()}")
            _lib = lib
        except (OSError, AttributeError) as e:  # pragma: no cover - exercised only on broken installs
            _load_error = f"{type(e).__name__}: {e}"
    if _lib is None and required:
        raise RuntimeError(
            f"monai_b200: the CUDA library {LIB_PATH} is not available ({_load_error}). "
            "Build it with `python -m monai_b200._build`; there is no CPU fallback."
        )
    return _lib


def available() -> bool:
    return load(required=False) is not None


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().b200_last_error().decode("utf-8", "replace")
        if rc == 1:
            raise ValueError(f"monai_b200 {what}: {msg}")
        raise RuntimeError(f"monai_b200 {what}: {msg}")


def dt(t: torch.Tensor | torch.dtype) -> int:
    d = t if isinstance(t, torch.dtype) else t.dtype
    try:
        return _DT[d]
    except KeyError:
        raise TypeError(f"monai_b200 kernels take float32 or float16 tensors, got {d}") from None


def ptr(t: torch.Tensor | None) -> int | None:
    return None if t is None else t.data_ptr()


_last_stream_device: torch.device | None = None


def stream_ptr(device: torch.device | None = None) -> int:
    """Handle of torch's current stream on `device`; the device is remembered so that the launch that consumes the handle
    (monai_b200._kernels._call evaluates it as its last argument) runs with that device current."""
    global _last_stream_device
    _last_stream_device = device if device is None or isinstance(device, torch.device) else torch.device(device)
    return torch.cuda.current_stream(device).cuda_stream


def take_stream_device() -> torch.device | None:
    global _last_stream_device
    d, _last_stream_device = _last_stream_device, None
    return d


def require_cuda(*tensors: torch.Tensor) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("monai_b200 kernels need CUDA tensors (no CPU fallback exists in this package)")


_replayed_launches = 0


def add_replayed_launches(n: int) -> None:
    """Kernels re-launched by a CUDA-graph replay (the C counter only sees them once, at capture time)."""
    global _replayed_launches
    _replayed_launches += int(n)


def launch_count() -> int:
    """monai_b200 kernels launched by this process: direct C-ABI launches + launches replayed from captured graphs."""
    lib = load(required=False)
    return (int(lib.b200_launch_count()) if lib is not None else 0) + _replayed_launches


if os.environ.get("MONAI_B200_EAGER_LOAD"):
    load()
