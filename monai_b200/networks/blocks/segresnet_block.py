"""SegResNet building blocks (monai/networks/blocks/segresnet_block.py:22-96, blocks/upsample.py) on CUDA kernels.

`ResBlock`: norm - act - conv3 - norm - act - conv3 + identity, pre-activation order; GroupNorm statistics come from
`b200_instnorm_stats` on the grouped view, normalise + affine + ReLU is one `b200_norm_act` pass, the final add is fused into a pass
of the same kernel.  `UpSample`: the two modes SegResNet and SegResNetDS use -- "nontrainable" (optional 1x1 preconv, then trilinear, align_corners=False:
`b200_resample_affine` with the matrix src = dst / s - (s - 1) / (2 s) per axis and border clamping, which is what `F.interpolate`
computes) and "deconv" (transposed convolution, kernel = stride = scale, or a given kernel with the reference's padding).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from ... import _kernels as K
from ... import _lib as L
from ..layers.factories import get_act_layer, get_norm_layer
from .acti_norm import norm_act_from_modules
from .convolutions import Convolution, run_conv_module

__all__ = ["ResBlock", "UpSample", "get_conv_layer", "get_upsample_layer"]


def get_conv_layer(spatial_dims: int, in_channels: int, out_channels: int, kernel_size: int = 3, stride: int = 1, bias: bool = False) -> Convolution:
    return Convolution(spatial_dims, in_channels, out_channels, strides=stride, kernel_size=kernel_size, bias=bias, conv_only=True)


class UpSample(nn.Sequential):
    """blocks/upsample.py:26-175: child names as in the reference ("deconv" | optional "preconv" + "upsample_non_trainable").
    `scale_factor` and `kernel_size` are ints or per-axis sequences; with a `kernel_size` the transposed convolution pads by (k - 1) // 2
    and adds output_padding s - 1 - (k - 1) % 2 per axis (upsample.py:94-115), without one its kernel is the scale.  In the
    non-trainable mode a 1x1 "preconv" (with `bias`) maps in_channels to out_channels when they differ."""

    def __init__(self, spatial_dims: int, in_channels: int, out_channels: int | None = None, scale_factor=2, mode: str = "deconv",
                 interp_mode: str = "linear", align_corners: bool | None = False, bias: bool = True, kernel_size=None):
        super().__init__()
        mode = getattr(mode, "value", mode)
        out_channels = out_channels or in_channels
        scale = tuple(int(s) for s in scale_factor) if isinstance(scale_factor, (tuple, list)) else (int(scale_factor),) * spatial_dims
        if len(scale) != spatial_dims:
            raise ValueError(f"scale_factor {scale_factor} does not match spatial_dims {spatial_dims}")
        self.scale, self.spatial_dims = scale, spatial_dims
        if mode == "deconv":
            conv_t = {1: nn.ConvTranspose1d, 2: nn.ConvTranspose2d, 3: nn.ConvTranspose3d}[spatial_dims]
            if not kernel_size:
                k, pad, out_pad = scale, 0, 0
            else:
                k = tuple(kernel_size) if isinstance(kernel_size, (tuple, list)) else (kernel_size,) * spatial_dims
                pad = tuple((i - 1) // 2 for i in k)
                out_pad = tuple(s - 1 - (i - 1) % 2 for i, s in zip(k, scale))
            self.add_module("deconv", conv_t(in_channels, out_channels, kernel_size=k, stride=scale, padding=pad, output_padding=out_pad,
                                             bias=bias))
        elif mode == "nontrainable":
            if str(getattr(interp_mode, "value", interp_mode)).lower() not in ("linear", "trilinear", "bilinear") or align_corners:
                raise NotImplementedError("monai_b200 UpSample: linear interpolation with align_corners=False only")
            if in_channels != out_channels:   # the reference's default pre_conv
                conv = {1: nn.Conv1d, 2: nn.Conv2d, 3: nn.Conv3d}[spatial_dims]
                self.add_module("preconv", conv(in_channels, out_channels, kernel_size=1, bias=bias))
            up = nn.Upsample(scale_factor=scale if isinstance(scale_factor, (tuple, list)) else scale_factor,
                             mode={1: "linear", 2: "bilinear", 3: "trilinear"}[spatial_dims], align_corners=False)
            self.add_module("upsample_non_trainable", up)   # parameter-free container, never called
        else:
            raise NotImplementedError(f"monai_b200 UpSample supports 'deconv' and 'nontrainable', got {mode!r}")

    def forward(self, x: torch.Tensor) -> torch.Tensor:  # type: ignore[override]
        if hasattr(self, "deconv"):
            return run_conv_module(self.deconv, x)
        if hasattr(self, "preconv"):
            x = run_conv_module(self.preconv, x)
        nd = x.dim() - 2
        s3 = (1,) * (3 - nd) + self.scale
        sp3 = (1,) * (3 - nd) + tuple(x.shape[2:])
        out3 = tuple(v * s for v, s in zip(sp3, s3))
        # trilinear, align_corners=False: src = (dst + 0.5) / s - 0.5 per axis, clamped at the border
        diag = [1.0 / s for s in s3]
        off = [-(s - 1) / (2.0 * s) for s in s3]
        mat = [diag[0], 0, 0, off[0], 0, diag[1], 0, off[1], 0, 0, diag[2], off[2]]
        y = K.resample_affine(x.reshape(x.shape[0] * x.shape[1], *sp3), out3, mat, 1, 1, False, out_dtype=x.dtype)
        return y.reshape(x.shape[0], x.shape[1], *out3[3 - nd:])


def get_upsample_layer(spatial_dims: int, in_channels: int, upsample_mode: str = "nontrainable", scale_factor: int = 2) -> UpSample:
    return UpSample(spatial_dims=spatial_dims, in_channels=in_channels, out_channels=in_channels, scale_factor=scale_factor, mode=upsample_mode,
                    interp_mode="linear", align_corners=False)


class ResBlock(nn.Module):
    def __init__(self, spatial_dims: int, in_channels: int, norm, kernel_size: int = 3, act=("RELU", {"inplace": True})) -> None:
        super().__init__()
        if kernel_size % 2 != 1:
            raise AssertionError("kernel_size should be an odd number.")
        self.norm1 = get_norm_layer(name=norm, spatial_dims=spatial_dims, channels=in_channels)
        self.norm2 = get_norm_layer(name=norm, spatial_dims=spatial_dims, channels=in_channels)
        self.act = get_act_layer(act)
        self.conv1 = get_conv_layer(spatial_dims, in_channels=in_channels, out_channels=in_channels, kernel_size=kernel_size)
        self.conv2 = get_conv_layer(spatial_dims, in_channels=in_channels, out_channels=in_channels, kernel_size=kernel_size)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        y = self.conv1(norm_act_from_modules(x, self.norm1, self.act))
        y = self.conv2(norm_act_from_modules(y, self.norm2, self.act))
        return K.norm_act(y, None, res=x, act=L.ACT_NONE)   # y + identity
