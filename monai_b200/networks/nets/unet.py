"""`UNet` (monai/networks/nets/unet.py:27-301): recursive Sequential(down, SkipConnection(sub), up).

Constructor arguments, module tree and state_dict keys are those of the reference (`model.0.conv.weight`,
`model.1.submodule...`, `model.2.conv.weight`, `...adn.A.weight`), so reference checkpoints load unchanged.
Every layer executes on the monai_b200 CUDA kernels; activations follow the input dtype (fp16 or fp32) and all
accumulation is fp32.
"""
from __future__ import annotations

import warnings
from collections.abc import Sequence

import torch
import torch.nn as nn

from ... import _kernels as K
from ... import _lib as L
from ..blocks.convolutions import Convolution, ResidualUnit
from ..layers.simplelayers import SkipConnection
from ._tc_blocks import TcNet

__all__ = ["UNet", "Unet"]


class UNet(TcNet, nn.Module):
    def __init__(
        self,
        spatial_dims: int,
        in_channels: int,
        out_channels: int,
        channels: Sequence[int],
        strides: Sequence[int],
        kernel_size: Sequence[int] | int = 3,
        up_kernel_size: Sequence[int] | int = 3,
        num_res_units: int = 0,
        act="PRELU",
        norm="INSTANCE",
        dropout: float = 0.0,
        bias: bool = True,
        adn_ordering: str = "NDA",
    ) -> None:
        super().__init__()
        if len(channels) < 2:
            raise ValueError("the length of `channels` should be no less than 2.")
        delta = len(strides) - (len(channels) - 1)
        if delta < 0:
            raise ValueError("the length of `strides` should equal to `len(channels) - 1`.")
        if delta > 0:
            warnings.warn(f"`len(strides) > len(channels) - 1`, the last {delta} values of strides will not be used.")
        if isinstance(kernel_size, Sequence) and len(kernel_size) != spatial_dims:
            raise ValueError("the length of `kernel_size` should equal to `dimensions`.")
        if isinstance(up_kernel_size, Sequence) and len(up_kernel_size) != spatial_dims:
            raise ValueError("the length of `up_kernel_size` should equal to `dimensions`.")
        self.dimensions = spatial_dims
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.channels = channels
        self.strides = strides
        self.kernel_size = kernel_size
        self.up_kernel_size = up_kernel_size
        self.num_res_units = num_res_units
        self.act = act
        self.norm = norm
        self.dropout = dropout
        self.bias = bias
        self.adn_ordering = adn_ordering
        self.model = self._level(in_channels, out_channels, list(channels), list(strides), True)
        self._tc_setup()
        # eager: a graph replay copies the input and the output (130 MB per batch of 25 96^3 windows), which costs more than the
        # ~17 launches of this forward take to issue
        self._graph_enabled = False

    # -- builders (same construction order as the reference so that seeded initialisation matches) -------------
    def _level(self, inc: int, outc: int, channels: list[int], strides: list[int], is_top: bool) -> nn.Module:
        c, s = channels[0], strides[0]
        if len(channels) > 2:
            sub = self._level(c, c, channels[1:], strides[1:], False)
            upc = c * 2
        else:
            sub = self._get_bottom_layer(c, channels[1])
            upc = c + channels[1]
        down = self._get_down_layer(inc, c, s, is_top)
        up = self._get_up_layer(upc, outc, s, is_top)
        return nn.Sequential(down, SkipConnection(sub), up)

    def _common(self) -> dict:
        return dict(act=self.act, norm=self.norm, dropout=self.dropout, bias=self.bias, adn_ordering=self.adn_ordering)

    def _get_down_layer(self, in_channels: int, out_channels: int, strides: int, is_top: bool) -> nn.Module:
        if self.num_res_units > 0:
            return ResidualUnit(
                self.dimensions, in_channels, out_channels, strides=strides, kernel_size=self.kernel_size,
                subunits=self.num_res_units, **self._common(),
            )
        return Convolution(self.dimensions, in_channels, out_channels, strides=strides, kernel_size=self.kernel_size, **self._common())

    def _get_bottom_layer(self, in_channels: int, out_channels: int) -> nn.Module:
        return self._get_down_layer(in_channels, out_channels, 1, False)

    def _get_up_layer(self, in_channels: int, out_channels: int, strides: int, is_top: bool) -> nn.Module:
        conv: nn.Module = Convolution(
            self.dimensions, in_channels, out_channels, strides=strides, kernel_size=self.up_kernel_size,
            conv_only=is_top and self.num_res_units == 0, is_transposed=True, **self._common(),
        )
        if self.num_res_units > 0:
            ru = ResidualUnit(
                self.dimensions, out_channels, out_channels, strides=1, kernel_size=self.kernel_size, subunits=1,
                last_conv_only=is_top, **self._common(),
            )
            conv = nn.Sequential(conv, ru)
        return conv

    # ------------------------------------------------------------------------------------------ tensor-core path
    def _check_input(self, x: torch.Tensor) -> None:
        if not x.is_cuda:
            raise RuntimeError("monai_b200.UNet runs on CUDA tensors only (there is no CPU fallback)")

    def _use_tc(self, x: torch.Tensor) -> bool:
        """fp16 3-D single-channel input, plain conv levels (no residual units), InstanceNorm (non-affine) + PReLU(1) /
        LeakyReLU / ReLU in "NDA" order, 3x3x3 kernels, strides 1 or 2, inner channel counts that are multiples of 16."""
        if x.dtype != torch.float16 or self.dimensions != 3 or self.num_res_units != 0 or self.in_channels != 1:
            return False
        if self.kernel_size != 3 or self.up_kernel_size != 3 or self.adn_ordering.upper() != "NDA" or self.dropout not in (0, 0.0, None):
            return False
        if any(c % 16 for c in self.channels) or any(s not in (1, 2) for s in self.strides[: len(self.channels) - 1]):
            return False
        for m in self.modules():
            if isinstance(m, (nn.InstanceNorm3d,)) and (m.affine or m.track_running_stats):
                return False
            if isinstance(m, (nn.BatchNorm3d, nn.GroupNorm, nn.LayerNorm)):
                return False
            if isinstance(m, nn.PReLU) and m.weight.numel() != 1:
                return False
            # every conv block on this path applies InstanceNorm (with the module's eps) and then the activation: a block
            # without a norm (norm=None), with another ordering or with dropout takes the generic path instead
            if isinstance(m, Convolution) and m is not self.model[2]:   # model[2]: the top transposed conv (conv only)
                adn = getattr(m, "adn", None)
                if adn is None or not isinstance(getattr(adn, "N", None), nn.InstanceNorm3d):
                    return False
                drop = getattr(adn, "D", None)   # Dropout(p=0) / eval-mode dropout is the identity; an active one is not on this path
                if drop is not None and getattr(drop, "p", 0.0) > 0 and drop.training:
                    return False
        return all(isinstance(m, (nn.PReLU, nn.LeakyReLU, nn.ReLU)) for m in self.modules() if type(m).__module__.startswith("torch.nn.modules.activation"))

    def _act_of(self, conv: Convolution):
        act = getattr(conv.adn, "A", None)
        if isinstance(act, nn.PReLU):
            return L.ACT_LEAKY, self._cache.get(("slope", id(act)), [act.weight], lambda: float(act.weight.detach().float().item()))
        if isinstance(act, nn.LeakyReLU):
            return L.ACT_LEAKY, float(act.negative_slope)
        if isinstance(act, nn.ReLU):
            return L.ACT_RELU, 0.0
        return L.ACT_NONE, 0.0

    def _tc_conv(self, conv: Convolution, x, cin: int, in_coff: int, out, out_coff: int, raw=None):
        """Convolution block (conv + InstanceNorm + activation) on tensor cores; result goes to out[:, out_coff:...]."""
        m = conv.conv
        transposed = isinstance(m, nn.ConvTranspose3d)
        cout = m.out_channels
        k, s, p = m.kernel_size[0], m.stride[0], m.padding[0]
        if raw is not None:
            y, st = K.conv_cin1_nc8(raw, m.weight, m.bias, k, s, p, want_stats=True)
        else:
            pw = self._cache.get(("w", id(m)), [m.weight], lambda: K.conv_gather_tc_pack_weight(m.weight, k, s, p, transposed))
            y, st = K.conv_gather_tc(x, pw, cin, cout, k, s, p, transposed=transposed, output_padding=m.output_padding[0] if transposed else 0,
                                     in_coff=in_coff, bias=m.bias, want_stats=True)
        act, slope = self._act_of(conv)
        if out is None:
            out, out_coff = y, 0
        K.norm_act_nc8(y, cout, st, act=act, slope=slope, out=out, out_coff=out_coff, eps=float(conv.adn.N.eps))
        return out

    def _tc_level(self, block: nn.Sequential, x, cin: int, raw, top: bool, out, out_coff: int, out_dtype):
        down, skip, up = block[0], block[1], block[2]
        sub = skip.submodule
        c = down.conv.out_channels
        bottom = isinstance(sub, Convolution)
        c_sub = sub.conv.out_channels if bottom else sub[2].conv.out_channels
        # `down` output and the sub-network's output share one buffer: torch.cat([x, sub(x)], 1) without a copy
        sp_in = raw.shape[2:] if raw is not None else x.sp
        st = down.conv.stride[0]
        sp = tuple((int(s) + 2 - 3) // st + 1 for s in sp_in)
        n = raw.shape[0] if raw is not None else x.N
        cat = K.NC8(n, c + c_sub, sp, (raw if raw is not None else x.buf).device)
        self._tc_conv(down, x, cin, 0, cat, 0, raw=raw)
        if bottom:
            self._tc_conv(sub, cat, c, 0, cat, c)
        else:
            self._tc_level(sub, cat, c, None, False, cat, c, None)
        upm = up.conv
        if top:  # conv only: logits straight to NCDHW
            if upm.out_channels <= 4 and upm.kernel_size[0] == 3 and upm.stride[0] == 2 and upm.padding[0] == 1 and upm.output_padding[0] == 1:
                return K.convt3s2_head_nc8(cat, c + c_sub, upm.weight, upm.bias, out_dtype=out_dtype)
            pw = self._cache.get(("w", id(upm)), [upm.weight], lambda: K.conv_gather_tc_pack_weight(upm.weight, upm.kernel_size[0], upm.stride[0], upm.padding[0], True))
            y, _ = K.conv_gather_tc(cat, pw, c + c_sub, upm.out_channels, upm.kernel_size[0], upm.stride[0], upm.padding[0], transposed=True,
                                    output_padding=upm.output_padding[0], bias=upm.bias, ncdhw_dtype=out_dtype)
            return y
        return self._tc_conv(up, cat, c + c_sub, 0, out, out_coff)

    def _forward_tc(self, x: torch.Tensor) -> torch.Tensor:
        with torch.no_grad():
            return self._tc_level(self.model, None, 1, x.contiguous(), True, None, 0, x.dtype)

    def _forward_generic(self, x: torch.Tensor) -> torch.Tensor:
        with torch.no_grad():
            return self.model(x.contiguous())


Unet = UNet
