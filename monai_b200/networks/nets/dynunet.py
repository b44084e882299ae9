"""DynUNet (monai/networks/nets/dynunet.py:24-380; nnU-Net style) behind the reference's constructor, module tree and state_dict
keys, with every convolution / normalisation / activation on the CUDA kernels of this package (SURVEY.md §8 row f4: "other
predictors used with sliding window").

Topology: input block, n down blocks, bottleneck, n + 1 up blocks (transposed convolution + skip concat + conv block), 1x1 output
block; anisotropic kernels / strides per level; optional residual blocks.  As in the reference the blocks are registered twice -- in
their flat containers (`input_block`, `downsamples`, `bottleneck`, `upsamples`) and in the recursive `skip_layers` chain -- so a
reference checkpoint loads key for key.  Inference only: deep-supervision heads are constructed (their parameters load) but only the
full-resolution output is produced, which is what the reference returns in eval mode.

Two forwards, chosen from the input and the configuration (DESIGN.md §8.4):
  * fp16 CUDA input and an eligible configuration (`_tc_ok`: 3-D, every kernel 3, strides [1, 2, 2, ...], upsample kernels equal
    to the strides, filters % 16 == 0, InstanceNorm with or without affine and without running statistics, LeakyReLU with a
    slope in [0, 1], out_channels <= 16; dropout inactive at call time): `_forward_tc`, the whole network on fp16 channel-blocked
    (NC8) buffers and Hopper tensor cores -- `b200_conv3x3x3_tc` for the stride-1 3x3x3 convolutions (the previous norm +
    LeakyReLU applied on the operand load), `b200_conv_gather_tc` for the stride-2 ones, `b200_gemm_tc` for the transposed
    convolutions, the affine output head `b200_head_conv_norm_affine_nc8` -- replayed from a CUDA graph per input shape;
  * everything else (fp32 input, anisotropic plans, other norms): `_forward_generic`, the fp32-faithful generic kernels.
"""
from __future__ import annotations

from typing import Sequence

import torch
import torch.nn as nn

from ... import _kernels as K
from .._graph import GraphedForward
from ..blocks.dynunet_block import UnetBasicBlock, UnetOutBlock, UnetResBlock, UnetUpBlock
from ._tc_blocks import TcBlocks, _Cache

__all__ = ["DynUNet", "DynUnet", "Dynunet"]


class DynUNetSkipLayer(nn.Module):
    """One level of the U (dynunet.py:24-53): down block, everything below, up block fed with the level's skip."""

    def __init__(self, index: int, downsample: nn.Module, upsample: nn.Module, next_layer: nn.Module, heads=None, super_head: nn.Module | None = None):
        super().__init__()
        self.downsample = downsample
        self.next_layer = next_layer
        self.upsample = upsample
        self.super_head = super_head
        self.heads = heads
        self.index = index

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        down = self.downsample(x)
        return self.upsample(self.next_layer(down), down)   # supervision heads only matter in training mode


def _all(v, want: int) -> bool:
    """An int or a per-axis sequence that equals `want` on every axis."""
    return all(int(i) == want for i in (v if isinstance(v, (list, tuple)) else [v]))


class DynUNet(TcBlocks, GraphedForward, nn.Module):
    def __init__(
        self,
        spatial_dims: int,
        in_channels: int,
        out_channels: int,
        kernel_size: Sequence[Sequence[int] | int],
        strides: Sequence[Sequence[int] | int],
        upsample_kernel_size: Sequence[Sequence[int] | int],
        filters: Sequence[int] | None = None,
        dropout=None,
        norm_name=("INSTANCE", {"affine": True}),
        act_name=("leakyrelu", {"inplace": True, "negative_slope": 0.01}),
        deep_supervision: bool = False,
        deep_supr_num: int = 1,
        res_block: bool = False,
        trans_bias: bool = False,
    ) -> None:
        super().__init__()
        self.spatial_dims, self.in_channels, self.out_channels = spatial_dims, in_channels, out_channels
        self.kernel_size, self.strides, self.upsample_kernel_size = kernel_size, strides, upsample_kernel_size
        self.norm_name, self.act_name, self.dropout = norm_name, act_name, dropout
        self.conv_block = UnetResBlock if res_block else UnetBasicBlock
        self.trans_bias = trans_bias
        if filters is not None:
            if len(filters) < len(strides):
                raise ValueError("length of filters should be no less than the length of strides.")
            self.filters = list(filters[: len(strides)])
        else:  # the nnU-Net rule: 32, 64, ... capped at 320 (3-D) / 512 (2-D)
            self.filters = [min(2 ** (5 + i), 320 if spatial_dims == 3 else 512) for i in range(len(strides))]
        f, ks, st = self.filters, kernel_size, strides
        common = dict(norm_name=norm_name, act_name=act_name, dropout=dropout)
        self.input_block = self.conv_block(spatial_dims, in_channels, f[0], ks[0], st[0], **common)
        self.downsamples = nn.ModuleList(
            [self.conv_block(spatial_dims, cin, cout, k, s, **common) for cin, cout, k, s in zip(f[:-2], f[1:-1], ks[1:-1], st[1:-1])])
        self.bottleneck = self.conv_block(spatial_dims, f[-2], f[-1], ks[-1], st[-1], **common)
        self.upsamples = nn.ModuleList([
            UnetUpBlock(spatial_dims, cin, cout, k, s, upsample_kernel_size=uk, trans_bias=trans_bias, **common)
            for cin, cout, k, s, uk in zip(f[1:][::-1], f[:-1][::-1], ks[1:][::-1], st[1:][::-1], upsample_kernel_size[::-1])])
        self.output_block = UnetOutBlock(spatial_dims, f[0], out_channels, dropout=dropout)
        self.deep_supervision, self.deep_supr_num = deep_supervision, deep_supr_num
        self.heads = [torch.rand(1)] * deep_supr_num
        if deep_supervision:
            self.deep_supervision_heads = nn.ModuleList([UnetOutBlock(spatial_dims, f[i + 1], out_channels, dropout=dropout) for i in range(deep_supr_num)])
            n_up = len(strides) - 1
            if deep_supr_num >= n_up:
                raise ValueError("deep_supr_num should be less than the number of up sample layers.")
            if deep_supr_num < 1:
                raise ValueError("deep_supr_num should be larger than 0.")
        self.apply(self.initialize_weights)
        self._check_kernel_stride()

        downs, ups = [self.input_block] + list(self.downsamples), list(self.upsamples)[::-1]
        heads = list(self.deep_supervision_heads) if deep_supervision else None

        def chain(index: int, downs, ups, heads):
            if len(downs) != len(ups):
                raise ValueError(f"{len(downs)} != {len(ups)}")
            if not downs:
                return self.bottleneck
            head, rest = None, heads
            if heads is not None and index > 0:   # the input block never gets a supervision head
                head, rest = (heads[0], heads[1:]) if heads else (None, [])
            nxt = chain(index + 1, downs[1:], ups[1:], rest)
            if head is not None:
                return DynUNetSkipLayer(index, downs[0], ups[0], nxt, heads=self.heads, super_head=head)
            return DynUNetSkipLayer(index, downs[0], ups[0], nxt)

        self.skip_layers = chain(0, downs, ups, heads)
        self._tc_ok = self._tc_eligible()
        self._cache = _Cache()
        self._graph_init()  # the ~100 launches of one tensor-core forward are captured into a CUDA graph per input shape

    def _tc_eligible(self) -> bool:
        """Whether `_forward_tc` implements this configuration (isotropic 3x3x3 / stride-2 plans, InstanceNorm, LeakyReLU)."""
        st, up = self.strides, self.upsample_kernel_size
        if self.spatial_dims != 3 or self.out_channels > 16 or any(f % 16 for f in self.filters):
            return False
        if not all(_all(k, 3) for k in self.kernel_size) or not _all(st[0], 1) or not all(_all(s, 2) for s in st[1:]):
            return False
        if len(up) != len(st) - 1 or not all(_all(u, 2) for u in up):
            return False
        blocks = [self.input_block, *self.downsamples, self.bottleneck, *(u.conv_block for u in self.upsamples)]
        for b in blocks:
            for name in ("norm1", "norm2", "norm3"):
                nm = getattr(b, name, None)
                if nm is not None and (not isinstance(nm, nn.InstanceNorm3d) or nm.track_running_stats):
                    return False
            if not isinstance(b.lrelu, nn.LeakyReLU) or not 0.0 <= b.lrelu.negative_slope <= 1.0:
                return False
            if getattr(b, "norm3", None) is not None and b.norm3.eps != b.norm2.eps:   # one eps per norm_act launch
                return False
        return True

    def _dropout_active(self) -> bool:
        return self.training and any(isinstance(m, nn.modules.dropout._DropoutNd) and m.p > 0 for m in self.modules())

    def _check_kernel_stride(self) -> None:
        ks, st = self.kernel_size, self.strides
        if len(ks) != len(st) or len(ks) < 3:
            raise ValueError("length of kernel_size and strides should be the same, and no less than 3.")
        for idx, (k, s) in enumerate(zip(ks, st)):
            if not isinstance(k, int) and len(k) != self.spatial_dims:
                raise ValueError(f"length of kernel_size in block {idx} should be the same as spatial_dims.")
            if not isinstance(s, int) and len(s) != self.spatial_dims:
                raise ValueError(f"length of stride in block {idx} should be the same as spatial_dims.")

    @staticmethod
    def initialize_weights(module: nn.Module) -> None:
        if isinstance(module, (nn.Conv3d, nn.Conv2d, nn.ConvTranspose3d, nn.ConvTranspose2d)):
            module.weight = nn.init.kaiming_normal_(module.weight, a=0.01)
            if module.bias is not None:
                module.bias = nn.init.constant_(module.bias, 0)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not (self._tc_ok and x.is_cuda and x.dtype == torch.float16) or self._dropout_active():
            return self._forward_generic(x)
        if self.training and self.deep_supervision:
            raise RuntimeError("monai_b200.DynUNet is inference-only: call .eval() (deep-supervision outputs exist in training mode only)")
        self._check_tc_input(x)
        if self._graph_ok():
            return self._forward_graphed(x, self._forward_tc)
        return self._forward_tc(x)

    def _forward_generic(self, x: torch.Tensor) -> torch.Tensor:
        if self.training and self.deep_supervision:
            raise RuntimeError("monai_b200.DynUNet is inference-only: call .eval() (deep-supervision outputs exist in training mode only)")
        return self.output_block(self.skip_layers(x))

    # ------------------------------------------------------------------------------------------- tensor-core path
    def _check_tc_input(self, x: torch.Tensor) -> None:
        div = 2 ** (len(self.strides) - 1)
        if x.dim() != 5 or x.shape[1] != self.in_channels:
            raise ValueError(f"DynUNet expects an [N, {self.in_channels}, D, H, W] input, got {tuple(x.shape)}")
        if any(int(s) % div for s in x.shape[2:]):
            raise ValueError(f"DynUNet with {len(self.strides)} levels needs spatial sizes divisible by {div}, got {tuple(x.shape[2:])}")

    def _forward_tc(self, x_in: torch.Tensor) -> torch.Tensor:
        """DynUNet.forward (dynunet.py:265-274, eval mode) on fp16 NC8 buffers and tensor cores; the output is fp16.

        Walks the flat containers.  Level i < last owns one concat buffer of 2 f_i channels: its down block (the input block at
        level 0) writes its normalised output into channels [f_i, 2 f_i) -- the skip, and the input of the next down block --
        and the matching up block's transposed convolution later writes channels [0, f_i)."""
        self._check_tc_input(x_in)
        with torch.no_grad():
            x_in = x_in.contiguous()
            n, dev, f = x_in.shape[0], x_in.device, self.filters
            nl = len(f)
            sp0 = tuple(int(s) for s in x_in.shape[2:])
            cats = [K.NC8(n, 2 * f[i], tuple(s >> i for s in sp0), dev) for i in range(nl - 1)]
            block = self._res_block if self.conv_block is UnetResBlock else self._basic_block

            if self.in_channels == 1:   # the raw NCDHW window feeds the single-channel stem kernels
                block(None, 1, 0, self.input_block, "in", out=cats[0], out_coff=f[0], x_in_raw=x_in)
            else:                       # several channels: zero-padded to 16 and packed
                cp = (self.in_channels + 15) // 16 * 16
                xz = torch.zeros((n, cp, *sp0), device=dev, dtype=torch.float16)
                K.copy_channels(x_in, xz, 0)
                block(K.pack_nc8(xz), cp, 0, self.input_block, "in", out=cats[0], out_coff=f[0], cin_pad=cp)
            for j, down in enumerate(self.downsamples):
                block(cats[j], f[j], f[j], down, f"d{j}", out=cats[j + 1], out_coff=f[j + 1], stride=2)
            cur = block(cats[nl - 2], f[nl - 2], f[nl - 2], self.bottleneck, "bn", stride=2)

            for u, up in enumerate(self.upsamples):
                lvl = nl - 2 - u
                tc = up.transp_conv.conv
                K.gemm_tc(cur, self._wup(tc, f"u{u}.t"), f[lvl + 1], 8 * f[lvl], bias=tc.bias, out=cats[lvl], out_coff=0, mode=2)
                if lvl > 0:
                    cur = self._basic_block(cats[lvl], 2 * f[lvl], 0, up.conv_block, f"u{u}")
            # the last up block's norm2 + LeakyReLU is applied by the output head on its operand load
            y2, st2 = self._basic_block(cats[0], 2 * f[0], 0, up.conv_block, f"u{u}", defer_tail=True)
            eps, g, b = self._norm(up.conv_block.norm2)
            oc = self.output_block.conv.conv
            return K.head_conv_norm_nc8(y2, st2, None, 0, None, self._slope(up.conv_block), eps, oc.weight, oc.bias, out_dtype=x_in.dtype,
                                        gamma=g, beta=b)


DynUnet = Dynunet = DynUNet
