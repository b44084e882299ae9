"""SegResNet (monai/networks/nets/segresnet.py:30-200; Myronenko 2018, without the VAE branch) behind the reference's constructor,
module tree and state_dict keys, on the CUDA kernels of this package (SURVEY.md §8 row f4).

convInit, then per level [stride-2 convolution] + pre-activation ResBlocks (GroupNorm by default); the decoder halves the channels
with a 1x1 convolution, upsamples x2 (trilinear or transposed convolution), adds the encoder feature and runs ResBlocks; final
norm - act - 1x1 convolution.  Inference only (dropout is the identity).

Two forwards, chosen from the input and the configuration (DESIGN.md §8.4):
  * fp16 CUDA input and an eligible configuration (`_tc_ok`: 3-D, init_filters % 16 == 0, GroupNorm (affine or not) or
    InstanceNorm3d without running statistics, ReLU or LeakyReLU with a slope in [0, 1], "nontrainable" or "deconv" upsampling;
    dropout inactive at call time): `_forward_tc`, the whole network on fp16 channel-blocked (NC8) buffers and Hopper tensor
    cores -- every 3x3x3 convolution on `b200_conv3x3x3_tc` with the previous GroupNorm + activation applied on its operand load
    (`b200_group_stats` folds the per-channel sums of the conv epilogues into group sums), the residual add in conv2's epilogue
    (the `add` of `b200_conv3x3x3_tc`), the stride-2 convolutions on `b200_conv_gather_tc`, the 1x1x1 / transposed convolutions on
    `b200_gemm_tc`, upsample + skip add in one pass (`b200_upsample_add_nc8`) -- replayed from a CUDA graph per input shape;
  * everything else (fp32 input, 2-D, init_filters % 16 != 0, BatchNorm, other activations): `_forward_generic`, the
    fp32-faithful generic kernels.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from ... import _kernels as K
from ... import _lib as L
from ..blocks.acti_norm import norm_act_from_modules
from ..blocks.segresnet_block import ResBlock, get_conv_layer, get_upsample_layer
from ..layers.factories import get_act_layer, get_norm_layer
from ._tc_blocks import TcNet

__all__ = ["SegResNet"]


class SegResNet(TcNet, nn.Module):
    def __init__(
        self,
        spatial_dims: int = 3,
        init_filters: int = 8,
        in_channels: int = 1,
        out_channels: int = 2,
        dropout_prob: float | None = None,
        act=("RELU", {"inplace": True}),
        norm=("GROUP", {"num_groups": 8}),
        norm_name: str = "",
        num_groups: int = 8,
        use_conv_final: bool = True,
        blocks_down: tuple = (1, 2, 2, 4),
        blocks_up: tuple = (1, 1, 1),
        upsample_mode: str = "nontrainable",
    ):
        super().__init__()
        if spatial_dims not in (2, 3):
            raise ValueError("`spatial_dims` can only be 2 or 3.")
        self.spatial_dims, self.init_filters, self.in_channels = spatial_dims, init_filters, in_channels
        self.blocks_down, self.blocks_up, self.dropout_prob = blocks_down, blocks_up, dropout_prob
        self.act = act
        self.act_mod = get_act_layer(act)
        if norm_name:
            if norm_name.lower() != "group":
                raise ValueError(f"Deprecating option 'norm_name={norm_name}', please use 'norm' instead.")
            norm = ("group", {"num_groups": num_groups})
        self.norm = norm
        self.upsample_mode = str(getattr(upsample_mode, "value", upsample_mode))
        self.use_conv_final = use_conv_final
        self.convInit = get_conv_layer(spatial_dims, in_channels, init_filters)
        self.down_layers = nn.ModuleList()
        for i, n_blocks in enumerate(blocks_down):
            ch = init_filters * 2**i
            pre = get_conv_layer(spatial_dims, ch // 2, ch, stride=2) if i > 0 else nn.Identity()
            self.down_layers.append(nn.Sequential(pre, *[ResBlock(spatial_dims, ch, norm=norm, act=act) for _ in range(n_blocks)]))
        self.up_layers, self.up_samples = nn.ModuleList(), nn.ModuleList()
        n_up = len(blocks_up)
        for i in range(n_up):
            ch = init_filters * 2 ** (n_up - i)
            self.up_layers.append(nn.Sequential(*[ResBlock(spatial_dims, ch // 2, norm=norm, act=act) for _ in range(blocks_up[i])]))
            self.up_samples.append(nn.Sequential(get_conv_layer(spatial_dims, ch, ch // 2, kernel_size=1),
                                                 get_upsample_layer(spatial_dims, ch // 2, upsample_mode=self.upsample_mode)))
        self.conv_final = nn.Sequential(get_norm_layer(name=norm, spatial_dims=spatial_dims, channels=init_filters), self.act_mod,
                                        get_conv_layer(spatial_dims, init_filters, out_channels, kernel_size=1, bias=True))
        if dropout_prob is not None:
            self.dropout = (nn.Dropout, nn.Dropout2d, nn.Dropout3d)[spatial_dims - 1](dropout_prob)
        self._tc_ok = self._tc_eligible()
        self._tc_setup()

    def _tc_eligible(self) -> bool:
        """Whether `_forward_tc` implements this configuration (3-D, init_filters % 16 == 0, GroupNorm / InstanceNorm, ReLU /
        LeakyReLU, trilinear or transposed-convolution upsampling)."""
        if self.spatial_dims != 3 or self.init_filters % 16 or self.upsample_mode not in ("nontrainable", "deconv"):
            return False
        if len(self.blocks_up) != len(self.blocks_down) - 1:   # the decoder ends at level 0 (the reference needs it too)
            return False
        blocks = [m for m in self.modules() if isinstance(m, ResBlock)]
        norms = [self.conv_final[0]] + [n for b in blocks for n in (b.norm1, b.norm2)]
        acts = [self.conv_final[1]] + [b.act for b in blocks]
        for nm in norms:
            if not (isinstance(nm, nn.GroupNorm) or (isinstance(nm, nn.InstanceNorm3d) and not nm.track_running_stats)):
                return False
        for a in acts:
            if not (type(a) is nn.ReLU or (type(a) is nn.LeakyReLU and 0.0 <= a.negative_slope <= 1.0)):
                return False
        return True

    def _dropout_active(self) -> bool:
        return bool(self.training and self.dropout_prob)

    def encode(self, x: torch.Tensor):
        if self.training and self.dropout_prob:
            raise RuntimeError("monai_b200.SegResNet is inference-only: call .eval()")
        x = self.convInit(x)
        down_x = []
        for down in self.down_layers:
            for m in down:
                if not isinstance(m, nn.Identity):
                    x = m(x)
            down_x.append(x)
        return x, down_x

    def decode(self, x: torch.Tensor, down_x) -> torch.Tensor:
        for i, (up, upl) in enumerate(zip(self.up_samples, self.up_layers)):
            x = K.norm_act(up[1](up[0](x)), None, res=down_x[i + 1], act=L.ACT_NONE)   # up(x) + skip
            for m in upl:
                x = m(x)
        if self.use_conv_final:
            x = self.conv_final[2](norm_act_from_modules(x, self.conv_final[0], self.conv_final[1]))
        return x

    def _use_tc(self, x: torch.Tensor) -> bool:
        return super()._use_tc(x) and not self._dropout_active()

    def _forward_generic(self, x: torch.Tensor) -> torch.Tensor:
        x, down_x = self.encode(x)
        down_x.reverse()
        return self.decode(x, down_x)

    # ------------------------------------------------------------------------------------------- tensor-core path
    def _check_tc_input(self, x: torch.Tensor) -> None:
        self._check_levels(x, len(self.blocks_down))

    @staticmethod
    def _norm_tc(norm: nn.Module, stats: torch.Tensor, N: int, C: int):
        """(statistics, eps, gamma, beta) for the NC8 norm consumers: a GroupNorm's per-channel sums are folded into group sums."""
        eps, g, b = TcNet._norm(norm)
        groups = norm.num_groups if isinstance(norm, nn.GroupNorm) else C
        return K.group_stats(stats, N, C, groups), eps, g, b

    @staticmethod
    def _act_tc(act: nn.Module) -> tuple[int, float]:
        if isinstance(act, nn.LeakyReLU):
            return L.ACT_LEAKY, float(act.negative_slope)
        return L.ACT_RELU, 0.0

    def _res_block_tc(self, x: K.NC8, st: torch.Tensor, blk: ResBlock, key: str):
        """ResBlock.forward (segresnet_block.py: x + conv2(act(norm2(conv1(act(norm1(x))))))) in two launches: each norm + act runs
        on its convolution's operand load, and the identity is added in conv2's epilogue, whose statistics are those of the sum."""
        C, act = x.C, self._act_tc(blk.act)
        s1, e1, g1, b1 = self._norm_tc(blk.norm1, st, x.N, C)
        y1, st1 = K.conv3x3x3_tc(x, self._w3(blk.conv1.conv, key + ".c1"), C, C, bias=blk.conv1.conv.bias, want_stats=True,
                                 in_norm=(s1, e1, *act), in_affine=(g1, b1))
        s2, e2, g2, b2 = self._norm_tc(blk.norm2, st1, x.N, C)
        return K.conv3x3x3_tc(y1, self._w3(blk.conv2.conv, key + ".c2"), C, C, bias=blk.conv2.conv.bias, want_stats=True,
                              in_norm=(s2, e2, *act), in_affine=(g2, b2), add=(x, 0))

    def _forward_tc(self, x_in: torch.Tensor) -> torch.Tensor:
        """SegResNet.forward (segresnet.py encode + decode, eval mode) on fp16 NC8 buffers and tensor cores; the output is fp16.

        Every tensor travels with its per-(n, channel) {sum, sumsq}, produced by the epilogue of the launch that wrote it, so each
        GroupNorm costs one tiny `group_stats` launch and is applied on the load of the convolution (or head) that consumes it."""
        with torch.no_grad():
            x_in = x_in.contiguous()
            n, f0 = x_in.shape[0], self.init_filters
            ci = self.convInit.conv
            if self.in_channels == 1:   # the raw NCDHW window feeds the single-channel stem kernel
                x, st = K.conv_cin1_nc8(x_in, ci.weight, ci.bias, 3, 1, 1, want_stats=True)
            else:
                xp, cp = self._pack_input(x_in)
                x, st = K.conv3x3x3_tc(xp, self._w3(ci, "init", cp), cp, f0, bias=ci.bias, want_stats=True)
            # dropout after convInit is the identity in eval mode (forward routes active dropout to the generic path)

            down = []
            for i, layer in enumerate(self.down_layers):
                mods = list(layer)
                if i > 0:
                    pre = mods[0].conv
                    x, st = K.conv_gather_tc(x, self._wg(pre, f"d{i}.pre", 3, 2, 1), pre.in_channels, pre.out_channels, 3, 2, 1,
                                             bias=pre.bias, want_stats=True)
                for j, blk in enumerate(mods[1:]):
                    x, st = self._res_block_tc(x, st, blk, f"d{i}.{j}")
                down.append(x)
            down.reverse()

            for i, (up, upl) in enumerate(zip(self.up_samples, self.up_layers)):
                pc = up[0].conv                                 # 1x1x1, ch -> ch / 2, at the low resolution
                half = pc.out_channels
                z, _ = K.gemm_tc(x, self._wlin(pc.weight, f"u{i}.pre"), pc.in_channels, half, bias=pc.bias)
                if self.upsample_mode == "deconv":              # ConvTranspose3d k2 s2, then the skip add
                    dc = up[1].deconv
                    z, _ = K.gemm_tc(z, self._wup(dc, f"u{i}.up"), half, 8 * half, bias=dc.bias, mode=2)
                    x, st = K.upsample_add_nc8(z, half, 1, down[i + 1], want_stats=True)
                else:                                           # trilinear x2 and the skip add in one pass
                    x, st = K.upsample_add_nc8(z, half, 2, down[i + 1], want_stats=True)
                for j, blk in enumerate(upl):
                    x, st = self._res_block_tc(x, st, blk, f"u{i}.{j}")

            if not self.use_conv_final:
                return K.unpack_nc8(x, dtype=x_in.dtype)
            norm, act, conv = self.conv_final[0], self.conv_final[1], self.conv_final[2].conv
            sf, eps, g, b = self._norm_tc(norm, st, n, f0)
            return self._norm_act_head(x, sf, eps, g, b, *self._act_tc(act), conv, x_in.dtype)
