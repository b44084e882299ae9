"""`BasicUNet` (monai/networks/nets/basic_unet.py:27-282) on the monai_b200 CUDA kernels.

Module tree and state_dict keys follow the reference (`conv_0.conv_0.conv.weight`, `down_1.convs.conv_1.adn.N.weight`,
`upcat_4.upsample.deconv.weight`, `final_conv.weight`, ...).  Only the default `upsample="deconv"` mode is on the
north-star path; the other modes raise NotImplementedError.

Two forwards, chosen from the input and the configuration (DESIGN.md §8.4):
  * fp16 CUDA input with every spatial size divisible by 16, dropout inactive, and an eligible configuration (`_tc_ok`: InstanceNorm3d
    without running statistics, affine or not; ReLU or LeakyReLU with a slope in [0, 1]; features[0..5] % 16 == 0 and
    features[2..4] % 32 == 0, so that both halves of every concat are whole 16-channel tiles): `_forward_tc`, the whole network on
    fp16 channel-blocked (NC8) buffers and Hopper tensor cores -- every 3x3x3 convolution on `b200_conv3x3x3_tc` (a one-channel
    stem on `b200_conv_cin1_nc8`) with conv_0's InstanceNorm + activation applied on conv_1's operand load, conv_1's norm +
    activation in one `b200_norm_act_nc8` pass straight into the skip half of the decoder's concat buffer, the 2x max pool on
    `b200_maxpool2_nc8`, the transposed convolutions on `b200_gemm_tc` into the other half, and the last norm + activation fused
    into the 1x1x1 head -- replayed from a CUDA graph per input shape;
  * everything else (fp32 input, other sizes, which the reference pads, BatchNorm, other activations or widths): `_forward_generic`,
    the fp32-faithful generic kernels.
"""
from __future__ import annotations

from collections.abc import Sequence

import torch
import torch.nn as nn

from ... import _kernels as K
from ..blocks.convolutions import Convolution, run_conv_module
from ._tc_blocks import TcNet

__all__ = ["BasicUNet", "BasicUnet", "Basicunet", "basicunet", "TwoConv", "Down", "UpCat"]

_CONV = {1: nn.Conv1d, 2: nn.Conv2d, 3: nn.Conv3d}
_CONVT = {1: nn.ConvTranspose1d, 2: nn.ConvTranspose2d, 3: nn.ConvTranspose3d}
_POOL = {1: nn.MaxPool1d, 2: nn.MaxPool2d, 3: nn.MaxPool3d}


class TwoConv(nn.Sequential):
    """two convolutions (basic_unet.py:27-58)."""

    def __init__(self, spatial_dims: int, in_chns: int, out_chns: int, act, norm, bias: bool, dropout=0.0):
        super().__init__()
        self.add_module("conv_0", Convolution(spatial_dims, in_chns, out_chns, act=act, norm=norm, dropout=dropout, bias=bias, padding=1))
        self.add_module("conv_1", Convolution(spatial_dims, out_chns, out_chns, act=act, norm=norm, dropout=dropout, bias=bias, padding=1))


class Down(nn.Sequential):
    """max-pool by 2 then TwoConv (basic_unet.py:61-89)."""

    def __init__(self, spatial_dims: int, in_chns: int, out_chns: int, act, norm, bias: bool, dropout=0.0):
        super().__init__()
        self.add_module("max_pooling", _POOL[spatial_dims](kernel_size=2))
        self.add_module("convs", TwoConv(spatial_dims, in_chns, out_chns, act, norm, bias, dropout))

    def forward(self, x: torch.Tensor) -> torch.Tensor:  # type: ignore[override]
        nd = x.dim() - 2
        x3 = x.reshape(x.shape[0], x.shape[1], *([1] * (3 - nd)), *x.shape[2:])
        if nd != 3:
            raise NotImplementedError("monai_b200 BasicUNet pooling is implemented for 3 spatial dims")
        return self.convs(K.maxpool3d_2(x3))


class _UpSampleDeconv(nn.Module):
    """UpSample(mode="deconv") (monai/networks/blocks/upsample.py:102-116): ConvTranspose(k=2, s=2)."""

    def __init__(self, spatial_dims: int, in_chns: int, out_chns: int):
        super().__init__()
        self.add_module("deconv", _CONVT[spatial_dims](in_chns, out_chns, kernel_size=2, stride=2, bias=True))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return run_conv_module(self.deconv, x)


class UpCat(nn.Module):
    """upsample, replicate-pad to the skip's size, concatenate [skip, up], TwoConv (basic_unet.py:92-175)."""

    def __init__(self, spatial_dims, in_chns, cat_chns, out_chns, act, norm, bias, dropout=0.0, upsample="deconv", halves=True, is_pad=True):
        super().__init__()
        if upsample != "deconv":
            raise NotImplementedError("monai_b200 BasicUNet implements upsample='deconv' only")
        up_chns = in_chns // 2 if halves else in_chns
        self.upsample = _UpSampleDeconv(spatial_dims, in_chns, up_chns)
        self.convs = TwoConv(spatial_dims, cat_chns + up_chns, out_chns, act, norm, bias, dropout)
        self.is_pad = is_pad

    def forward(self, x: torch.Tensor, x_e: torch.Tensor | None) -> torch.Tensor:
        x_0 = self.upsample(x)
        if x_e is None:
            return self.convs(x_0)
        n, ce = x_e.shape[:2]
        cu = x_0.shape[1]
        sp = tuple(x_e.shape[2:]) if self.is_pad else tuple(x_0.shape[2:])
        if any(a - b not in (0, 1) for a, b in zip(sp, x_0.shape[2:])):
            raise ValueError(f"skip {tuple(x_e.shape)} and upsampled {tuple(x_0.shape)} tensors differ by more than one voxel")
        cat = torch.empty((n, ce + cu, *sp), device=x.device, dtype=x.dtype)
        K.copy_channels(x_e, cat, 0)
        K.copy_channels(x_0, cat, ce)  # replicate-pads the high side when the skip is one voxel larger
        return self.convs(cat)


class BasicUNet(TcNet, nn.Module):
    def __init__(
        self,
        spatial_dims: int = 3,
        in_channels: int = 1,
        out_channels: int = 2,
        features: Sequence[int] = (32, 32, 64, 128, 256, 32),
        act=("LeakyReLU", {"negative_slope": 0.1, "inplace": True}),
        norm=("instance", {"affine": True}),
        bias: bool = True,
        dropout=0.0,
        upsample: str = "deconv",
    ):
        super().__init__()
        if spatial_dims != 3:
            raise NotImplementedError("monai_b200 BasicUNet is implemented for spatial_dims=3 (the sliding-window hot path)")
        fea = tuple(features)
        if len(fea) != 6:
            raise ValueError(f"Sequence must have length 6, got {len(fea)}.")
        print(f"BasicUNet features: {fea}.")
        self.in_channels, self._features, self._upsample = in_channels, fea, upsample
        self.conv_0 = TwoConv(spatial_dims, in_channels, fea[0], act, norm, bias, dropout)
        self.down_1 = Down(spatial_dims, fea[0], fea[1], act, norm, bias, dropout)
        self.down_2 = Down(spatial_dims, fea[1], fea[2], act, norm, bias, dropout)
        self.down_3 = Down(spatial_dims, fea[2], fea[3], act, norm, bias, dropout)
        self.down_4 = Down(spatial_dims, fea[3], fea[4], act, norm, bias, dropout)
        self.upcat_4 = UpCat(spatial_dims, fea[4], fea[3], fea[3], act, norm, bias, dropout, upsample)
        self.upcat_3 = UpCat(spatial_dims, fea[3], fea[2], fea[2], act, norm, bias, dropout, upsample)
        self.upcat_2 = UpCat(spatial_dims, fea[2], fea[1], fea[1], act, norm, bias, dropout, upsample)
        self.upcat_1 = UpCat(spatial_dims, fea[1], fea[0], fea[5], act, norm, bias, dropout, upsample, halves=False)
        self.final_conv = _CONV[spatial_dims](fea[5], out_channels, kernel_size=1)
        self._tc_ok = self._tc_eligible()
        self._tc_setup()

    def _tc_eligible(self) -> bool:
        """Whether `_forward_tc` implements this configuration: transposed-convolution upsampling, every norm an InstanceNorm3d
        without running statistics (affine or not), every activation ReLU or LeakyReLU with a slope in [0, 1], and channel counts
        that are whole 16-channel tiles, the halves of the upcat_4 ... upcat_2 concats included (features[2..4] // 2)."""
        fea = self._features
        if self._upsample != "deconv" or any(f % 16 for f in fea) or any(fea[k] % 32 for k in (2, 3, 4)):
            return False
        for m in self.modules():
            if isinstance(m, Convolution):
                n, a = getattr(getattr(m, "adn", None), "N", None), getattr(getattr(m, "adn", None), "A", None)
                if not (isinstance(n, nn.InstanceNorm3d) and not n.track_running_stats):
                    return False
                if not (type(a) is nn.ReLU or (type(a) is nn.LeakyReLU and 0.0 <= a.negative_slope <= 1.0)):
                    return False
        return True

    def _dropout_active(self) -> bool:
        return any(m.training and m.p > 0 for m in self.modules() if isinstance(m, nn.modules.dropout._DropoutNd))

    def _check_input(self, x: torch.Tensor) -> None:
        if not x.is_cuda:
            raise RuntimeError("monai_b200.BasicUNet runs on CUDA tensors only (there is no CPU fallback)")

    def _use_tc(self, x: torch.Tensor) -> bool:
        # a size not divisible by 16 takes the generic path, which pads it as the reference does (UpCat's is_pad)
        return (super()._use_tc(x) and not self._dropout_active()
                and (x.dim() != 5 or all(int(s) % 16 == 0 for s in x.shape[2:])))

    def _check_tc_input(self, x: torch.Tensor) -> None:
        self._check_levels(x, 5)

    def _forward_generic(self, x: torch.Tensor) -> torch.Tensor:
        with torch.no_grad():
            x0 = self.conv_0(x.contiguous())
            x1 = self.down_1(x0)
            x2 = self.down_2(x1)
            x3 = self.down_3(x2)
            x4 = self.down_4(x3)
            u4 = self.upcat_4(x4, x3)
            u3 = self.upcat_3(u4, x2)
            u2 = self.upcat_2(u3, x1)
            u1 = self.upcat_1(u2, x0)
            return run_conv_module(self.final_conv, u1)

    # ------------------------------------------------------------------------------------------- tensor-core path
    def _two_conv_tc(self, x: K.NC8 | None, cin: int, tc: TwoConv, key: str, cin_pad: int | None = None, raw: torch.Tensor | None = None):
        """TwoConv up to conv_1's raw output: conv_0 (raw output + statistics; the one-channel stem reads the NCDHW window `raw`),
        then conv_1 with conv_0's InstanceNorm + activation applied on its operand load.  Returns (y, statistics of y)."""
        c0, c1 = tc.conv_0.conv, tc.conv_1.conv
        if raw is not None:
            y, st = K.conv_cin1_nc8(raw, c0.weight, c0.bias, 3, 1, 1, want_stats=True)
        else:
            y, st = K.conv3x3x3_tc(x, self._w3(c0, key + ".c0", cin_pad), cin, c0.out_channels, bias=c0.bias, want_stats=True)
        _, eps, g, b, act, slope = self._adn(tc.conv_0)
        return K.conv3x3x3_tc(y, self._w3(c1, key + ".c1"), c1.in_channels, c1.out_channels, bias=c1.bias, want_stats=True,
                              in_norm=(st, eps, act, slope), in_affine=(g, b))

    def _forward_tc(self, x_in: torch.Tensor) -> torch.Tensor:
        """BasicUNet.forward (basic_unet.py, eval mode) on fp16 NC8 buffers and tensor cores; the output is fp16 NCDHW.

        Encoder level k < 4 owns the concat buffer of upcat_{k+1}: channels [0, fea[k]) receive x_k (the reference concatenates
        [skip, upsampled]), so torch.cat needs no copy, and the max pool reads x_k from there.  The decoder's transposed
        convolution writes the upper channels, and conv_0 reads the whole buffer."""
        with torch.no_grad():
            x_in = x_in.contiguous()
            enc = [self.conv_0, self.down_1.convs, self.down_2.convs, self.down_3.convs, self.down_4.convs]
            ups = [self.upcat_4, self.upcat_3, self.upcat_2, self.upcat_1]
            if self.in_channels == 1:   # the raw NCDHW window feeds the single-channel stem kernel
                y, st = self._two_conv_tc(None, 1, enc[0], "e0", raw=x_in)
            else:
                xp, cp = self._pack_input(x_in)
                y, st = self._two_conv_tc(xp, cp, enc[0], "e0", cin_pad=cp)
            cats = []
            for k in range(1, 5):
                c = enc[k - 1].conv_1.conv.out_channels
                cat = K.NC8(y.N, c + ups[4 - k].upsample.deconv.out_channels, y.sp, y.buf.device)
                self._finish(y, c, st, enc[k - 1].conv_1, out=cat)   # x_{k-1}: act(norm(y)) into the skip channels
                cats.append(cat)
                y, st = self._two_conv_tc(K.maxpool2_nc8(cat, c), c, enc[k], f"e{k}")
            x = self._finish(y, y.C, st, enc[4].conv_1)   # x4
            for i, uc in enumerate(ups):                  # upcat_4 ... upcat_1
                cat, dc = cats[3 - i], uc.upsample.deconv
                self._up(x, x.C, dc, f"u{i}.up", out=cat, out_coff=cat.C - dc.out_channels)
                y, st = self._two_conv_tc(cat, cat.C, uc.convs, f"u{i}")
                if i < 3:   # gemm_tc has no operand normalisation: the next transposed convolution reads act(norm(y))
                    x = self._finish(y, y.C, st, uc.convs.conv_1)
            _, eps, g, b, act, slope = self._adn(self.upcat_1.convs.conv_1)
            return self._norm_act_head(y, st, eps, g, b, act, slope, self.final_conv, x_in.dtype)


BasicUnet = Basicunet = basicunet = BasicUNet
