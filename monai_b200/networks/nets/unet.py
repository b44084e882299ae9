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
        # without residual units: eager, since a graph replay copies the input and the output (130 MB per batch of 25 96^3 windows),
        # which costs more than the ~17 launches of this forward take to issue.  The residual forward issues about 40 launches per
        # call, and replaying them wins (DESIGN.md §7)
        if num_res_units == 0:
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
        return x.dtype == torch.float16 and self._tc_eligible()

    def _tc_eligible(self) -> bool:
        """Whether the modules allow the tensor-core forward (the input checks aside): 3-D, 3x3x3 kernels, strides 1 or 2, channel
        counts that are multiples of 16, "NDA" blocks without active dropout and with PReLU(1) / LeakyReLU / ReLU.
          * num_res_units == 0: one input channel, non-affine InstanceNorm;
          * num_res_units > 0: any input and output channels; InstanceNorm without running statistics (affine or not), or an
            eval-mode BatchNorm3d with running statistics (folded into the convolution weights)."""
        if self.dimensions != 3 or self.kernel_size != 3 or self.up_kernel_size != 3 or self.adn_ordering.upper() != "NDA":
            return False
        if any(c % 16 for c in self.channels) or any(s not in (1, 2) for s in self.strides[: len(self.channels) - 1]):
            return False
        if self.num_res_units == 0:
            return self._plain_eligible()
        top_unit = self.model[2][1].conv[-1]   # the last unit of the top ResidualUnit: a bare convolution (last_conv_only)
        for m in self.modules():
            if isinstance(m, (nn.GroupNorm, nn.LayerNorm)) or (isinstance(m, nn.PReLU) and m.weight.numel() != 1):
                return False
            if isinstance(m, nn.modules.dropout._DropoutNd) and m.p > 0 and m.training:
                return False
            if isinstance(m, Convolution) and m is not top_unit:
                adn = getattr(m, "adn", None)
                n, a = getattr(adn, "N", None), getattr(adn, "A", None)
                inorm = isinstance(n, nn.InstanceNorm3d) and not n.track_running_stats
                bnorm = isinstance(n, nn.BatchNorm3d) and not n.training and n.track_running_stats
                if not (inorm or bnorm) or not isinstance(a, (nn.PReLU, nn.LeakyReLU, nn.ReLU)):
                    return False
        return all(isinstance(m, (nn.PReLU, nn.LeakyReLU, nn.ReLU)) for m in self.modules() if type(m).__module__.startswith("torch.nn.modules.activation"))

    def _plain_eligible(self) -> bool:
        """The rule of the forward without residual units: single-channel input, InstanceNorm (non-affine) + activation blocks."""
        if self.in_channels != 1 or self.dropout not in (0, 0.0, None):
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

    def _check_tc_input(self, x: torch.Tensor) -> None:
        if self.num_res_units == 0:
            return
        div = 1
        for s in self.strides[: len(self.channels) - 1]:
            div *= int(s)
        if x.dim() != 5 or x.shape[1] != self.in_channels:
            raise ValueError(f"UNet expects an [N, {self.in_channels}, D, H, W] input, got {tuple(x.shape)}")
        if any(int(s) % div for s in x.shape[2:]):
            raise ValueError(f"UNet with strides {tuple(self.strides[: len(self.channels) - 1])} needs spatial sizes divisible by {div}, "
                             f"got {tuple(x.shape[2:])}")

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

    # ----------------------------------------------------------------------------- tensor-core path, residual units
    # ResidualUnit (convolutions.py:112-161) is `units(x) + residual(x)` with each unit act(norm(conv(.))) ("NDA") and the residual
    # a bare convolution (k3 with the unit's stride, 1x1x1 when only the channels change) or the identity.  An eval-mode BatchNorm
    # is a fixed per-channel affine: it is folded into the convolution's weight and bias, and its unit's activation runs on
    # norm_act_nc8 without statistics.  An InstanceNorm takes its statistics from the convolution epilogues and is applied on the
    # next convolution's operand load where that kernel allows the slope (in [0, 1]), else materialised by norm_act_nc8.
    @staticmethod
    def _tensors(*mods) -> list:
        """The tensors a packed weight depends on: weight and bias of convolutions and norms, and a BatchNorm's running statistics
        (buffers, which load_state_dict changes without touching a parameter)."""
        out = []
        for m in mods:
            if m is not None:
                out += [t for t in (m.weight, m.bias) if t is not None]
                if isinstance(m, nn.BatchNorm3d):
                    out += [m.running_mean, m.running_var]
        return out

    def _folded(self, blk: Convolution, cout_pad: int | None = None) -> tuple[torch.Tensor, torch.Tensor]:
        """float32 (weight, bias) of a block's convolution with an eval-mode BatchNorm folded in: w * s and (b - mean) * s + beta with
        s = gamma / sqrt(var + eps) per output channel (dim 1 of a transposed weight).  Output channels zero-padded to `cout_pad`."""
        m = blk.conv
        ax = 1 if isinstance(m, nn.ConvTranspose3d) else 0
        w = m.weight.detach().float()
        b = m.bias.detach().float() if m.bias is not None else torch.zeros(w.shape[ax], device=w.device)
        bn = self._bn(blk)
        if bn is not None:
            g = bn.weight.detach().float() if bn.affine else 1.0
            sc = g / torch.sqrt(bn.running_var.float() + bn.eps)
            shape = [1] * w.dim()
            shape[ax] = -1
            w = w * sc.reshape(shape)
            b = (b - bn.running_mean.float()) * sc + (bn.bias.detach().float() if bn.affine else 0.0)
        if cout_pad is not None and cout_pad != w.shape[ax]:
            wp = torch.zeros((*w.shape[:ax], cout_pad, *w.shape[ax + 1:]), device=w.device)
            wp.narrow(ax, 0, w.shape[ax]).copy_(w)
            bp = torch.zeros(cout_pad, device=w.device)
            bp[: b.numel()] = b
            w, b = wp, bp
        return w, b

    def _w3f(self, blk: Convolution, cin_pad: int | None = None, cout_pad: int | None = None):
        """(conv3x3x3_tc image, float32 bias) of a stride-1 block, BatchNorm folded."""
        def build():
            w, b = self._folded(blk, cout_pad)
            return K.conv3x3x3_tc_pack_weight(self._pad_cin(w, cin_pad)), b

        return self._cache.get(("w3f", id(blk), cin_pad, cout_pad), self._tensors(blk.conv, self._bn(blk)), build)

    def _wtf(self, blk: Convolution, cout_pad: int | None = None):
        """(conv_gather_tc image, float32 bias) of a transposed k3 block (stride 1 or 2), BatchNorm folded."""
        m = blk.conv

        def build():
            w, b = self._folded(blk, cout_pad)
            return K.conv_gather_tc_pack_weight(w, 3, m.stride[0], 1, True), b

        return self._cache.get(("wtf", id(blk), cout_pad), self._tensors(m, self._bn(blk)), build)

    def _wfirst(self, ru: ResidualUnit, cin_pad: int | None, cin1: bool):
        """unit0 and the residual convolution of a ResidualUnit, which read the same input, as ONE convolution: the weights
        concatenated along Cout (unit0 first), a 1x1x1 residual as the centre tap of a 3x3x3 kernel (the same convolution at
        padding 1).  Returns (weight, float32 bias): the float32 weight itself for conv_cin1_nc8 (cin1), else the conv_gather_tc
        image."""
        u0, r = ru.conv.unit0, ru.residual

        def build():
            w0, b0 = self._folded(u0)
            wr = r.weight.detach().float()
            br = r.bias.detach().float() if r.bias is not None else torch.zeros(wr.shape[0], device=wr.device)
            if wr.shape[2] == 1:
                wr = torch.nn.functional.pad(wr, (1, 1, 1, 1, 1, 1))
            w, b = torch.cat([w0, wr]), torch.cat([b0, br])
            if cin1:
                return w.contiguous(), b
            return K.conv_gather_tc_pack_weight(self._pad_cin(w, cin_pad), 3, u0.conv.stride[0], 1, False), b

        return self._cache.get(("wfirst", id(ru), cin_pad, cin1), self._tensors(u0.conv, self._bn(u0), r), build)

    def _wres(self, ru: ResidualUnit, cin_pad: int | None):
        """(gemm_tc image, float32 bias) of a 1x1x1 residual convolution."""
        r = ru.residual

        def build():
            w = self._pad_cin(r.weight.detach().float(), cin_pad)
            b = r.bias.detach().float() if r.bias is not None else None
            return K.gemm_tc_pack_weight(w.reshape(w.shape[0], -1)), b

        return self._cache.get(("wres", id(ru), cin_pad), self._tensors(r), build)

    def _padded(self, t: torch.Tensor | None, n: int) -> torch.Tensor | None:
        """A per-channel parameter zero-padded to n channels (float32, cached); None and full-length ones as they are."""
        if t is None or t.numel() == n:
            return t
        return self._cache.get(("pad", id(t), n), [t], lambda: torch.nn.functional.pad(t.detach().float(), (0, n - t.numel())))

    @staticmethod
    def _on_load(inorm: bool, act: int, slope: float) -> bool:
        """Whether conv3x3x3_tc can apply this norm + activation on its operand load (it takes slopes in [0, 1] only)."""
        return inorm and (act != L.ACT_LEAKY or 0.0 <= slope <= 1.0)

    def _tc_ru(self, ru: ResidualUnit, x, cin: int, in_coff: int, out: K.NC8, out_coff: int, raw=None, cin_pad: int | None = None) -> None:
        """A ResidualUnit with an "NDA" last unit: out[:, out_coff:...] = act(norm(y_last)) + residual(x)."""
        units = list(ru.conv)
        u0 = units[0]
        cout = u0.conv.out_channels
        want = self._adn(u0)[0]
        if raw is not None or self._strided(u0.conv):
            # unit0 and the residual convolution in one launch: channels [0, cout) are unit0's, [cout, 2 cout) the residual's
            s = u0.conv.stride[0]
            w, b = self._wfirst(ru, cin_pad, raw is not None)
            if raw is not None:
                y, st = K.conv_cin1_nc8(raw, w, b, 3, s, 1, want_stats=want)
            else:
                y, st = K.conv_gather_tc(x, w, cin, 2 * cout, 3, s, 1, in_coff=in_coff, bias=b, want_stats=want)
            if st is not None:
                st = st.view(y.N, 2 * cout, 2)[:, :cout].contiguous().view(y.N * cout, 2)
            res, res_coff = y, cout
        else:
            w, b = self._w3f(u0, cin_pad)
            y, st = K.conv3x3x3_tc(x, w, cin, cout, in_coff=in_coff, bias=b, want_stats=want)
            if isinstance(ru.residual, nn.Identity):
                res, res_coff = x, in_coff
            else:
                wr, br = self._wres(ru, cin_pad)
                res, _ = K.gemm_tc(x, wr, cin, cout, bias=br, in_coff=in_coff)
                res_coff = 0
        prev = u0
        for u in units[1:]:
            inorm, eps, g, be, act, slope = self._adn(prev)
            w, b = self._w3f(u)
            want = self._adn(u)[0]
            if self._on_load(inorm, act, slope):
                y, st = K.conv3x3x3_tc(y, w, cout, cout, bias=b, want_stats=want, in_norm=(st, eps, act, slope), in_affine=(g, be))
            else:
                y, st = K.conv3x3x3_tc(self._finish(y, cout, st, prev), w, cout, cout, bias=b, want_stats=want)
            prev = u
        self._finish(y, cout, st, prev, out=out, out_coff=out_coff, res=res, res_coff=res_coff)

    def _tc_res_up(self, up: nn.Sequential, cat: K.NC8, cin: int, top: bool, out, out_coff: int, out_dtype):
        """Transposed Convolution (NDA) -> x_u, then ResidualUnit(subunits=1, identity residual): act(norm(conv(x_u))) + x_u into
        `out`, or at the top conv(x_u) + x_u (last_conv_only) as NCDHW logits in `out_dtype`."""
        tconv, unit = up[0], up[1].conv.unit0
        m = tconv.conv
        cout = m.out_channels
        cp = (cout + 15) // 16 * 16 if top else cout   # the top's few output channels run zero-padded on 16-channel tiles
        inorm, eps, g, be, act, slope = self._adn(tconv)
        g, be = self._padded(g, cp), self._padded(be, cp)
        wt, bt = self._wtf(tconv, cp if top else None)
        t, st = K.conv_gather_tc(cat, wt, cin, cp, 3, m.stride[0], 1, transposed=True, output_padding=m.output_padding[0], bias=bt,
                                 want_stats=inorm)
        xu = K.norm_act_nc8(t, cp, st, act=act, slope=slope, eps=eps, gamma=g, beta=be)
        if not top:
            w, b = self._w3f(unit)
            y, st2 = K.conv3x3x3_tc(xu, w, cout, cout, bias=b, want_stats=self._adn(unit)[0])
            return self._finish(y, cout, st2, unit, out=out, out_coff=out_coff, res=xu)
        w, b = self._w3f(unit, cp, cp)
        if self._on_load(inorm, act, slope):
            z, _ = K.conv3x3x3_tc(t, w, cp, cp, bias=b, in_norm=(st, eps, act, slope), in_affine=(g, be), add=(xu, 0))
        else:
            z, _ = K.conv3x3x3_tc(xu, w, cp, cp, bias=b)
            K.norm_act_nc8(z, cp, None, res=xu, out=z, res_after_act=True)
        y = K.unpack_nc8(z, (cout + 7) // 8 * 8, 0, out_dtype)
        return y if y.shape[1] == cout else y[:, :cout].contiguous()

    def _tc_res_level(self, block: nn.Sequential, x, cin: int, raw, cin_pad, top: bool, out, out_coff: int, out_dtype):
        down, skip, up = block[0], block[1], block[2]
        sub = skip.submodule
        c = down.out_channels
        bottom = isinstance(sub, ResidualUnit)
        c_sub = sub.out_channels if bottom else sub[2][0].conv.out_channels
        s = down.conv.unit0.conv.stride[0]
        src = raw if raw is not None else x.buf
        sp = tuple(int(v) // s for v in (raw.shape[2:] if raw is not None else x.sp))
        # `down` output and the sub-network's output share one buffer: torch.cat([x, sub(x)], 1) without a copy
        cat = K.NC8(raw.shape[0] if raw is not None else x.N, c + c_sub, sp, src.device)
        self._tc_ru(down, x, cin, 0, cat, 0, raw=raw, cin_pad=cin_pad)
        if bottom:
            self._tc_ru(sub, cat, c, 0, cat, c)
        else:
            self._tc_res_level(sub, cat, c, None, None, False, cat, c, None)
        return self._tc_res_up(up, cat, c + c_sub, top, out, out_coff, out_dtype)

    def _forward_tc(self, x: torch.Tensor) -> torch.Tensor:
        with torch.no_grad():
            x = x.contiguous()
            if self.num_res_units == 0:
                return self._tc_level(self.model, None, 1, x, True, None, 0, x.dtype)
            if self.in_channels == 1:
                return self._tc_res_level(self.model, None, 1, x, None, True, None, 0, x.dtype)
            xp, cp = self._pack_input(x)
            return self._tc_res_level(self.model, xp, cp, None, cp, True, None, 0, x.dtype)

    def _forward_generic(self, x: torch.Tensor) -> torch.Tensor:
        with torch.no_grad():
            return self.model(x.contiguous())


Unet = UNet
