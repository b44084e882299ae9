"""SegResNetDS (monai/networks/nets/segresnet_ds.py:30-428; the network of MONAI's Auto3DSeg `segresnet` algorithm) behind the
reference's constructor, module tree and state_dict keys, on the CUDA kernels of this package.

conv_init, then per level pre-activation SegResBlocks (`x + conv2(act2(norm2(conv1(act1(norm1(x))))))`, BatchNorm by default) and
a strided convolution; the decoder upsamples (transposed convolution or 1x1 + trilinear), adds the encoder feature, runs
SegResBlocks and ends in a 1x1 head.  With `resolution`, the first levels use one-plane kernels ([3,3,1], [1,3,3], ...) and strides
that bring the spacing towards isotropy.  Inference only: in eval mode the output is the reference's `outputs[0]`; the deep
supervision heads (`dsdepth > 1`) are parameters whose outputs exist in training mode only.

Two forwards, chosen from the input and the configuration (DESIGN.md §8.4):
  * fp16 CUDA input and an eligible configuration (`_tc_ok`, decided at construction: 3-D, init_filters % 16 == 0, 3x3x3 kernels or
    3x3 kernels in one plane, InstanceNorm3d without running statistics / GroupNorm / BatchNorm3d with running statistics, ReLU or
    LeakyReLU with a slope in [0, 1], a decoder down to level 0, "deconv" upsampling or "nontrainable" with every scale 2; BatchNorm in
    eval mode at call time): `_forward_tc`, the whole network on fp16 NC8 buffers and Hopper tensor cores, replayed from a CUDA graph
    per input shape -- each SegResBlock is two launches of `b200_conv3x3x3_tc` / `b200_conv3x3_tc` with its norm + activation applied
    on the operand load (from the statistics of the previous epilogue, or the given BatchNorm scale / shift table) and the identity
    added in conv2's epilogue;
  * everything else: `_forward_generic`, the fp32-faithful generic kernels.
"""
from __future__ import annotations

import inspect

import numpy as np
import torch
import torch.nn as nn

from ... import _kernels as K
from ... import _lib as L
from ..blocks.acti_norm import norm_act_from_modules
from ..blocks.convolutions import run_conv_module
from ..blocks.segresnet_block import UpSample
from ..layers.factories import _ACTS, get_act_layer, get_norm_layer, split_args
from ._tc_blocks import TcNet

__all__ = ["SegResNetDS", "SegResBlock", "SegResEncoder", "scales_for_resolution", "aniso_kernel"]


def scales_for_resolution(resolution: tuple | list, n_stages: int | None = None):
    """The per-level (stride) scales that bring `resolution` (in mm) towards isotropy (segresnet_ds.py:30-55)."""
    ndim = len(resolution)
    res = np.array(resolution)
    if not all(res > 0):
        raise ValueError("Resolution must be positive")
    nl = np.floor(np.log2(np.max(res) / res)).astype(np.int32)
    scales = [tuple(np.where(2**i >= 2**nl, 1, 2)) for i in range(max(nl))]
    if n_stages and n_stages > max(nl):
        scales = scales + [(2,) * ndim] * (n_stages - max(nl))
    else:
        scales = scales[:n_stages]
    return scales


def aniso_kernel(scale: tuple | list):
    """(kernel_size, padding, stride) of a level with the given scale: kernel 3 where the scale is > 1, else 1 (segresnet_ds.py:58-67)."""
    kernel_size = [3 if scale[k] > 1 else 1 for k in range(len(scale))]
    padding = [k // 2 for k in kernel_size]
    return kernel_size, padding, scale


def _conv(spatial_dims: int, *args, **kw) -> nn.Module:
    return (nn.Conv1d, nn.Conv2d, nn.Conv3d)[spatial_dims - 1](*args, **kw)


def _layer_args(norm, act):
    """The reference's defaults (segresnet_ds.py:161-169, 297-305): a norm that takes `affine` gets affine=True unless given, an
    activation that takes `inplace` gets inplace=True unless given.  Every norm `get_norm_layer` builds (instance, batch, group)
    takes `affine`."""
    norm_name, norm_kw = split_args(norm)
    norm_kw = dict(norm_kw)
    norm_kw.setdefault("affine", True)
    act_name, act_kw = split_args(act)
    act_kw = dict(act_kw)
    cls = _ACTS.get(str(act_name).lower())
    if cls is not None and "inplace" in inspect.signature(cls.__init__).parameters:
        act_kw.setdefault("inplace", True)
    return (norm_name, norm_kw), (act_name, act_kw)


class SegResBlock(nn.Module):
    """Pre-activation residual block (segresnet_ds.py:70-125): x + conv2(act2(norm2(conv1(act1(norm1(x))))))."""

    def __init__(self, spatial_dims: int, in_channels: int, norm, kernel_size=3, act="relu") -> None:
        super().__init__()
        if isinstance(kernel_size, (tuple, list)):
            padding = tuple(k // 2 for k in kernel_size)
        else:
            padding = kernel_size // 2
        self.norm1 = get_norm_layer(name=norm, spatial_dims=spatial_dims, channels=in_channels)
        self.act1 = get_act_layer(act)
        self.conv1 = _conv(spatial_dims, in_channels, in_channels, kernel_size=kernel_size, stride=1, padding=padding, bias=False)
        self.norm2 = get_norm_layer(name=norm, spatial_dims=spatial_dims, channels=in_channels)
        self.act2 = get_act_layer(act)
        self.conv2 = _conv(spatial_dims, in_channels, in_channels, kernel_size=kernel_size, stride=1, padding=padding, bias=False)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        y = run_conv_module(self.conv1, norm_act_from_modules(x, self.norm1, self.act1))
        y = run_conv_module(self.conv2, norm_act_from_modules(y, self.norm2, self.act2))
        return K.norm_act(y, None, res=x, act=L.ACT_NONE)   # y + identity


class SegResEncoder(nn.Module):
    """conv_init, then per level `blocks` and a strided `downsample` convolution (segresnet_ds.py:128-232); forward returns the output
    of every level's blocks."""

    def __init__(self, spatial_dims: int = 3, init_filters: int = 32, in_channels: int = 1, act="relu", norm="batch",
                 blocks_down: tuple = (1, 2, 2, 4), head_module: nn.Module | None = None, anisotropic_scales: tuple | None = None):
        super().__init__()
        if spatial_dims not in (1, 2, 3):
            raise ValueError("`spatial_dims` can only be 1, 2 or 3.")
        norm, act = _layer_args(norm, act)
        filters = init_filters
        kernel_size, padding, _ = aniso_kernel(anisotropic_scales[0]) if anisotropic_scales else (3, 1, 1)
        self.conv_init = _conv(spatial_dims, in_channels, filters, kernel_size=kernel_size, padding=padding, stride=1, bias=False)
        self.layers = nn.ModuleList()
        for i in range(len(blocks_down)):
            level = nn.ModuleDict()
            kernel_size, padding, stride = aniso_kernel(anisotropic_scales[i]) if anisotropic_scales else (3, 1, 2)
            level["blocks"] = nn.Sequential(*[SegResBlock(spatial_dims, filters, kernel_size=kernel_size, norm=norm, act=act)
                                              for _ in range(blocks_down[i])])
            if i < len(blocks_down) - 1:
                level["downsample"] = _conv(spatial_dims, filters, 2 * filters, bias=False, kernel_size=kernel_size, stride=stride, padding=padding)
            else:
                level["downsample"] = nn.Identity()
            self.layers.append(level)
            filters *= 2
        self.head_module = head_module
        self.in_channels, self.blocks_down, self.init_filters = in_channels, blocks_down, init_filters
        self.norm, self.act, self.spatial_dims = norm, act, spatial_dims

    def forward(self, x: torch.Tensor) -> list[torch.Tensor]:
        outputs = []
        x = run_conv_module(self.conv_init, x)
        for level in self.layers:
            x = level["blocks"](x)
            outputs.append(x)
            if not isinstance(level["downsample"], nn.Identity):
                x = run_conv_module(level["downsample"], x)
        if self.head_module is not None:
            outputs = self.head_module(outputs)
        return outputs


class SegResNetDS(TcNet, nn.Module):
    def __init__(
        self,
        spatial_dims: int = 3,
        init_filters: int = 32,
        in_channels: int = 1,
        out_channels: int = 2,
        act="relu",
        norm="batch",
        blocks_down: tuple = (1, 2, 2, 4),
        blocks_up: tuple | None = None,
        dsdepth: int = 1,
        preprocess=None,
        upsample_mode: str = "deconv",
        resolution: tuple | None = None,
    ):
        super().__init__()
        if spatial_dims not in (1, 2, 3):
            raise ValueError("`spatial_dims` can only be 1, 2 or 3.")
        self.spatial_dims, self.init_filters, self.in_channels, self.out_channels = spatial_dims, init_filters, in_channels, out_channels
        self.act, self.norm, self.blocks_down = act, norm, blocks_down
        self.dsdepth = max(dsdepth, 1)
        self.resolution, self.preprocess = resolution, preprocess
        self.upsample_mode = str(getattr(upsample_mode, "value", upsample_mode))
        if resolution is not None:
            if not isinstance(resolution, (list, tuple)):
                raise TypeError("resolution must be a tuple")
            elif not all(r > 0 for r in resolution):
                raise ValueError("resolution must be positive")
        norm, act = _layer_args(norm, act)
        anisotropic_scales = scales_for_resolution(resolution, n_stages=len(blocks_down)) if resolution else None
        self.anisotropic_scales = anisotropic_scales
        self.encoder = SegResEncoder(spatial_dims=spatial_dims, init_filters=init_filters, in_channels=in_channels, act=act, norm=norm,
                                     blocks_down=blocks_down, anisotropic_scales=anisotropic_scales)
        n_up = len(blocks_down) - 1
        if blocks_up is None:
            blocks_up = (1,) * n_up
        self.blocks_up = blocks_up
        filters = init_filters * 2**n_up
        self.up_layers = nn.ModuleList()
        for i in range(n_up):
            filters = filters // 2
            kernel_size, _, stride = aniso_kernel(anisotropic_scales[len(blocks_up) - i - 1]) if anisotropic_scales else (3, 1, 2)
            level = nn.ModuleDict()
            level["upsample"] = UpSample(mode=self.upsample_mode, spatial_dims=spatial_dims, in_channels=2 * filters, out_channels=filters,
                                         kernel_size=kernel_size, scale_factor=stride, bias=False, align_corners=False)
            level["blocks"] = nn.Sequential(*[SegResBlock(spatial_dims, filters, kernel_size=kernel_size, norm=norm, act=act)
                                              for _ in range(blocks_up[i])])
            if len(blocks_up) - i <= dsdepth:   # deep supervision heads
                level["head"] = _conv(spatial_dims, filters, out_channels, kernel_size=1, bias=True)
            else:
                level["head"] = nn.Identity()
            self.up_layers.append(level)
        if n_up == 0:   # a flat structure (no downsampling) gets a single head
            self.up_layers.append(nn.ModuleDict({"upsample": nn.Identity(), "blocks": nn.Identity(),
                                                 "head": _conv(spatial_dims, filters, out_channels, kernel_size=1, bias=True)}))
        self._tc_ok = self._tc_eligible()
        self._tc_setup()

    def shape_factor(self):
        """The factors (divisors) each spatial size of the input must be divisible by (segresnet_ds.py:374-382)."""
        if self.anisotropic_scales is None:
            return [2 ** (len(self.blocks_down) - 1)] * self.spatial_dims
        return list(np.prod(np.array(self.anisotropic_scales[:-1]), axis=0))

    def is_valid_shape(self, x):
        """Whether the input's spatial shape is divisible by `shape_factor()` (segresnet_ds.py:384-389)."""
        return all(i % j == 0 for i, j in zip(x.shape[2:], self.shape_factor()))

    # ------------------------------------------------------------------------------------------------- dispatch
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        # segresnet_ds.py:391-396: preprocess, then the divisibility check, before either path launches anything (and outside any
        # CUDA graph: preprocess is arbitrary user code)
        if self.preprocess is not None:
            x = self.preprocess(x)
        if not self.is_valid_shape(x):
            raise ValueError(f"Input spatial dims {x.shape} must be divisible by {self.shape_factor()}")
        return TcNet.forward(self, x)

    def _check_input(self, x: torch.Tensor) -> None:
        if self.training and self.dsdepth > 1 and len(self.up_layers) > 1:
            raise RuntimeError("monai_b200.SegResNetDS is inference-only: call .eval() (deep-supervision outputs exist in training mode only)")
        if x.dim() != self.spatial_dims + 2 or x.shape[1] != self.in_channels:
            raise ValueError(f"SegResNetDS expects an [N, {self.in_channels}, *spatial] input with {self.spatial_dims} spatial axes, "
                             f"got {tuple(x.shape)}")

    def _norms(self) -> list[nn.Module]:
        return [n for m in self.modules() if isinstance(m, SegResBlock) for n in (m.norm1, m.norm2)]

    def _tc_eligible(self) -> bool:
        """Whether `_forward_tc` implements this configuration; eval mode of a BatchNorm is checked at call time (`_use_tc`)."""
        if self.spatial_dims != 3 or self.init_filters % 16 or len(self.blocks_up) != len(self.blocks_down) - 1:
            return False
        scales = self.anisotropic_scales or [(2, 2, 2)] * len(self.blocks_down)
        if any(sum(int(s) == 1 for s in sc) > 1 for sc in scales):   # kernels with two axes of size 1
            return False
        if self.upsample_mode == "nontrainable":
            if any(tuple(int(s) for s in sc) != (2, 2, 2) for sc in scales[:-1]):
                return False
        elif self.upsample_mode != "deconv":
            return False
        for nm in self._norms():
            inorm = isinstance(nm, nn.InstanceNorm3d) and not nm.track_running_stats
            bnorm = isinstance(nm, nn.BatchNorm3d) and nm.track_running_stats
            if not (inorm or bnorm or isinstance(nm, nn.GroupNorm)):
                return False
        for m in self.modules():
            if isinstance(m, SegResBlock):
                for a in (m.act1, m.act2):
                    if not (type(a) is nn.ReLU or (type(a) is nn.LeakyReLU and 0.0 <= a.negative_slope <= 1.0)):
                        return False
        return True

    def _use_tc(self, x: torch.Tensor) -> bool:
        return super()._use_tc(x) and not any(isinstance(n, nn.BatchNorm3d) and n.training for n in self._norms())

    # ------------------------------------------------------------------------------------------------- generic path
    def _forward_generic(self, x: torch.Tensor) -> torch.Tensor:
        """segresnet_ds.py:398-422 on the generic kernels; returns the finest head's output (`outputs[0]`)."""
        x_down = self.encoder(x)
        x_down.reverse()
        x = x_down.pop(0)
        if len(self.up_layers) and len(self.blocks_down) > 1:
            for level in self.up_layers:
                x = level["upsample"](x)
                x = K.norm_act(x, None, res=x_down.pop(0), act=L.ACT_NONE)   # up(x) + skip
                x = level["blocks"](x)
        # n_up == 0: the reference adds a zero, and its single level has identity upsample and blocks
        return run_conv_module(self.up_layers[-1]["head"], x)

    # ------------------------------------------------------------------------------------------- tensor-core path
    @staticmethod
    def _act_tc(act: nn.Module) -> tuple[int, float]:
        if isinstance(act, nn.LeakyReLU):
            return L.ACT_LEAKY, float(act.negative_slope)
        return L.ACT_RELU, 0.0

    def _operand_norm(self, norm: nn.Module, act: nn.Module, stats: torch.Tensor | None, N: int, C: int, key: str) -> dict:
        """The operand-load normalisation of a convolution that consumes norm + act: `in_scale_shift` for an eval-mode BatchNorm (the
        float32 table is cached on gamma, beta and the running statistics), else `in_norm` / `in_affine` from the statistics of the
        producing launch (a GroupNorm's per-channel sums folded into group sums)."""
        a, slope = self._act_tc(act)
        if isinstance(norm, nn.BatchNorm3d):
            params = [t for t in (norm.weight, norm.bias, norm.running_mean, norm.running_var) if t is not None]
            tab = self._cache.get(("bn", key, norm.running_var.device), params, lambda: K.batchnorm_scale_shift(norm))
            return {"in_scale_shift": (tab, a, slope)}
        eps, g, b = TcNet._norm(norm)
        groups = norm.num_groups if isinstance(norm, nn.GroupNorm) else C
        return {"in_norm": (K.group_stats(stats, N, C, groups), eps, a, slope), "in_affine": (g, b)}

    def _want_stats(self) -> bool:
        return not isinstance(self._norms()[0], nn.BatchNorm3d) if self._norms() else False

    def _block_tc(self, x: K.NC8, st, blk: SegResBlock, key: str, want: bool):
        """SegResBlock.forward in two launches: each norm + act runs on its convolution's operand load, and the identity is added in
        conv2's epilogue (whose statistics are those of the sum)."""
        C = x.C
        y1, st1 = self._conv_s1(x, C, blk.conv1, key + ".c1", want_stats=want, **self._operand_norm(blk.norm1, blk.act1, st, x.N, C, key + ".n1"))
        return self._conv_s1(y1, C, blk.conv2, key + ".c2", want_stats=want, add=(x, 0),
                             **self._operand_norm(blk.norm2, blk.act2, st1, x.N, C, key + ".n2"))

    def _forward_tc(self, x_in: torch.Tensor) -> torch.Tensor:
        """SegResNetDS._forward (segresnet_ds.py:391-422, eval mode) on fp16 NC8 buffers and tensor cores; the output is in the input's
        dtype.  Statistics are produced only when the norms are instance or group norms."""
        with torch.no_grad():
            x_in = x_in.contiguous()
            want = self._want_stats()
            enc = self.encoder
            ci = enc.conv_init
            if self.in_channels == 1 and tuple(ci.kernel_size) == (3, 3, 3):   # the raw NCDHW window feeds the single-channel stem
                x, st = K.conv_cin1_nc8(x_in, ci.weight, None, 3, 1, 1, want_stats=want)
            else:
                xp, cp = self._pack_input(x_in)
                x, st = self._conv_s1(xp, cp, ci, "init", cin_pad=cp, want_stats=want)

            down = []
            for i, level in enumerate(enc.layers):
                for j, blk in enumerate(level["blocks"]):
                    x, st = self._block_tc(x, st, blk, f"d{i}.{j}", want)
                down.append(x)
                ds = level["downsample"]
                if not isinstance(ds, nn.Identity):
                    k, s, p = (tuple(int(v) for v in t) for t in (ds.kernel_size, ds.stride, ds.padding))
                    x, st = K.conv_gather_tc(x, self._wg(ds, f"d{i}.down", k, s, p), ds.in_channels, ds.out_channels, k, s, p, want_stats=want)
            down.reverse()

            if len(self.blocks_down) > 1:
                for i, level in enumerate(self.up_layers):
                    up, skip = level["upsample"], down[i + 1]
                    if hasattr(up, "deconv"):   # ConvTranspose3d (k3 s2 p1 op1, or k1 s1 on a scale-1 axis), then the skip add
                        dc = up.deconv
                        k, s, p, op = (tuple(int(v) for v in t) for t in (dc.kernel_size, dc.stride, dc.padding, dc.output_padding))
                        z, _ = K.conv_gather_tc(x, self._wg(dc, f"u{i}.up", k, s, p, transposed=True), dc.in_channels, dc.out_channels, k, s, p,
                                                transposed=True, output_padding=op, bias=dc.bias)
                        x, st = K.upsample_add_nc8(z, dc.out_channels, 1, skip, want_stats=want)
                    else:                       # 1x1x1 preconv at the low resolution, then trilinear x2 and the skip add in one pass
                        if hasattr(up, "preconv"):
                            pc = up.preconv
                            x, _ = K.gemm_tc(x, self._wlin(pc.weight, f"u{i}.pre"), pc.in_channels, pc.out_channels, bias=pc.bias)
                        x, st = K.upsample_add_nc8(x, skip.C, 2, skip, want_stats=want)
                    for j, blk in enumerate(level["blocks"]):
                        x, st = self._block_tc(x, st, blk, f"u{i}.{j}", want)

            head = self.up_layers[-1]["head"]
            if head.out_channels <= 16:
                return K.head_conv_nc8(x, head.weight, head.bias, out_dtype=x_in.dtype)
            npad = (head.out_channels + 15) // 16 * 16
            wp, bp = self._whead(head, npad)
            y, _ = K.gemm_tc(x, wp, x.C, npad, bias=bp)
            # the padding channels are dropped by a view (the graph replay returns a contiguous copy)
            return K.unpack_nc8(y, dtype=x_in.dtype).narrow(1, 0, head.out_channels)
