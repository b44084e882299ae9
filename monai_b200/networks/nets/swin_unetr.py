"""`SwinUNETR` (monai/networks/nets/swin_unetr.py:45-330, 919-1075) on Hopper wgmma tensor cores.

The module tree only holds parameters under the reference's names (159 state_dict keys for the default config:
`swinViT.layers1.0.blocks.0.attn.qkv.weight`, `encoder1.layer.conv1.conv.weight`, `decoder5.transp_conv.conv.weight`,
`out.conv.conv.bias`, ...), so reference checkpoints load unchanged.  `forward` never calls a torch op on activations:
the whole network runs on fp16 channel-blocked ("NC8") buffers through the C ABI --

  * 3x3x3 convolutions: implicit GEMM on wgmma (`b200_conv3x3x3_tc`), InstanceNorm partial sums in the epilogue;
  * Linear / 1x1x1 conv / ConvTranspose k2 s2: `b200_gemm_tc` (bias, GELU, residual, window-reverse scatter,
    2x upsample scatter fused in the epilogue);
  * LayerNorm + pad + cyclic shift + window partition: one gather kernel (`b200_layernorm_nc8`);
  * windowed attention with relative-position bias and shift mask: `b200_window_attention_tc` (wgmma), or
    `b200_window_attention_nc8` (mma.sync) for windows it has no schedule for (more than 352 tokens or more than 8 mask patterns);
  * PatchMerging gather + LayerNorm, the single-channel stems and the output head: dedicated kernels.

Skip concatenations are zero-copy: producers write straight into channel slices of the decoder's input buffer.

Supported on this path: spatial_dims=3, any number of input channels (several channels: zero-padded to 16-channel tiles),
feature_size % 48 == 0 with head_dim 16 (the default num_heads for feature_size 48), norm_name="instance" (non-affine),
downsample "merging"/"mergingv2", use_v2 (the residual conv block in front of every stage), inference only.
"""
from __future__ import annotations

import itertools
import warnings
from collections.abc import Sequence

import numpy as np
import torch
import torch.nn as nn

from ... import _kernels as K
from ... import _lib as L
from ._tc_blocks import TcNet
from ..blocks.acti_norm import norm_act_from_modules
from ..blocks.convolutions import Convolution, run_conv_module

__all__ = ["SwinUNETR", "PatchMerging", "PatchMergingV2", "window_plan"]


def _rep(v, n):
    return tuple(v) if isinstance(v, (list, tuple)) else (v,) * n


# ----------------------------------------------------------------------------------------- parameter containers
class PatchEmbed(nn.Module):
    """monai/networks/blocks/patchembedding.py:141-219 (Conv3d k=s=patch_size, optional LayerNorm)."""

    def __init__(self, patch_size, in_chans: int, embed_dim: int, norm_layer=None):
        super().__init__()
        self.patch_size = patch_size
        self.embed_dim = embed_dim
        self.proj = nn.Conv3d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)
        self.norm = norm_layer(embed_dim) if norm_layer is not None else None


class MLPBlock(nn.Module):
    """monai/networks/blocks/mlp.py:25-80 with dropout_mode="swin": linear1 -> GELU -> linear2."""

    def __init__(self, hidden_size: int, mlp_dim: int):
        super().__init__()
        self.linear1 = nn.Linear(hidden_size, mlp_dim)
        self.linear2 = nn.Linear(mlp_dim, hidden_size)
        self.fn = nn.GELU()


class WindowAttention(nn.Module):
    """swin_unetr.py:426-532 (parameters + the relative_position_index buffer)."""

    def __init__(self, dim: int, num_heads: int, window_size: Sequence[int], qkv_bias: bool = False):
        super().__init__()
        self.dim, self.window_size, self.num_heads = dim, tuple(window_size), num_heads
        self.scale = (dim // num_heads) ** -0.5
        ws = self.window_size
        self.relative_position_bias_table = nn.Parameter(torch.zeros((2 * ws[0] - 1) * (2 * ws[1] - 1) * (2 * ws[2] - 1), num_heads))
        coords = torch.stack(torch.meshgrid(torch.arange(ws[0]), torch.arange(ws[1]), torch.arange(ws[2]), indexing="ij")).flatten(1)
        rel = (coords[:, :, None] - coords[:, None, :]).permute(1, 2, 0).contiguous()
        rel[:, :, 0] += ws[0] - 1
        rel[:, :, 1] += ws[1] - 1
        rel[:, :, 2] += ws[2] - 1
        rel[:, :, 0] *= (2 * ws[1] - 1) * (2 * ws[2] - 1)
        rel[:, :, 1] *= 2 * ws[2] - 1
        self.register_buffer("relative_position_index", rel.sum(-1))
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)
        nn.init.trunc_normal_(self.relative_position_bias_table, std=0.02)


class SwinTransformerBlock(nn.Module):
    def __init__(self, dim, num_heads, window_size, shift_size, mlp_ratio=4.0, qkv_bias=True, norm_layer=nn.LayerNorm):
        super().__init__()
        self.dim, self.num_heads, self.window_size, self.shift_size = dim, num_heads, tuple(window_size), tuple(shift_size)
        self.norm1 = norm_layer(dim)
        self.attn = WindowAttention(dim, num_heads, window_size, qkv_bias)
        self.norm2 = norm_layer(dim)
        self.mlp = MLPBlock(dim, int(dim * mlp_ratio))


class PatchMergingV2(nn.Module):
    """swin_unetr.py:701-746 (itertools.product slice order)."""

    v2 = True

    def __init__(self, dim: int, norm_layer=nn.LayerNorm, spatial_dims: int = 3):
        super().__init__()
        self.dim = dim
        self.reduction = nn.Linear(8 * dim, 2 * dim, bias=False)
        self.norm = norm_layer(8 * dim)


class PatchMerging(PatchMergingV2):
    """swin_unetr.py:749-773 (the v0.9.0 slice order x0..x7)."""

    v2 = False


MERGING_MODE = {"merging": PatchMerging, "mergingv2": PatchMergingV2}


class BasicLayer(nn.Module):
    def __init__(self, dim, depth, num_heads, window_size, mlp_ratio, qkv_bias, norm_layer, downsample):
        super().__init__()
        self.window_size = tuple(window_size)
        self.shift_size = tuple(i // 2 for i in window_size)
        self.no_shift = tuple(0 for _ in window_size)
        self.depth = depth
        self.blocks = nn.ModuleList(
            [
                SwinTransformerBlock(dim, num_heads, self.window_size, self.no_shift if i % 2 == 0 else self.shift_size, mlp_ratio, qkv_bias, norm_layer)
                for i in range(depth)
            ]
        )
        self.downsample = downsample(dim=dim, norm_layer=norm_layer, spatial_dims=3) if downsample is not None else None


class SwinTransformer(nn.Module):
    def __init__(self, in_chans, embed_dim, window_size, patch_size, depths, num_heads, mlp_ratio=4.0, qkv_bias=True,
                 norm_layer=nn.LayerNorm, patch_norm=False, downsample="merging", use_v2=False):
        super().__init__()
        self.use_v2 = use_v2
        self.num_layers = len(depths)
        self.embed_dim, self.patch_norm, self.window_size, self.patch_size = embed_dim, patch_norm, tuple(window_size), tuple(patch_size)
        self.patch_embed = PatchEmbed(self.patch_size, in_chans, embed_dim, norm_layer if patch_norm else None)
        self.pos_drop = nn.Dropout(p=0.0)
        self.layers1, self.layers2, self.layers3, self.layers4 = nn.ModuleList(), nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        down = MERGING_MODE[downsample] if isinstance(downsample, str) else downsample
        if use_v2:   # SwinUNETR-V2: a residual convolution block in front of every stage (swin_unetr.py:990-1036)
            self.layers1c, self.layers2c, self.layers3c, self.layers4c = nn.ModuleList(), nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        for i in range(self.num_layers):
            layer = BasicLayer(int(embed_dim * 2**i), depths[i], num_heads[i], self.window_size, mlp_ratio, qkv_bias, norm_layer, down)
            (self.layers1, self.layers2, self.layers3, self.layers4)[i].append(layer)
            if use_v2:
                (self.layers1c, self.layers2c, self.layers3c, self.layers4c)[i].append(UnetrBasicBlock(int(embed_dim * 2**i), int(embed_dim * 2**i)))
        self.num_features = int(embed_dim * 2 ** (self.num_layers - 1))


class UnetResBlock(nn.Module):
    """monai/networks/blocks/dynunet_block.py:25-111 (containers; kernel 3, stride 1, instance norm, LeakyReLU 0.01)."""

    def __init__(self, in_channels: int, out_channels: int):
        super().__init__()
        kw = dict(strides=1, act=None, norm=None, dropout=None, bias=False, conv_only=False)
        self.conv1 = Convolution(3, in_channels, out_channels, kernel_size=3, padding=1, **kw)
        self.conv2 = Convolution(3, out_channels, out_channels, kernel_size=3, padding=1, **kw)
        self.lrelu = nn.LeakyReLU(negative_slope=0.01, inplace=True)
        self.norm1 = nn.InstanceNorm3d(out_channels)
        self.norm2 = nn.InstanceNorm3d(out_channels)
        self.downsample = in_channels != out_channels
        if self.downsample:
            self.conv3 = Convolution(3, in_channels, out_channels, kernel_size=1, padding=0, **kw)
            self.norm3 = nn.InstanceNorm3d(out_channels)


class UnetrBasicBlock(nn.Module):
    def __init__(self, in_channels: int, out_channels: int):
        super().__init__()
        self.layer = UnetResBlock(in_channels, out_channels)


class UnetrUpBlock(nn.Module):
    def __init__(self, in_channels: int, out_channels: int):
        super().__init__()
        self.transp_conv = Convolution(3, in_channels, out_channels, strides=2, kernel_size=2, act=None, norm=None, dropout=None,
                                       bias=False, conv_only=True, is_transposed=True, padding=0, output_padding=0)
        self.conv_block = UnetResBlock(out_channels + out_channels, out_channels)


class UnetOutBlock(nn.Module):
    def __init__(self, in_channels: int, out_channels: int):
        super().__init__()
        self.conv = Convolution(3, in_channels, out_channels, strides=1, kernel_size=1, act=None, norm=None, dropout=None, bias=True,
                                conv_only=False, padding=0)


# --------------------------------------------------------------------------------------------- host-side planning
def _get_window_size(x_size, window_size, shift_size):
    """swin_unetr.py:399-423: clamp the window to the feature map and drop the shift on clamped axes."""
    ws, ss = list(window_size), list(shift_size)
    for i in range(len(x_size)):
        if x_size[i] <= window_size[i]:
            ws[i] = x_size[i]
            ss[i] = 0
    return tuple(ws), tuple(ss)


def window_plan(dims, window_size, shift_size):
    """Index tables for pad + roll(-shift) + window_partition (swin_unetr.py:596-625) and compute_mask (779-816).

    Returns (src int32 [nW*n] with -1 for zero-padded tokens, region int32 [nW, n] or None, nW, n).
    Row r of the windowed tensor is token src[r] of the (d,h,w) grid; window_reverse + roll(+shift) + crop is the
    inverse of the same table, so the projection GEMM scatters through it."""
    ws, ss = _get_window_size(dims, window_size, shift_size)
    pdims = [int(np.ceil(d / w)) * w for d, w in zip(dims, ws)]
    grids = []
    for ax in range(3):
        p = np.arange(pdims[ax])                       # coordinate in the shifted, padded volume
        o = (p + ss[ax]) % pdims[ax]                   # coordinate in the padded volume before the roll
        grids.append((p, o))
    P = np.stack(np.meshgrid(grids[0][0], grids[1][0], grids[2][0], indexing="ij"), -1)
    O = np.stack(np.meshgrid(grids[0][1], grids[1][1], grids[2][1], indexing="ij"), -1)
    valid = (O[..., 0] < dims[0]) & (O[..., 1] < dims[1]) & (O[..., 2] < dims[2])
    lin = (O[..., 0] * dims[1] + O[..., 1]) * dims[2] + O[..., 2]
    lin = np.where(valid, lin, -1)

    def part(a):  # window_partition on a (dp,hp,wp) array
        a = a.reshape(pdims[0] // ws[0], ws[0], pdims[1] // ws[1], ws[1], pdims[2] // ws[2], ws[2])
        return a.transpose(0, 2, 4, 1, 3, 5).reshape(-1, ws[0] * ws[1] * ws[2])

    src = part(lin).astype(np.int32)
    region = None
    if any(s > 0 for s in ss):
        lab = np.zeros(pdims, dtype=np.int32)
        for ax in range(3):
            p = P[..., ax]
            if ss[ax] > 0:
                a = np.where(p < pdims[ax] - ws[ax], 0, np.where(p < pdims[ax] - ss[ax], 1, 2))
            else:
                a = np.zeros_like(p)  # all three slices collapse onto the whole axis: a single label
            lab = lab * 3 + a
        region = part(lab).astype(np.int32)
    return src.reshape(-1), region, src.shape[0], src.shape[1]


class SwinUNETR(TcNet, nn.Module):
    patch_size: int = 2

    def __init__(
        self,
        in_channels: int,
        out_channels: int,
        patch_size: int = 2,
        depths: Sequence[int] = (2, 2, 2, 2),
        num_heads: Sequence[int] = (3, 6, 12, 24),
        window_size: Sequence[int] | int = 7,
        qkv_bias: bool = True,
        mlp_ratio: float = 4.0,
        feature_size: int = 24,
        norm_name: tuple | str = "instance",
        drop_rate: float = 0.0,
        attn_drop_rate: float = 0.0,
        dropout_path_rate: float = 0.0,
        normalize: bool = True,
        norm_layer: type[nn.LayerNorm] = nn.LayerNorm,
        patch_norm: bool = False,
        use_checkpoint: bool = False,
        spatial_dims: int = 3,
        downsample: str | nn.Module = "merging",
        use_v2: bool = False,
        img_size: Sequence[int] | int | None = None,  # accepted and ignored (older bundles pass it; SURVEY.md section 0)
    ) -> None:
        super().__init__()
        if spatial_dims not in (2, 3):
            raise ValueError("spatial dimension should be 2 or 3.")
        for name, v in (("dropout rate", drop_rate), ("attention dropout rate", attn_drop_rate), ("drop path rate", dropout_path_rate)):
            if not (0 <= v <= 1):
                raise ValueError(f"{name} should be between 0 and 1.")
        if feature_size % 12 != 0:
            raise ValueError("feature_size should be divisible by 12.")
        if spatial_dims != 3:
            raise NotImplementedError("monai_b200 SwinUNETR implements spatial_dims=3")
        # The tensor-core path needs 16-channel multiples (feature_size % 48 == 0) and head_dim 16; every other configuration of the
        # reference (e.g. its default feature_size = 24: head_dim 8) runs on the generic fp32-faithful kernels (_forward_generic).
        head_dims = [(feature_size * 2**i) // h for i, h in enumerate(num_heads)]
        if any((feature_size * 2**i) % h for i, h in enumerate(num_heads)) or any(d not in (8, 16, 24, 32, 48, 64) for d in head_dims):
            raise NotImplementedError(f"monai_b200 window attention supports head dimensions 8, 16, 24, 32, 48, 64 (got {head_dims})")
        self._tc_ok = feature_size % 48 == 0 and all(d == 16 for d in head_dims)
        self.fp32_faithful = False   # set True to run fp32-storage generic kernels: <= 1e-3 of the fp32 reference
        nn_name = norm_name if isinstance(norm_name, str) else norm_name[0]
        if str(nn_name).lower() != "instance" or (not isinstance(norm_name, str) and norm_name[1].get("affine")):
            raise NotImplementedError("monai_b200 SwinUNETR implements norm_name='instance' (non-affine)")
        if patch_size != 2:
            raise NotImplementedError("monai_b200 SwinUNETR implements patch_size=2")
        self.patch_size = patch_size
        self.normalize = normalize
        self.feature_size = feature_size
        self.out_channels = out_channels
        self.in_channels = in_channels
        if in_channels < 1:
            raise ValueError("in_channels must be positive")
        self.use_v2 = use_v2
        ws = _rep(window_size, 3)
        self.swinViT = SwinTransformer(in_channels, feature_size, ws, _rep(patch_size, 3), depths, num_heads, mlp_ratio, qkv_bias,
                                       norm_layer, patch_norm, downsample, use_v2)
        fs = feature_size
        self.encoder1 = UnetrBasicBlock(in_channels, fs)
        self.encoder2 = UnetrBasicBlock(fs, fs)
        self.encoder3 = UnetrBasicBlock(2 * fs, 2 * fs)
        self.encoder4 = UnetrBasicBlock(4 * fs, 4 * fs)
        self.encoder10 = UnetrBasicBlock(16 * fs, 16 * fs)
        self.decoder5 = UnetrUpBlock(16 * fs, 8 * fs)
        self.decoder4 = UnetrUpBlock(8 * fs, 4 * fs)
        self.decoder3 = UnetrUpBlock(4 * fs, 2 * fs)
        self.decoder2 = UnetrUpBlock(2 * fs, fs)
        self.decoder1 = UnetrUpBlock(fs, fs)
        self.out = UnetOutBlock(fs, out_channels)
        self._tc_setup()

    def _check_input_size(self, spatial_shape):
        img_size = np.array(spatial_shape)
        remainder = (img_size % np.power(self.patch_size, 5)) > 0
        if remainder.any():
            wrong_dims = (np.where(remainder)[0] + 2).tolist()
            raise ValueError(
                f"spatial dimensions {wrong_dims} of input image (spatial shape: {spatial_shape})"
                f" must be divisible by {self.patch_size}**5."
            )

    # ----------------------------------------------------------------------------------------------- weight prep
    def _plan(self, dims, ws, ss, dev):
        def build():
            src, region, nW, n = window_plan(dims, ws, ss)
            # schedule of the tensor-core attention: windows grouped by shift-mask pattern (at most 8 patterns)
            sched, reps, ntypes = K.window_attention_tc_plan(region, nW, n)
            tc = None
            if ntypes <= 8 and n <= 352:
                tc = (torch.from_numpy(sched).to(dev), None if reps is None else torch.from_numpy(reps).contiguous().to(dev), ntypes)
            return (torch.from_numpy(src).to(dev), None if region is None else torch.from_numpy(region).to(dev), nW, n, tc)

        return self._cache.get(("plan", tuple(dims), tuple(ws), tuple(ss), dev), [], build)

    def _attn_bias(self, attn: WindowAttention, key, n: int, tc):
        _, reps, ntypes = tc
        return self._cache.get(("attnb", key, n, ntypes, attn.relative_position_bias_table.device), [attn.relative_position_bias_table],
                               lambda: K.window_attention_tc_pack_bias(attn.relative_position_bias_table, attn.num_heads, n, attn.window_size, reps, ntypes))

    # ------------------------------------------------------------------------------------------------- sub-graphs
    def _swin_stage(self, cur: K.NC8, layer: BasicLayer, key: str, pre: UnetrBasicBlock | None = None) -> K.NC8:
        dims, C = cur.sp, cur.C
        dev = cur.buf.device
        if pre is not None:   # SwinUNETR-V2: residual conv block on the token grid (swin_unetr.py:1059-1072)
            cur = self._res_block(cur, C, 0, pre.layer, key + ".c")
        for bi, blk in enumerate(layer.blocks):
            ws, ss = _get_window_size(dims, blk.window_size, blk.shift_size)
            src, region, nW, n, tc = self._plan(dims, ws, ss, dev)
            bkey = f"{key}.b{bi}"
            xw = K.layernorm_nc8(cur, blk.norm1.weight, blk.norm1.bias, blk.norm1.eps, src=src, out_sp=(1, nW, n))
            if tc is not None:
                # tensor-core attention: S accumulates onto the packed bias + shift mask, scores in log2 units
                wq, bq = self._wqkv_scaled(blk.attn.qkv.weight, blk.attn.qkv.bias, C, blk.attn.scale, bkey)
                qkv, _ = K.gemm_tc(xw, wq, C, 3 * C, bias=bq)
                att = K.window_attention_tc(qkv, C, blk.num_heads, nW, n, self._attn_bias(blk.attn, (bkey, tuple(dims), tuple(ws), tuple(ss)), n, tc), tc[0], tc[2])
            else:
                # mma.sync attention: windows without a wgmma schedule (more than 352 tokens or more than 8 shift-mask patterns)
                qkv, _ = K.gemm_tc(xw, self._wlin(blk.attn.qkv.weight, bkey + ".qkv"), C, 3 * C, bias=blk.attn.qkv.bias)
                att = K.window_attention_nc8(qkv, C, blk.num_heads, nW, n, blk.attn.scale, blk.attn.relative_position_bias_table, blk.attn.window_size,
                                             region if any(s > 0 for s in ss) else None)
            # x = shortcut + window_reverse(proj(att)): scattered back through the same table, residual fused
            x1, _ = K.gemm_tc(att, self._wlin(blk.attn.proj.weight, bkey + ".proj"), C, C, bias=blk.attn.proj.bias, res=cur, row_map=src, out_sp=dims, mode=1)
            hid = blk.mlp.linear1.out_features
            w1, w2 = self._wlin(blk.mlp.linear1.weight, bkey + ".fc1"), self._wlin(blk.mlp.linear2.weight, bkey + ".fc2")
            if K.mlp_fused_supported(C, hid):
                # x = x + mlp(norm2(x)) in one launch: the 4C-wide hidden tensor never reaches HBM
                cur = K.mlp_fused_tc(x1, w1, blk.mlp.linear1.bias, w2, blk.mlp.linear2.bias, hid, blk.norm2.weight, blk.norm2.bias, blk.norm2.eps)
            else:
                y = K.layernorm_nc8(x1, blk.norm2.weight, blk.norm2.bias, blk.norm2.eps)
                h, _ = K.gemm_tc(y, w1, C, hid, bias=blk.mlp.linear1.bias, act=L.ACT_GELU)
                cur, _ = K.gemm_tc(h, w2, hid, C, bias=blk.mlp.linear2.bias, res=x1)
        if layer.downsample is not None:
            ds = layer.downsample
            m = K.patch_merge_ln_nc8(cur, ds.norm.weight, ds.norm.bias, ds.norm.eps, v2=ds.v2)
            cur, _ = K.gemm_tc(m, self._wlin(ds.reduction.weight, key + ".red"), 8 * C, 2 * C)
        return cur

    def _proj_out(self, t: K.NC8, out: K.NC8 | None = None, out_coff: int = 0) -> K.NC8:
        """SwinTransformer.proj_out (swin_unetr.py:1040-1053): channel LayerNorm without affine when normalize=True."""
        if not self.normalize:
            if out is None:
                return t
            return K.norm_act_nc8(t, t.C, None, out=out, out_coff=out_coff)
        if out is None:
            return K.layernorm_nc8(t, None, None, 1e-5)
        # LayerNorm into a private buffer, then place into the concat slice (layernorm writes whole buffers)
        tmp = K.layernorm_nc8(t, None, None, 1e-5)
        return K.norm_act_nc8(tmp, t.C, None, out=out, out_coff=out_coff)

    def _check_input(self, x_in: torch.Tensor) -> None:
        if not x_in.is_cuda:
            raise RuntimeError("monai_b200.SwinUNETR runs on CUDA tensors only (there is no CPU fallback)")
        self._check_input_size(x_in.shape[2:])
        if x_in.shape[1] != self.in_channels:
            raise ValueError(f"expected {self.in_channels} input channel(s), got {x_in.shape[1]}")
        if x_in.dtype not in (torch.float16, torch.float32):
            raise TypeError(f"SwinUNETR takes float16/float32 inputs, got {x_in.dtype}")

    def _use_tc(self, x_in: torch.Tensor) -> bool:
        return self._tc_ok and not self.fp32_faithful

    def _check_tc_input(self, x_in: torch.Tensor) -> None:
        if x_in.dtype == torch.float32 and not getattr(self, "_warned_fp32", False):
            # no silent degradation: the tensor-core path stores activations in fp16 (fp32 accumulation everywhere); an fp32
            # input gets fp32 logits of that fp16-storage computation (DESIGN.md section 2: measured ~5e-3 of the output scale)
            warnings.warn("monai_b200.SwinUNETR computes with fp16 activation storage (fp32 accumulation); float32 inputs are converted. "
                          "Expect ~1e-2 relative agreement with an fp32 reference, not 1e-3 (set net.fp32_faithful = True for the fp32 path).")
            self._warned_fp32 = True

    # --------------------------------------------------------------------------- fp32-faithful generic path
    def _plan_direct(self, dims, ws, ss, dev):
        """window_plan tables on the device + the inverse table (token -> row of the windowed tensor) for window_reverse."""
        def build():
            src, region, nW, n = window_plan(dims, ws, ss)
            inv = np.full(int(np.prod(dims)), -1, dtype=np.int32)
            rows = np.nonzero(src >= 0)[0]
            inv[src[rows]] = rows.astype(np.int32)
            return (torch.from_numpy(src).to(dev), None if region is None else torch.from_numpy(np.ascontiguousarray(region)).to(dev),
                    torch.from_numpy(inv).to(dev), nW, n)

        return self._cache.get(("plan_direct", tuple(dims), tuple(ws), tuple(ss), dev), [], build)

    def _dense_bias(self, attn: WindowAttention, n: int, key):
        """relative_position_bias_table[relative_position_index[:n, :n]] as float32 [heads, n, n] (swin_unetr.py:514-518)."""
        def build():
            idx = attn.relative_position_index[:n, :n].reshape(-1)
            return attn.relative_position_bias_table.detach().float()[idx].reshape(n, n, -1).permute(2, 0, 1).contiguous()

        return self._cache.get(("dense_bias", key, n, attn.relative_position_bias_table.device), [attn.relative_position_bias_table], build)

    def _merge_params(self, ds, C: int, key):
        """PatchMerging on the patchified tensor: b200_patchify orders the 8C channels (c, offset a*4 + b*2 + e), the reference
        concatenates offset-major in its slice order (swin_unetr.py:726-773); permute LayerNorm affine and reduction columns once."""
        def build():
            order = list(itertools.product(range(2), range(2), range(2))) if ds.v2 else \
                [(0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 1, 1)]
            ref_of_pat = np.empty(8 * C, dtype=np.int64)       # reference channel index of every patchified channel
            for k, (a, b, e) in enumerate(order):
                for c in range(C):
                    ref_of_pat[c * 8 + a * 4 + b * 2 + e] = k * C + c
            idx = torch.from_numpy(ref_of_pat).to(ds.norm.weight.device)
            return (ds.norm.weight.detach().float()[idx].contiguous(), ds.norm.bias.detach().float()[idx].contiguous(),
                    ds.reduction.weight.detach().float()[:, idx].contiguous())

        return self._cache.get(("merge", key, C, ds.norm.weight.device), [ds.norm.weight, ds.norm.bias, ds.reduction.weight], build)

    @staticmethod
    def _lin(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor | None) -> torch.Tensor:
        """nn.Linear over the channel axis of channels-first tokens [N, Cin, S] (a 1x1x1 convolution with fp32 accumulation)."""
        N, Cin, S = x.shape
        return K.conv3d_direct(x.reshape(N, Cin, 1, 1, S), weight.reshape(weight.shape[0], Cin, 1, 1, 1), bias).reshape(N, weight.shape[0], S)

    @staticmethod
    def _res_block_direct(x: torch.Tensor, blk: UnetResBlock) -> torch.Tensor:
        """UnetResBlock.forward (dynunet_block.py:97-111) on NCDHW tensors."""
        out = norm_act_from_modules(run_conv_module(blk.conv1.conv, x), blk.norm1, blk.lrelu)
        out = run_conv_module(blk.conv2.conv, out)
        res = x
        if hasattr(blk, "conv3"):
            res = norm_act_from_modules(run_conv_module(blk.conv3.conv, x), blk.norm3, None)
        return norm_act_from_modules(out, blk.norm2, blk.lrelu, res=res)

    def _swin_stage_direct(self, t: torch.Tensor, layer: BasicLayer, key: str, pre: UnetrBasicBlock | None) -> torch.Tensor:
        """BasicLayer.forward (swin_unetr.py:819-916) on a channels-first [N, C, d, h, w] tensor."""
        if pre is not None:
            t = self._res_block_direct(t, pre.layer)
        N, C = t.shape[:2]
        dims = tuple(int(v) for v in t.shape[2:])
        S = dims[0] * dims[1] * dims[2]
        x = t.reshape(N, C, S)
        add = lambda a, b: K.norm_act(a, None, res=b, act=L.ACT_NONE)   # noqa: E731
        for bi, blk in enumerate(layer.blocks):
            ws, ss = _get_window_size(dims, blk.window_size, blk.shift_size)
            src, region, inv, nW, n = self._plan_direct(dims, ws, ss, t.device)
            h = K.layernorm_cf(x, blk.norm1.weight, blk.norm1.bias, blk.norm1.eps)
            hw = K.gather_cf(h, src)                                                       # pad + roll + window_partition
            qkv = self._lin(hw, blk.attn.qkv.weight, blk.attn.qkv.bias)
            att = K.mhsa_cf(qkv, blk.num_heads, C // blk.num_heads, blk.attn.scale, win=n, bias=self._dense_bias(blk.attn, n, f"{key}.b{bi}"),
                            region=region.reshape(-1) if (region is not None and any(s_ > 0 for s_ in ss)) else None)
            o = self._lin(att, blk.attn.proj.weight, blk.attn.proj.bias)
            x = add(K.gather_cf(o, inv), x)                                                # window_reverse + roll back + crop, shortcut
            h2 = K.layernorm_cf(x, blk.norm2.weight, blk.norm2.bias, blk.norm2.eps)
            m = K.norm_act(self._lin(h2, blk.mlp.linear1.weight, blk.mlp.linear1.bias), None, act=L.ACT_GELU)
            x = add(self._lin(m, blk.mlp.linear2.weight, blk.mlp.linear2.bias), x)
        t = x.reshape(N, C, *dims)
        if layer.downsample is not None:
            if any(d % 2 for d in dims):
                raise NotImplementedError("monai_b200 SwinUNETR (generic path): odd token grids in PatchMerging are not implemented")
            g, b, w = self._merge_params(layer.downsample, C, key)
            cols = K.patchify(t, (2, 2, 2))                                                # [N, 8C, S / 8]
            cols = K.layernorm_cf(cols, g, b, layer.downsample.norm.eps)
            t = self._lin(cols, w, None).reshape(N, 2 * C, *(d // 2 for d in dims))
        return t

    def _forward_generic(self, x_in: torch.Tensor) -> torch.Tensor:
        """SwinUNETR.forward (swin_unetr.py:316-330) on the generic kernels: activations keep the input's dtype (float32: the
        reference's arithmetic to <= 1e-3), every product accumulates in fp32.  Any feature_size / head dimension of the reference."""
        with torch.no_grad():
            x_in = x_in.contiguous()
            vit = self.swinViT
            pe = vit.patch_embed

            def proj_out(t):
                if not self.normalize:
                    return t
                N, C = t.shape[:2]
                return K.layernorm_cf(t.reshape(N, C, -1), None, None, 1e-5).reshape(t.shape)

            t0 = run_conv_module(pe.proj, x_in)
            if pe.norm is not None:
                N, C = t0.shape[:2]
                t0 = K.layernorm_cf(t0.reshape(N, C, -1), pe.norm.weight, pe.norm.bias, pe.norm.eps).reshape(t0.shape)
            v2 = (lambda i: getattr(vit, f"layers{i}c")[0]) if self.use_v2 else (lambda i: None)
            hs = [proj_out(t0)]
            t = t0
            for i in range(1, 5):
                t = self._swin_stage_direct(t, getattr(vit, f"layers{i}")[0], f"d{i}", v2(i))
                hs.append(proj_out(t))
            enc0 = self._res_block_direct(x_in, self.encoder1.layer)
            enc1 = self._res_block_direct(hs[0], self.encoder2.layer)
            enc2 = self._res_block_direct(hs[1], self.encoder3.layer)
            enc3 = self._res_block_direct(hs[2], self.encoder4.layer)
            dec4 = self._res_block_direct(hs[4], self.encoder10.layer)

            def up(inp, skip, block: UnetrUpBlock):
                return self._res_block_direct(K.cat_channels([block.transp_conv(inp), skip]), block.conv_block)

            dec3 = up(dec4, hs[3], self.decoder5)
            dec2 = up(dec3, enc3, self.decoder4)
            dec1 = up(dec2, enc2, self.decoder3)
            dec0 = up(dec1, enc1, self.decoder2)
            out = up(dec0, enc0, self.decoder1)
            return self.out.conv(out)

    def _forward_tc(self, x_in: torch.Tensor) -> torch.Tensor:
        with torch.no_grad():
            x_in = x_in.contiguous()
            n = x_in.shape[0]
            dev = x_in.device
            fs = self.feature_size
            sp0 = tuple(int(s) for s in x_in.shape[2:])
            sp = [tuple(s // (2 ** (i + 1)) for s in sp0) for i in range(5)]  # resolutions of hidden states 0..4
            vit = self.swinViT

            # decoder input buffers: [upsampled | skip] channel slices, written in place by their producers
            cat1 = K.NC8(n, 2 * fs, sp0, dev)       # decoder1: [up(dec0) | enc0]
            cat2 = K.NC8(n, 2 * fs, sp[0], dev)     # decoder2: [up(dec1) | enc1]
            cat3 = K.NC8(n, 4 * fs, sp[1], dev)     # decoder3: [up(dec2) | enc2]
            cat4 = K.NC8(n, 8 * fs, sp[2], dev)     # decoder4: [up(dec3) | enc3]
            cat5 = K.NC8(n, 16 * fs, sp[3], dev)    # decoder5: [up(dec4) | hidden3]

            # ---- Swin transformer encoder (swin_unetr.py:1055-1075)
            pe = vit.patch_embed
            xp = None
            if self.in_channels == 1:
                t0, _ = K.conv_cin1_nc8(x_in, pe.proj.weight, pe.proj.bias, 2, 2, 0)
            else:
                # several input channels: the volume is repacked once and the stems run on the general tensor-core kernels with
                # zero-padded weights
                xp, cp = self._pack_input(x_in)
                pw = self._cache.get(("pe", cp, pe.proj.weight.device), [pe.proj.weight],
                                     lambda: K.conv_gather_tc_pack_weight(self._pad_cin(pe.proj.weight, cp), 2, 2, 0, False))
                t0, _ = K.conv_gather_tc(xp, pw, cp, fs, 2, 2, 0, bias=pe.proj.bias)
            if pe.norm is not None:
                t0 = K.layernorm_nc8(t0, pe.norm.weight, pe.norm.bias, pe.norm.eps)
            v2 = (lambda i: getattr(vit, f"layers{i}c")[0]) if self.use_v2 else (lambda i: None)
            h0 = self._proj_out(t0)
            t1 = self._swin_stage(t0, vit.layers1[0], "l1", v2(1))
            h1 = self._proj_out(t1)
            t2 = self._swin_stage(t1, vit.layers2[0], "l2", v2(2))
            h2 = self._proj_out(t2)
            t3 = self._swin_stage(t2, vit.layers3[0], "l3", v2(3))
            self._proj_out(t3, out=cat5, out_coff=8 * fs)
            t4 = self._swin_stage(t3, vit.layers4[0], "l4", v2(4))
            h4 = self._proj_out(t4)

            # ---- CNN encoders on the hidden states (swin_unetr.py:319-324)
            if xp is None:
                self._res_block(None, 1, 0, self.encoder1.layer, "enc1", out=cat1, out_coff=fs, x_in_raw=x_in)
            else:
                self._res_block(xp, cp, 0, self.encoder1.layer, "enc1", out=cat1, out_coff=fs, cin_pad=cp)
            self._res_block(h0, fs, 0, self.encoder2.layer, "enc2", out=cat2, out_coff=fs)
            self._res_block(h1, 2 * fs, 0, self.encoder3.layer, "enc3", out=cat3, out_coff=2 * fs)
            self._res_block(h2, 4 * fs, 0, self.encoder4.layer, "enc4", out=cat4, out_coff=4 * fs)
            dec4 = self._res_block(h4, 16 * fs, 0, self.encoder10.layer, "enc10")

            # ---- decoders: ConvTranspose k2 s2 scatter into the concat buffer, then the residual block
            dec3 = self._up_block(dec4, 16 * fs, self.decoder5, cat5, "dec5")
            dec2 = self._up_block(dec3, 8 * fs, self.decoder4, cat4, "dec4")
            dec1 = self._up_block(dec2, 4 * fs, self.decoder3, cat3, "dec3")
            dec0 = self._up_block(dec1, 2 * fs, self.decoder2, cat2, "dec2")
            # decoder1's norm2 + residual + lrelu is applied by the output head on its operand load (one pass less over 96^3 x 48)
            tail = self._up_block(dec0, fs, self.decoder1, cat1, "dec1", defer_tail=True)
            return self._tail_head(tail, self.decoder1.conv_block, self.out.conv.conv, x_in.dtype)
