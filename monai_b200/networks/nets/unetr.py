"""UNETR (monai/networks/nets/unetr.py:24-213; Hatamizadeh et al.) behind the reference's constructor, module tree and state_dict
keys (SURVEY.md §8 row f4): a ViT encoder on 16^3 patches whose hidden states 3 / 6 / 9 / 12 feed a convolutional decoder
(projection up-blocks, transposed convolutions, residual blocks); inference only.

Two forwards, chosen from the input and the configuration (DESIGN.md §8.4):
  * fp16 CUDA input, head_dim 64, feature_size % 16 == 0, mlp_dim % 16 == 0, out_channels <= 16, non-affine instance norm and
    residual conv blocks (the reference's defaults): `_forward_tc`, the whole network on fp16 channel-blocked (NC8) buffers and
    Hopper tensor cores -- `b200_gemm_tc` for every Linear, the patch embedding and the transposed convolutions,
    `b200_mhsa_tc` for the attention, `b200_conv3x3x3_tc` for the decoder, replayed from a CUDA graph per input shape;
  * everything else: `_forward_generic`, the fp32-faithful generic kernels (b200_conv3d_direct for convolutions AND linear
    layers, b200_layernorm_cf, b200_mhsa_cf, b200_instnorm_stats + b200_norm_act)."""
from __future__ import annotations

from typing import Sequence

import torch
import torch.nn as nn

from ... import _kernels as K
from ... import _lib as L
from .._graph import GraphedForward
from ..blocks.dynunet_block import UnetOutBlock
from ..blocks.unetr_block import UnetrBasicBlock, UnetrPrUpBlock, UnetrUpBlock
from ._tc_blocks import TcBlocks, _Cache
from .vit import ViT

__all__ = ["UNETR"]


def _instance_non_affine(norm_name) -> bool:
    name, args = (norm_name, {}) if isinstance(norm_name, str) else (norm_name[0], norm_name[1] if len(norm_name) > 1 else {})
    return str(name).lower() in ("instance", "instancenorm") and not args.get("affine", False)


class UNETR(TcBlocks, GraphedForward, nn.Module):
    def __init__(self, in_channels: int, out_channels: int, img_size: Sequence[int] | int, feature_size: int = 16, hidden_size: int = 768,
                 mlp_dim: int = 3072, num_heads: int = 12, proj_type: str = "conv", norm_name="instance", conv_block: bool = True,
                 res_block: bool = True, dropout_rate: float = 0.0, spatial_dims: int = 3, qkv_bias: bool = False, save_attn: bool = False) -> None:
        super().__init__()
        if not (0 <= dropout_rate <= 1):
            raise ValueError("dropout_rate should be between 0 and 1.")
        if hidden_size % num_heads != 0:
            raise ValueError("hidden_size should be divisible by num_heads.")
        self.num_layers = 12
        img_size = (img_size,) * spatial_dims if isinstance(img_size, int) else tuple(img_size)
        self.patch_size = (16,) * spatial_dims
        self.feat_size = tuple(i // p for i, p in zip(img_size, self.patch_size))
        self.hidden_size = hidden_size
        self.classification = False
        self.vit = ViT(in_channels=in_channels, img_size=img_size, patch_size=self.patch_size, hidden_size=hidden_size, mlp_dim=mlp_dim,
                       num_layers=self.num_layers, num_heads=num_heads, proj_type=proj_type, classification=False, dropout_rate=dropout_rate,
                       spatial_dims=spatial_dims, qkv_bias=qkv_bias, save_attn=save_attn)
        sd, f = spatial_dims, feature_size
        self.encoder1 = UnetrBasicBlock(sd, in_channels, f, kernel_size=3, stride=1, norm_name=norm_name, res_block=res_block)
        pr = dict(kernel_size=3, stride=1, upsample_kernel_size=2, norm_name=norm_name, conv_block=conv_block, res_block=res_block)
        self.encoder2 = UnetrPrUpBlock(sd, hidden_size, f * 2, num_layer=2, **pr)
        self.encoder3 = UnetrPrUpBlock(sd, hidden_size, f * 4, num_layer=1, **pr)
        self.encoder4 = UnetrPrUpBlock(sd, hidden_size, f * 8, num_layer=0, **pr)
        up = dict(kernel_size=3, upsample_kernel_size=2, norm_name=norm_name, res_block=res_block)
        self.decoder5 = UnetrUpBlock(sd, hidden_size, f * 8, **up)
        self.decoder4 = UnetrUpBlock(sd, f * 8, f * 4, **up)
        self.decoder3 = UnetrUpBlock(sd, f * 4, f * 2, **up)
        self.decoder2 = UnetrUpBlock(sd, f * 2, f, **up)
        self.out = UnetOutBlock(spatial_dims=sd, in_channels=f, out_channels=out_channels)
        self.in_channels, self.feature_size, self.num_heads, self.mlp_dim = in_channels, feature_size, num_heads, mlp_dim
        # configurations the tensor-core forward implements (every other one keeps the generic path)
        self._tc_ok = (spatial_dims == 3 and hidden_size // num_heads == 64 and feature_size % 16 == 0 and mlp_dim % 16 == 0
                       and out_channels <= 16 and _instance_non_affine(norm_name) and conv_block and res_block)
        self._cache = _Cache()
        self._graph_init()  # the ~150 launches of one tensor-core forward are captured into a CUDA graph per input shape

    def proj_feat(self, x: torch.Tensor) -> torch.Tensor:
        """tokens -> feature map.  The reference permutes [N, S, hidden] to [N, hidden, *feat_size]; tokens are already channels-first here."""
        return x.reshape(x.shape[0], self.hidden_size, *self.feat_size)

    def forward(self, x_in: torch.Tensor) -> torch.Tensor:
        if tuple(x_in.shape[2:]) != tuple(f * p for f, p in zip(self.feat_size, self.patch_size)):
            raise ValueError(f"UNETR was built for inputs of size {tuple(f * p for f, p in zip(self.feat_size, self.patch_size))}, got {tuple(x_in.shape[2:])}")
        if not (self._tc_ok and x_in.is_cuda and x_in.dtype == torch.float16):
            return self._forward_generic(x_in)
        if x_in.shape[1] != self.in_channels:
            raise ValueError(f"expected {self.in_channels} input channel(s), got {x_in.shape[1]}")
        if self._graph_ok():
            return self._forward_graphed(x_in, self._forward_tc)
        return self._forward_tc(x_in)

    def _forward_generic(self, x_in: torch.Tensor) -> torch.Tensor:
        x, hidden = self.vit(x_in)
        enc1 = self.encoder1(x_in)
        enc2 = self.encoder2(self.proj_feat(hidden[3]))
        enc3 = self.encoder3(self.proj_feat(hidden[6]))
        enc4 = self.encoder4(self.proj_feat(hidden[9]))
        dec3 = self.decoder5(self.proj_feat(x), enc4)
        dec2 = self.decoder4(dec3, enc3)
        dec1 = self.decoder3(dec2, enc2)
        return self.out(self.decoder2(dec1, enc1))

    # ------------------------------------------------------------------------------------------- tensor-core path
    def _pos_nc8(self, n: int, dev) -> K.NC8:
        """The learnable position embedding [1, S, hidden] as an NC8 residual operand expanded to the batch."""
        pos = self.vit.patch_embedding.position_embeddings

        def build():
            p = pos.detach().float().transpose(1, 2).reshape(1, self.hidden_size, *self.feat_size)
            return K.pack_nc8(p.expand(n, -1, -1, -1, -1).contiguous())

        return self._cache.get(("pos", n, tuple(self.feat_size), dev), [pos], build)

    def _vit_tc(self, x_in: torch.Tensor) -> tuple[K.NC8, list[K.NC8]]:
        """ViT.forward on NC8 tokens: the token buffer [N][hidden/8][S][8] IS the NC8 image of the feat_size volume, so the
        reference's proj_feat costs nothing.  Returns (vit.norm(tokens), hidden states 3, 6, 9)."""
        n, dev = x_in.shape[0], x_in.device
        hid, mlp = self.hidden_size, self.mlp_dim
        pe = self.vit.patch_embedding
        conv = pe.patch_embeddings
        # patch embedding: a Linear over the flattened 16^3 patch (K = in_channels * 4096), position embedding as the residual
        cols = K.patchify(x_in, self.patch_size)
        xp = K.pack_nc8(cols.reshape(n, cols.shape[1], *self.feat_size))
        cur, _ = K.gemm_tc(xp, self._wlin(conv.weight, "pe"), cols.shape[1], hid, bias=conv.bias, res=self._pos_nc8(n, dev))
        hidden = []
        for i, blk in enumerate(self.vit.blocks):
            key = f"b{i}"
            at = blk.attn
            h = K.layernorm_nc8(cur, blk.norm1.weight, blk.norm1.bias, blk.norm1.eps)
            wq, bq = self._wqkv_scaled(at.qkv.weight, at.qkv.bias, hid, at.scale, key)
            qkv, _ = K.gemm_tc(h, wq, hid, 3 * hid, bias=bq)
            att = K.mhsa_tc(qkv, hid, at.num_heads)
            x1, _ = K.gemm_tc(att, self._wlin(at.out_proj.weight, key + ".o"), hid, hid, bias=at.out_proj.bias, res=cur)
            y = K.layernorm_nc8(x1, blk.norm2.weight, blk.norm2.bias, blk.norm2.eps)
            m, _ = K.gemm_tc(y, self._wlin(blk.mlp.linear1.weight, key + ".fc1"), hid, mlp, bias=blk.mlp.linear1.bias, act=L.ACT_GELU)
            cur, _ = K.gemm_tc(m, self._wlin(blk.mlp.linear2.weight, key + ".fc2"), mlp, hid, bias=blk.mlp.linear2.bias, res=x1)
            if i in (3, 6, 9):
                hidden.append(cur)
        nrm = self.vit.norm
        return K.layernorm_nc8(cur, nrm.weight, nrm.bias, nrm.eps), hidden

    def _up(self, x: K.NC8, cin: int, conv: nn.ConvTranspose3d, key: str, out: K.NC8 | None = None, out_coff: int = 0) -> K.NC8:
        """ConvTranspose3d k2 s2 as a GEMM whose epilogue scatters to the 2x upsampled voxels (optionally a concat slice)."""
        y, _ = K.gemm_tc(x, self._wup(conv, key), cin, 8 * conv.out_channels, out=out, out_coff=out_coff, mode=2)
        return y

    def _pr_up(self, x: K.NC8, blk: UnetrPrUpBlock, key: str, out: K.NC8, out_coff: int) -> None:
        """UnetrPrUpBlock.forward: the last layer writes the skip slice of the decoder's concat buffer."""
        cout = blk.transp_conv_init.conv.out_channels
        if not blk.blocks:
            self._up(x, self.hidden_size, blk.transp_conv_init.conv, key + ".t0", out=out, out_coff=out_coff)
            return
        t = self._up(x, self.hidden_size, blk.transp_conv_init.conv, key + ".t0")
        for j, sub in enumerate(blk.blocks):
            t = self._up(t, cout, sub[0].conv, f"{key}.t{j + 1}")
            last = j == len(blk.blocks) - 1
            t = self._res_block(t, cout, 0, sub[1], f"{key}.r{j + 1}", out=out if last else None, out_coff=out_coff if last else 0)

    def _forward_tc(self, x_in: torch.Tensor) -> torch.Tensor:
        """UNETR.forward (unetr.py:199-213) on fp16 NC8 buffers and tensor cores; the output is fp16."""
        with torch.no_grad():
            x_in = x_in.contiguous()
            n, dev, fs = x_in.shape[0], x_in.device, self.feature_size
            sp0 = tuple(int(s) for s in x_in.shape[2:])
            sp = [tuple(s // 2**k for s in sp0) for k in range(4)]   # full, 1/2, 1/4, 1/8 resolution

            # decoder input buffers: [upsampled | skip] channel slices, written in place by their producers
            cat1 = K.NC8(n, 2 * fs, sp[0], dev)     # decoder2: [up(dec1) | enc1]
            cat2 = K.NC8(n, 4 * fs, sp[1], dev)     # decoder3: [up(dec2) | enc2]
            cat3 = K.NC8(n, 8 * fs, sp[2], dev)     # decoder4: [up(dec3) | enc3]
            cat4 = K.NC8(n, 16 * fs, sp[3], dev)    # decoder5: [up(tokens) | enc4]

            tokens, (h3, h6, h9) = self._vit_tc(x_in)

            # encoder1: the residual block on the raw input (one channel: direct stem kernels; several: channel-padded NC8)
            if self.in_channels == 1:
                self._res_block(None, 1, 0, self.encoder1.layer, "enc1", out=cat1, out_coff=fs, x_in_raw=x_in)
            else:
                cp = (self.in_channels + 15) // 16 * 16
                xz = torch.zeros((n, cp, *sp0), device=dev, dtype=torch.float16)
                K.copy_channels(x_in, xz, 0)
                xp = K.pack_nc8(xz)
                self._res_block(xp, cp, 0, self.encoder1.layer, "enc1", out=cat1, out_coff=fs, cin_pad=cp)
            self._pr_up(h3, self.encoder2, "enc2", cat2, 2 * fs)
            self._pr_up(h6, self.encoder3, "enc3", cat3, 4 * fs)
            self._pr_up(h9, self.encoder4, "enc4", cat4, 8 * fs)

            # decoders: ConvTranspose k2 s2 scatter into the concat buffer, then the residual block
            def up(dec_in: K.NC8, cin: int, block: UnetrUpBlock, cat: K.NC8, key: str, defer_tail: bool = False):
                self._up(dec_in, cin, block.transp_conv.conv, key, out=cat, out_coff=0)
                return self._res_block(cat, cat.C, 0, block.conv_block, key + ".rb", defer_tail=defer_tail)

            dec3 = up(tokens, self.hidden_size, self.decoder5, cat4, "dec5")
            dec2 = up(dec3, 8 * fs, self.decoder4, cat3, "dec4")
            dec1 = up(dec2, 4 * fs, self.decoder3, cat2, "dec3")
            # decoder2's norm2 + residual + lrelu is applied by the output head on its operand load
            y2, st2, res, res_coff, res_st = up(dec1, 2 * fs, self.decoder2, cat1, "dec2", defer_tail=True)
            oc = self.out.conv.conv
            return K.head_conv_norm_nc8(y2, st2, res, res_coff, res_st, 0.01, 1e-5, oc.weight, oc.bias, out_dtype=x_in.dtype)
