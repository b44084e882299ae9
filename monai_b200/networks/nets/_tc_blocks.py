"""Pieces shared by the tensor-core forwards of the transformer segmenters (SwinUNETR, UNETR): the packed-weight cache and the
residual block of their CNN decoders on fp16 NC8 buffers.

`TcBlocks` is a mixin for an nn.Module that sets `self._cache = _Cache()`.  The residual-block helper accepts any module with
the `conv1.conv` / `conv2.conv` / optional `conv3.conv` structure of UnetResBlock (dynunet_block.py:25-111; kernel 3,
stride 1, non-affine InstanceNorm, LeakyReLU 0.01)."""
from __future__ import annotations

from collections.abc import Sequence

import torch
import torch.nn as nn

from ... import _kernels as K
from ... import _lib as L

__all__ = ["TcBlocks"]


class _Cache:
    """Packed weights and index tables keyed by (name, device); invalidated when a parameter is modified."""

    def __init__(self):
        self.store: dict = {}

    def get(self, key, params: Sequence[torch.Tensor], build):
        ver = tuple((p.data_ptr(), p._version, p.dtype) for p in params)
        hit = self.store.get(key)
        if hit is not None and hit[0] == ver:
            return hit[1]
        val = build()
        self.store[key] = (ver, val)
        return val


class TcBlocks:
    _cache: _Cache

    # ----------------------------------------------------------------------------------------------- weight prep
    @staticmethod
    def _pad_cin(w: torch.Tensor, cin_pad: int | None) -> torch.Tensor:
        """Zero-pad the input-channel axis (dim 1) of a conv / linear weight: the multi-channel stems run on 16-channel tiles."""
        if cin_pad is None or w.shape[1] == cin_pad:
            return w
        out = torch.zeros((w.shape[0], cin_pad, *w.shape[2:]), device=w.device, dtype=torch.float32)
        out[:, : w.shape[1]] = w.detach().float()
        return out

    def _w3(self, conv: nn.Conv3d, key: str, cin_pad: int | None = None):
        return self._cache.get(("w3", key, cin_pad, conv.weight.device), [conv.weight], lambda: K.conv3x3x3_tc_pack_weight(self._pad_cin(conv.weight, cin_pad)))

    def _wlin(self, w: torch.Tensor, key: str, cin_pad: int | None = None):
        def build():
            wp = self._pad_cin(w, cin_pad)
            return K.gemm_tc_pack_weight(wp.reshape(wp.shape[0], -1))

        return self._cache.get(("lin", key, cin_pad, w.device), [w], build)

    def _wup(self, conv: nn.ConvTranspose3d, key: str):
        # ConvTranspose3d weight [Cin, Cout, 2,2,2] -> GEMM W[(tap, cout), cin]
        def build():
            w = conv.weight.detach().float()
            return K.gemm_tc_pack_weight(w.permute(2, 3, 4, 1, 0).reshape(8 * w.shape[1], w.shape[0]).contiguous())

        return self._cache.get(("up", key, conv.weight.device), [conv.weight], build)

    def _wqkv_scaled(self, weight: torch.Tensor, bias: torch.Tensor | None, C: int, scale: float, key: str):
        """Packed qkv projection [3C, C] with scale * log2(e) folded into its q rows (the tensor-core attention kernels work in
        log2 units); returns (packed weight, float32 bias or None)."""
        def build():
            f = scale * K.LOG2E
            w = weight.detach().float().clone()
            w[:C] *= f
            b = None
            if bias is not None:
                b = bias.detach().float().clone()
                b[:C] *= f
            return K.gemm_tc_pack_weight(w), b

        params = [weight] + ([bias] if bias is not None else [])
        return self._cache.get(("qkvs", key, weight.device), params, build)

    # ------------------------------------------------------------------------------------------------- sub-graphs
    def _res_block(self, x: K.NC8, cin: int, in_coff: int, blk: nn.Module, key: str, out: K.NC8 | None = None, out_coff: int = 0,
                   x_in_raw: torch.Tensor | None = None, defer_tail: bool = False, cin_pad: int | None = None):
        """UnetResBlock.forward (dynunet_block.py:97-111) on NC8 buffers; `out` may be a slice of a concat buffer.
        With `defer_tail` the final norm2 + residual + lrelu is NOT applied: the pieces (y2, stats2, res, res_coff,
        res_stats) are returned so that the consumer (the output head) applies them on its operand load."""
        cout = blk.conv1.conv.out_channels
        folded = None
        if x_in_raw is not None:  # single input channel: direct stem kernels read the raw NCDHW window
            y1, st1 = K.conv_cin1_nc8(x_in_raw, blk.conv1.conv.weight, None, 3, 1, 1, want_stats=True)
        elif hasattr(blk, "conv3") and cout <= 128 and cin_pad is None and blk.conv3.conv.bias is None:
            # conv3 (1x1x1 residual branch) reads the same input as conv1: one launch produces both tensors and both statistics
            y1, st1, y3f, st3f = K.conv3x3x3_tc(x, self._w3(blk.conv1.conv, key + ".c1", cin_pad), cin, cout, in_coff=in_coff, want_stats=True,
                                                res_w=self._wlin(blk.conv3.conv.weight, key + ".c3", cin_pad))
            folded = (y3f, st3f)
        else:
            y1, st1 = K.conv3x3x3_tc(x, self._w3(blk.conv1.conv, key + ".c1", cin_pad), cin, cout, in_coff=in_coff, want_stats=True)
        # norm1 + lrelu on conv2's operand load: y1 stays raw, no pass over the tensor in between
        y2, st2 = K.conv3x3x3_tc(y1, self._w3(blk.conv2.conv, key + ".c2"), cout, cout, want_stats=True, in_norm=(st1, 1e-5, L.ACT_LEAKY, 0.01))
        if hasattr(blk, "conv3"):
            if x_in_raw is not None and x_in_raw.dtype == torch.float16 and blk.conv3.conv.bias is None and not defer_tail:
                # one input channel: norm3(conv3(u)) is an affine function of u per channel -- no conv3 launch, no y3 tensor
                if out is None:
                    out = K.NC8(y2.N, cout, y2.sp, y2.buf.device)
                K.norm_act_cin1res_nc8(y2, cout, st2, x_in_raw, K.instnorm_stats(x_in_raw), blk.conv3.conv.weight, act=L.ACT_LEAKY, slope=0.01,
                                       out=out, out_coff=out_coff)
                return out
            if folded is not None:
                y3, st3 = folded
            elif x_in_raw is not None:
                y3, st3 = K.conv_cin1_nc8(x_in_raw, blk.conv3.conv.weight, None, 1, 1, 0, want_stats=True)
            else:
                y3, st3 = K.gemm_tc(x, self._wlin(blk.conv3.conv.weight, key + ".c3", cin_pad), cin, cout, in_coff=in_coff, want_stats=True)
            if defer_tail:
                return y2, st2, y3, 0, st3
        elif defer_tail:
            return y2, st2, x, in_coff, None
        if out is None:
            out = K.NC8(y2.N, cout, y2.sp, y2.buf.device)
        if hasattr(blk, "conv3"):
            K.norm_act_nc8(y2, cout, st2, res=y3, res_stats=st3, act=L.ACT_LEAKY, slope=0.01, out=out, out_coff=out_coff)
        else:
            K.norm_act_nc8(y2, cout, st2, res=x, res_coff=in_coff, act=L.ACT_LEAKY, slope=0.01, out=out, out_coff=out_coff)
        return out
