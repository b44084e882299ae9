"""Pieces shared by the tensor-core forwards (SwinUNETR, UNETR, DynUNet): the packed-weight cache and the residual / basic
blocks of their CNN parts on fp16 NC8 buffers.

`TcBlocks` is a mixin for an nn.Module that sets `self._cache = _Cache()`.  The block helpers accept any module with the
`conv1.conv` / `conv2.conv` / optional `conv3.conv`, `norm1/2/3` and `lrelu` structure of UnetResBlock / UnetBasicBlock
(dynunet_block.py:25-177; kernel 3, stride 1 or 2, InstanceNorm with or without affine parameters, LeakyReLU).  eps, gamma /
beta and the slope are read from the block, so the non-affine blocks of the transformer segmenters (eps 1e-5, slope 0.01) call
exactly the entry points and arguments they did before the affine variants existed."""
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

    def _wg(self, conv: nn.Conv3d, key: str, k: int, stride: int, pad: int):
        return self._cache.get(("wg", key, k, stride, pad, conv.weight.device), [conv.weight],
                               lambda: K.conv_gather_tc_pack_weight(conv.weight, k, stride, pad, False))

    # ------------------------------------------------------------------------------------------------- sub-graphs
    @staticmethod
    def _norm(norm: nn.Module):
        """(eps, gamma, beta) of an InstanceNorm module; gamma / beta are None when it is not affine."""
        if norm.affine:
            return float(norm.eps), norm.weight, norm.bias
        return float(norm.eps), None, None

    @staticmethod
    def _slope(blk: nn.Module) -> float:
        return float(blk.lrelu.negative_slope)

    def _conv1(self, x: K.NC8, cin: int, in_coff: int, blk: nn.Module, key: str, stride: int, cin_pad: int | None):
        """conv1 of a block (raw output + statistics): 3x3x3 stride 1 on conv3x3x3_tc, stride 2 on conv_gather_tc."""
        cout = blk.conv1.conv.out_channels
        if stride == 2:
            return K.conv_gather_tc(x, self._wg(blk.conv1.conv, key + ".c1", 3, 2, 1), cin, cout, 3, 2, 1, in_coff=in_coff, want_stats=True)
        return K.conv3x3x3_tc(x, self._w3(blk.conv1.conv, key + ".c1", cin_pad), cin, cout, in_coff=in_coff, want_stats=True)

    def _conv2(self, y1: K.NC8, st1: torch.Tensor, blk: nn.Module, key: str):
        """conv2 with norm1 + lrelu of conv1's raw output applied on its operand load (no pass over the tensor in between)."""
        cout = blk.conv2.conv.out_channels
        eps1, g1, b1 = self._norm(blk.norm1)
        return K.conv3x3x3_tc(y1, self._w3(blk.conv2.conv, key + ".c2"), cout, cout, want_stats=True, in_norm=(st1, eps1, L.ACT_LEAKY, self._slope(blk)),
                              in_affine=(g1, b1))

    def _basic_block(self, x: K.NC8, cin: int, in_coff: int, blk: nn.Module, key: str, out: K.NC8 | None = None, out_coff: int = 0,
                     x_in_raw: torch.Tensor | None = None, defer_tail: bool = False, cin_pad: int | None = None, stride: int = 1):
        """UnetBasicBlock.forward (dynunet_block.py:165-177) on NC8 buffers: conv1, conv2 with norm1 + lrelu on its operand load,
        then norm2 + lrelu into `out` (may be a slice of a concat buffer).  With `defer_tail` the last step is NOT applied: (y2,
        stats2) are returned for the output head."""
        cout = blk.conv1.conv.out_channels
        if x_in_raw is not None:  # single input channel: direct stem kernel on the raw NCDHW window
            y1, st1 = K.conv_cin1_nc8(x_in_raw, blk.conv1.conv.weight, None, 3, 1, 1, want_stats=True)
        else:
            y1, st1 = self._conv1(x, cin, in_coff, blk, key, stride, cin_pad)
        y2, st2 = self._conv2(y1, st1, blk, key)
        if defer_tail:
            return y2, st2
        if out is None:
            out = K.NC8(y2.N, cout, y2.sp, y2.buf.device)
        eps2, g2, b2 = self._norm(blk.norm2)
        K.norm_act_nc8(y2, cout, st2, act=L.ACT_LEAKY, slope=self._slope(blk), out=out, out_coff=out_coff, eps=eps2, gamma=g2, beta=b2)
        return out

    def _res_block(self, x: K.NC8, cin: int, in_coff: int, blk: nn.Module, key: str, out: K.NC8 | None = None, out_coff: int = 0,
                   x_in_raw: torch.Tensor | None = None, defer_tail: bool = False, cin_pad: int | None = None, stride: int = 1):
        """UnetResBlock.forward (dynunet_block.py:97-111) on NC8 buffers; `out` may be a slice of a concat buffer.  eps, the
        (optional) affine parameters of norm1/2/3 and the LeakyReLU slope come from the block's modules.  stride 2: conv1 (k3 p1)
        and conv3 (k1 p0) run on conv_gather_tc.
        With `defer_tail` the final norm2 + residual + lrelu is NOT applied: the pieces (y2, stats2, res, res_coff,
        res_stats) are returned so that the consumer (the output head) applies them on its operand load; that needs a
        non-affine norm3."""
        cout = blk.conv1.conv.out_channels
        slope = self._slope(blk)
        eps2, g2, b2 = self._norm(blk.norm2)
        has3 = hasattr(blk, "conv3")
        eps3, g3, b3 = self._norm(blk.norm3) if has3 else (eps2, None, None)
        folded = None
        if x_in_raw is not None:  # single input channel: direct stem kernels read the raw NCDHW window
            y1, st1 = K.conv_cin1_nc8(x_in_raw, blk.conv1.conv.weight, None, 3, 1, 1, want_stats=True)
        elif stride == 1 and has3 and cout <= 128 and cin_pad is None and blk.conv3.conv.bias is None:
            # conv3 (1x1x1 residual branch) reads the same input as conv1: one launch produces both tensors and both statistics
            y1, st1, y3f, st3f = K.conv3x3x3_tc(x, self._w3(blk.conv1.conv, key + ".c1", cin_pad), cin, cout, in_coff=in_coff, want_stats=True,
                                                res_w=self._wlin(blk.conv3.conv.weight, key + ".c3", cin_pad))
            folded = (y3f, st3f)
        else:
            y1, st1 = self._conv1(x, cin, in_coff, blk, key, stride, cin_pad)
        y2, st2 = self._conv2(y1, st1, blk, key)
        if has3:
            if (x_in_raw is not None and x_in_raw.dtype == torch.float16 and blk.conv3.conv.bias is None and not defer_tail
                    and g2 is None and b2 is None and g3 is None and b3 is None and eps3 == eps2):
                # one input channel: norm3(conv3(u)) is an affine function of u per channel -- no conv3 launch, no y3 tensor
                if out is None:
                    out = K.NC8(y2.N, cout, y2.sp, y2.buf.device)
                K.norm_act_cin1res_nc8(y2, cout, st2, x_in_raw, K.instnorm_stats(x_in_raw), blk.conv3.conv.weight, act=L.ACT_LEAKY, slope=slope,
                                       out=out, out_coff=out_coff, eps=eps2)
                return out
            if folded is not None:
                y3, st3 = folded
            elif x_in_raw is not None:
                y3, st3 = K.conv_cin1_nc8(x_in_raw, blk.conv3.conv.weight, None, 1, 1, 0, want_stats=True)
            elif stride == 2:
                y3, st3 = K.conv_gather_tc(x, self._wg(blk.conv3.conv, key + ".c3", 1, 2, 0), cin, cout, 1, 2, 0, in_coff=in_coff, want_stats=True)
            else:
                y3, st3 = K.gemm_tc(x, self._wlin(blk.conv3.conv.weight, key + ".c3", cin_pad), cin, cout, in_coff=in_coff, want_stats=True)
            if defer_tail:
                return y2, st2, y3, 0, st3
        elif defer_tail:
            return y2, st2, x, in_coff, None
        if out is None:
            out = K.NC8(y2.N, cout, y2.sp, y2.buf.device)
        if has3:
            K.norm_act_nc8(y2, cout, st2, res=y3, res_stats=st3, act=L.ACT_LEAKY, slope=slope, out=out, out_coff=out_coff, eps=eps2,
                           gamma=g2, beta=b2, res_gamma=g3, res_beta=b3)
        else:
            K.norm_act_nc8(y2, cout, st2, res=x, res_coff=in_coff, act=L.ACT_LEAKY, slope=slope, out=out, out_coff=out_coff, eps=eps2,
                           gamma=g2, beta=b2)
        return out
