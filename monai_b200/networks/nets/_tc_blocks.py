"""`TcNet`: the mixin every network with a tensor-core forward (UNet, BasicUNet, SwinUNETR, UNETR, DynUNet, SegResNet, SegResNetDS)
inherits.

It owns what those networks share:
  * `forward`: the choice between `_forward_tc` (fp16 channel-blocked "NC8" buffers on Hopper tensor cores) and `_forward_generic`
    (the generic kernels), through the hooks `_check_input` (both paths), `_use_tc` and `_check_tc_input` (tensor-core path only);
  * CUDA-graph replay of `_forward_tc`.  One forward is tens to hundreds of short kernel launches; issuing them from Python
    through ctypes costs more than the kernels themselves once they are fast, so the launch sequence for a given input shape is
    captured once into a CUDA graph and replayed.  Graphs are keyed by (shape, dtype, device) and invalidated when any parameter
    or buffer changes (`load_state_dict`, `.half()`).  MONAI_B200_GRAPH=0 disables the mechanism;
  * the packed-weight cache, the channel-padded input stem, and the residual / basic blocks, transposed convolutions and output
    head of the CNN parts.  The block helpers accept any module with the `conv1.conv` / `conv2.conv` / optional `conv3.conv`,
    `norm1/2/3` and `lrelu` structure of UnetResBlock / UnetBasicBlock (dynunet_block.py:25-177; InstanceNorm with or without affine
    parameters, LeakyReLU) and read kernel, stride and padding from the block's own convolutions: a stride-1 3x3x3 kernel runs on
    conv3x3x3_tc, a stride-1 kernel of 3x3 in one plane and 1 along the third axis on conv3x3_tc, a kernel with stride 2 on any axis
    on conv_gather_tc (per axis), and a stride-1 1x1x1 kernel on gemm_tc.  eps, gamma / beta and the slope are read from the block; the
    non-affine blocks of the transformer segmenters (eps 1e-5, slope 0.01) pass no gamma / beta, so their kernels run the
    non-affine instantiations;
  * for the `Convolution` blocks of UNet and BasicUNet: the reader of a block's ADN (eps, gamma / beta, activation and slope) and
    the norm_act_nc8 pass that applies it; for SegResNet and BasicUNet: the output head after a norm + activation, fused into
    head_conv_norm_nc8 up to 16 outputs and on gemm_tc with zero-padded columns above.

A network calls `self._tc_setup()` in its constructor and supplies `_forward_tc` and `_forward_generic`."""
from __future__ import annotations

import os
from collections.abc import Sequence

import torch
import torch.nn as nn

from ... import _kernels as K
from ... import _lib as L

__all__ = ["TcNet"]


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


class TcNet:
    _cache: _Cache
    _tc_ok: bool

    def _tc_setup(self) -> None:
        self._cache = _Cache()
        self._graph_enabled = os.environ.get("MONAI_B200_GRAPH", "1") != "0"
        self._graphs: dict = {}

    # ------------------------------------------------------------------------------------------------- dispatch
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        self._check_input(x)
        if not self._use_tc(x):
            return self._forward_generic(x)
        self._check_tc_input(x)
        return self._forward_graphed(x) if self._graph_ok() else self._forward_tc(x)

    def _check_input(self, x: torch.Tensor) -> None:
        """Raises on input neither path accepts."""

    def _use_tc(self, x: torch.Tensor) -> bool:
        return self._tc_ok and x.is_cuda and x.dtype == torch.float16

    def _check_tc_input(self, x: torch.Tensor) -> None:
        """Raises, before any launch, on input the tensor-core path does not accept."""

    def _check_levels(self, x: torch.Tensor, levels: int) -> None:
        """[N, in_channels, D, H, W] with every spatial size divisible by 2^(levels - 1)."""
        name, div = type(self).__name__, 2 ** (levels - 1)
        if x.dim() != 5 or x.shape[1] != self.in_channels:
            raise ValueError(f"{name} expects an [N, {self.in_channels}, D, H, W] input, got {tuple(x.shape)}")
        if any(int(s) % div for s in x.shape[2:]):
            raise ValueError(f"{name} with {levels} levels needs spatial sizes divisible by {div}, got {tuple(x.shape[2:])}")

    def _graph_ok(self) -> bool:
        return self._graph_enabled and not K._Prof.on and not torch.cuda.is_current_stream_capturing()

    def _forward_graphed(self, x_in: torch.Tensor) -> torch.Tensor:
        # buffers too: load_state_dict may change only a BatchNorm's running statistics, which a folded weight depends on
        sig = tuple((p.data_ptr(), p._version) for p in (*self.parameters(), *self.buffers()))
        key = (tuple(x_in.shape), x_in.dtype, x_in.device)
        ent = self._graphs.get(key)
        if ent is None or ent["sig"] != sig:
            static_in = x_in.detach().clone().contiguous()
            self._forward_tc(static_in)  # eager warm-up: packs weights, sets kernel attributes, fills the plan caches
            torch.cuda.synchronize(x_in.device)
            graph = torch.cuda.CUDAGraph()
            n0 = L.launch_count()
            # thread_local: other threads (e.g. the NCCL watchdog) may issue CUDA calls while this thread captures
            with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                static_out = self._forward_tc(static_in)
            n_kernels = L.launch_count() - n0
            if len(self._graphs) >= 4:  # bound the private memory pools kept alive
                self._graphs.pop(next(iter(self._graphs)))
            ent = {"sig": sig, "graph": graph, "inp": static_in, "out": static_out, "n_kernels": n_kernels}
            self._graphs[key] = ent
        ent["inp"].copy_(x_in)
        ent["graph"].replay()
        L.add_replayed_launches(ent["n_kernels"])
        return ent["out"].clone()

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

    def _whead(self, conv: nn.Conv3d, npad: int):
        """The 1x1x1 output convolution with its output channels zero-padded to `npad`: (packed weight, float32 bias)."""
        def build():
            w = torch.zeros((npad, conv.in_channels), device=conv.weight.device, dtype=torch.float32)
            w[: conv.out_channels] = conv.weight.detach().float().reshape(conv.out_channels, -1)
            b = torch.zeros(npad, device=conv.weight.device, dtype=torch.float32)
            if conv.bias is not None:
                b[: conv.out_channels] = conv.bias.detach().float()
            return K.gemm_tc_pack_weight(w), b

        params = [conv.weight] + ([conv.bias] if conv.bias is not None else [])
        return self._cache.get(("head", npad, conv.weight.device), params, build)

    def _w33(self, conv: nn.Conv3d, key: str, axis: int, cin_pad: int | None = None):
        return self._cache.get(("w33", key, axis, cin_pad, conv.weight.device), [conv.weight],
                               lambda: K.conv3x3_tc_pack_weight(self._pad_cin(conv.weight, cin_pad), axis))

    def _wg(self, conv: nn.Module, key: str, k, stride, pad, transposed: bool = False):
        return self._cache.get(("wg", key, k, stride, pad, transposed, conv.weight.device), [conv.weight],
                               lambda: K.conv_gather_tc_pack_weight(conv.weight, k, stride, pad, transposed))

    # ------------------------------------------------------------------------------------------------- sub-graphs
    @staticmethod
    def _pack_input(x_in: torch.Tensor) -> tuple[K.NC8, int]:
        """The input zero-padded to a multiple of 16 channels (the multi-channel stems run on 16-channel tiles) as an fp16 NC8
        image; returns (image, padded channel count)."""
        cp = (x_in.shape[1] + 15) // 16 * 16
        xz = torch.zeros((x_in.shape[0], cp, *x_in.shape[2:]), device=x_in.device, dtype=torch.float16)
        K.copy_channels(x_in.to(torch.float16), xz, 0)
        return K.pack_nc8(xz), cp

    @staticmethod
    def _norm(norm: nn.Module):
        """(eps, gamma, beta) of an InstanceNorm module; gamma / beta are None when it is not affine."""
        if norm.affine:
            return float(norm.eps), norm.weight, norm.bias
        return float(norm.eps), None, None

    @staticmethod
    def _bn(blk: nn.Module):
        n = getattr(getattr(blk, "adn", None), "N", None)
        return n if isinstance(n, nn.BatchNorm3d) else None

    def _act_of(self, conv: nn.Module):
        """(act code, slope) of the activation of a `Convolution` block's ADN; a PReLU's single weight is read once per value."""
        act = getattr(conv.adn, "A", None)
        if isinstance(act, nn.PReLU):
            return L.ACT_LEAKY, self._cache.get(("slope", id(act)), [act.weight], lambda: float(act.weight.detach().float().item()))
        if isinstance(act, nn.LeakyReLU):
            return L.ACT_LEAKY, float(act.negative_slope)
        if isinstance(act, nn.ReLU):
            return L.ACT_RELU, 0.0
        return L.ACT_NONE, 0.0

    def _adn(self, blk: nn.Module):
        """(instance norm?, eps, gamma, beta, act, slope) of an "NDA" `Convolution` block; a BatchNorm block has no norm left to
        apply (it is folded into the convolution)."""
        act, slope = self._act_of(blk)
        if self._bn(blk) is not None:
            return False, 1e-5, None, None, act, slope
        eps, g, b = self._norm(blk.adn.N)
        return True, eps, g, b, act, slope

    def _finish(self, y: K.NC8, C_: int, st, blk: nn.Module, out=None, out_coff: int = 0, res=None, res_coff: int = 0) -> K.NC8:
        """act(norm(y)) of the "NDA" block `blk` (+ res after the activation) into `out`."""
        inorm, eps, g, b, act, slope = self._adn(blk)
        return K.norm_act_nc8(y, C_, st if inorm else None, res=res, res_coff=res_coff, act=act, slope=slope, out=out, out_coff=out_coff,
                              eps=eps, gamma=g, beta=b, res_after_act=res is not None)

    @staticmethod
    def _slope(blk: nn.Module) -> float:
        return float(blk.lrelu.negative_slope)

    @staticmethod
    def _strided(conv: nn.Module) -> bool:
        return any(int(s) != 1 for s in conv.stride)

    @staticmethod
    def _one_plane_axis(conv: nn.Module) -> int:
        """-1 for a 3x3x3 kernel, else the axis of size 1 of a 3x3 kernel in one plane (the kernels of conv3x3_tc)."""
        k = tuple(int(i) for i in conv.kernel_size)
        return -1 if k == (3, 3, 3) else k.index(1)

    def _conv_s1(self, x: K.NC8, cin: int, conv: nn.Conv3d, key: str, cin_pad: int | None = None, **kw):
        """A stride-1 convolution with a 3x3x3 kernel (conv3x3x3_tc) or a 3x3 kernel in one plane (conv3x3_tc)."""
        axis = self._one_plane_axis(conv)
        if axis < 0:
            return K.conv3x3x3_tc(x, self._w3(conv, key, cin_pad), cin, conv.out_channels, **kw)
        return K.conv3x3_tc(x, self._w33(conv, key, axis, cin_pad), cin, conv.out_channels, axis, **kw)

    def _conv_strided(self, x: K.NC8, cin: int, in_coff: int, conv: nn.Conv3d, key: str):
        """A convolution with stride 2 on some axis, on conv_gather_tc with the module's per-axis kernel, stride and padding."""
        k, s, p = (tuple(int(i) for i in v) for v in (conv.kernel_size, conv.stride, conv.padding))
        return K.conv_gather_tc(x, self._wg(conv, key, k, s, p), cin, conv.out_channels, k, s, p, in_coff=in_coff, want_stats=True)

    def _conv1(self, x: K.NC8, cin: int, in_coff: int, blk: nn.Module, key: str, cin_pad: int | None):
        """conv1 of a block (raw output + statistics)."""
        if self._strided(blk.conv1.conv):
            return self._conv_strided(x, cin, in_coff, blk.conv1.conv, key + ".c1")
        return self._conv_s1(x, cin, blk.conv1.conv, key + ".c1", cin_pad, in_coff=in_coff, want_stats=True)

    def _conv2(self, y1: K.NC8, st1: torch.Tensor, blk: nn.Module, key: str):
        """conv2 with norm1 + lrelu of conv1's raw output applied on its operand load (no pass over the tensor in between)."""
        eps1, g1, b1 = self._norm(blk.norm1)
        return self._conv_s1(y1, blk.conv2.conv.out_channels, blk.conv2.conv, key + ".c2", want_stats=True,
                             in_norm=(st1, eps1, L.ACT_LEAKY, self._slope(blk)), in_affine=(g1, b1))

    def _basic_block(self, x: K.NC8, cin: int, in_coff: int, blk: nn.Module, key: str, out: K.NC8 | None = None, out_coff: int = 0,
                     x_in_raw: torch.Tensor | None = None, defer_tail: bool = False, cin_pad: int | None = None):
        """UnetBasicBlock.forward (dynunet_block.py:165-177) on NC8 buffers: conv1, conv2 with norm1 + lrelu on its operand load,
        then norm2 + lrelu into `out` (may be a slice of a concat buffer).  With `defer_tail` the last step is NOT applied: the
        pieces are returned for `_tail_head` in the form `_res_block` returns them, without a residual."""
        cout = blk.conv1.conv.out_channels
        if x_in_raw is not None:  # single input channel: direct stem kernel on the raw NCDHW window
            y1, st1 = K.conv_cin1_nc8(x_in_raw, blk.conv1.conv.weight, None, 3, 1, 1, want_stats=True)
        else:
            y1, st1 = self._conv1(x, cin, in_coff, blk, key, cin_pad)
        y2, st2 = self._conv2(y1, st1, blk, key)
        if defer_tail:
            return y2, st2, None, 0, None
        if out is None:
            out = K.NC8(y2.N, cout, y2.sp, y2.buf.device)
        eps2, g2, b2 = self._norm(blk.norm2)
        K.norm_act_nc8(y2, cout, st2, act=L.ACT_LEAKY, slope=self._slope(blk), out=out, out_coff=out_coff, eps=eps2, gamma=g2, beta=b2)
        return out

    def _res_block(self, x: K.NC8, cin: int, in_coff: int, blk: nn.Module, key: str, out: K.NC8 | None = None, out_coff: int = 0,
                   x_in_raw: torch.Tensor | None = None, defer_tail: bool = False, cin_pad: int | None = None):
        """UnetResBlock.forward (dynunet_block.py:97-111) on NC8 buffers; `out` may be a slice of a concat buffer.  eps, the
        (optional) affine parameters of norm1/2/3 and the LeakyReLU slope come from the block's modules.  Strided: conv1 and conv3
        (k1 p0) run on conv_gather_tc.
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
        elif (has3 and not self._strided(blk.conv1.conv) and self._one_plane_axis(blk.conv1.conv) < 0 and cout <= 128 and cin_pad is None
              and blk.conv3.conv.bias is None):
            # conv3 (1x1x1 residual branch) reads the same input as conv1: one launch produces both tensors and both statistics
            y1, st1, y3f, st3f = K.conv3x3x3_tc(x, self._w3(blk.conv1.conv, key + ".c1", cin_pad), cin, cout, in_coff=in_coff, want_stats=True,
                                                res_w=self._wlin(blk.conv3.conv.weight, key + ".c3", cin_pad))
            folded = (y3f, st3f)
        else:
            y1, st1 = self._conv1(x, cin, in_coff, blk, key, cin_pad)
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
            elif self._strided(blk.conv3.conv):
                y3, st3 = self._conv_strided(x, cin, in_coff, blk.conv3.conv, key + ".c3")
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

    def _up(self, x: K.NC8, cin: int, conv: nn.ConvTranspose3d, key: str, out: K.NC8 | None = None, out_coff: int = 0) -> K.NC8:
        """ConvTranspose3d k2 s2 as a GEMM whose epilogue scatters to the 2x upsampled voxels (optionally a concat slice).  An
        anisotropic one with kernel = stride per axis (e.g. (1, 2, 2)) runs on conv_gather_tc: one tap per parity class."""
        s = tuple(int(i) for i in conv.stride)
        if s != (2, 2, 2):
            y, _ = K.conv_gather_tc(x, self._wg(conv, key, s, s, 0, transposed=True), cin, conv.out_channels, s, s, 0, transposed=True,
                                    bias=conv.bias, out=out, out_coff=out_coff)
            return y
        y, _ = K.gemm_tc(x, self._wup(conv, key), cin, 8 * conv.out_channels, bias=conv.bias, out=out, out_coff=out_coff, mode=2)
        return y

    def _up_block(self, x: K.NC8, cin: int, block: nn.Module, cat: K.NC8, key: str, defer_tail: bool = False):
        """UnetrUpBlock.forward: the transposed convolution writes channels [0, C) of `cat`, whose upper half already holds the
        skip, then the residual block runs on `cat`."""
        self._up(x, cin, block.transp_conv.conv, key, out=cat)
        return self._res_block(cat, cat.C, 0, block.conv_block, key + ".rb", defer_tail=defer_tail)

    def _norm_act_head(self, x: K.NC8, stats: torch.Tensor, eps: float, gamma, beta, act: int, slope: float, conv: nn.Conv3d,
                       dtype: torch.dtype) -> torch.Tensor:
        """conv(act(norm(x))) for the whole NC8 image x and a 1x1x1 `conv`, as NCDHW logits in `dtype`.  Up to 16 outputs: one
        head_conv_norm_nc8 launch with the norm and the activation (ReLU as slope 0) on its operand load.  More: norm_act_nc8,
        then gemm_tc with the output channels zero-padded to a multiple of 16."""
        if conv.out_channels <= 16:
            return K.head_conv_norm_nc8(x, stats, None, 0, None, slope, eps, conv.weight, conv.bias, out_dtype=dtype, gamma=gamma, beta=beta)
        npad = (conv.out_channels + 15) // 16 * 16
        xn = K.norm_act_nc8(x, x.C, stats, act=act, slope=slope, eps=eps, gamma=gamma, beta=beta)
        wp, bp = self._whead(conv, npad)
        y, _ = K.gemm_tc(xn, wp, x.C, npad, bias=bp)
        # the padding channels are dropped by a view (the graph replay returns a contiguous copy)
        return K.unpack_nc8(y, dtype=dtype).narrow(1, 0, conv.out_channels)

    def _tail_head(self, tail, block: nn.Module, out_conv: nn.Conv3d, dtype: torch.dtype) -> torch.Tensor:
        """The 1x1x1 output convolution with the deferred tail of the last block (`defer_tail=True`) -- its norm2, the residual
        branch if any, and LeakyReLU -- applied on the operand load."""
        y2, st2, res, res_coff, res_st = tail
        eps, g, b = self._norm(block.norm2)
        return K.head_conv_norm_nc8(y2, st2, res, res_coff, res_st, self._slope(block), eps, out_conv.weight, out_conv.bias, out_dtype=dtype,
                                    gamma=g, beta=b)
