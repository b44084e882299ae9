#!/usr/bin/env python
"""A network with a tensor-core forward as the predictor of a sliding-window inference, on deployed configurations:

  * unetr:               the reference's defaults (ViT-B/16, feature_size 16, 14 classes); a 256^3 fp16 volume, roi 96^3;
  * dynunet iso:         the nnU-Net default plan (6 levels, filters 32 ... 320, affine instance norm, 14 classes); a 384^3 fp16
                         volume, roi 128^3;
  * dynunet aniso_d:     an nnU-Net anisotropic plan for thick-slice CT / MR (kernels [1,3,3] at the two high-resolution levels,
                         strides [1,2,2], [1,2,2], [2,2,2], [2,2,2], [1,2,2]; filters 32 ... 320, 14 classes); a 64 x 512 x 512 fp16
                         volume, roi 32 x 256 x 256 (27 windows);
  * dynunet aniso_w:     a MONAI-style plan with kernel 1 along W (kernels [3,3,1] at two levels, strides [2,2,1], [2,2,1], [2,2,2],
                         [2,2,2]), residual blocks, filters 32 ... 320, 14 classes; a 384 x 384 x 64 fp16 volume, roi 192 x 192 x 32;
  * segresnet brats:     init_filters 16, 4 input modalities, 3 outputs, GroupNorm(8), blocks (1,2,2,4) / (1,1,1); a
                         4 x 240 x 240 x 160 fp16 volume, roi 128^3;
  * segresnet wholebody: init_filters 32, 1 input channel, 105 outputs, GroupNorm(8); a 256^3 fp16 volume, roi 96^3;
  * unet res_batch:      the spleen CT UNet of MONAI's tutorial and bundle (channels 16 ... 256, strides 2, two residual units,
                         eval-mode BatchNorm, PReLU, 1 -> 2 channels); a 256^3 fp16 volume, roi 160^3;
  * unet res_instance:   the same net with InstanceNorm (MONAI's default norm); a 256^3 fp16 volume, roi 96^3;
  * basic_unet:          the reference's defaults (features 32, 32, 64, 128, 256, 32, affine instance norm, LeakyReLU 0.1, 1 -> 2
                         channels); a 256^3 fp16 volume, roi 96^3;
  * segresnet_ds default:  the reference's defaults (init 32, eval-mode BatchNorm, ReLU, deconv, blocks (1,2,2,4), 1 -> 2 channels);
                         a 256^3 fp16 volume, roi 96^3;
  * segresnet_ds auto3dseg: the net of MONAI's Auto3DSeg `segresnet` algorithm on thick-slice CT (init 32, blocks (1,2,2,4,4),
                         instance norm, resolution (0.8, 0.8, 2.5): [3,3,1] kernels and (2,2,1) strides at level 0, 1 -> 14
                         channels); a 512 x 512 x 128 fp16 volume, roi 192 x 192 x 64.

    python scripts/sliding_window_tc.py --net unetr|dynunet|segresnet|unet|basic_unet|segresnet_ds [--workload brats|wholebody|both
                                        (SegResNet) | iso|aniso_d|aniso_w|all (DynUNet) | res_batch|res_instance|res (UNet) |
                                        default|auto3dseg|ds (SegResNetDS)] [--sw-batch 4] [--steps 3] [--warmup 1]

Overlap 0.5, gaussian blending.  Every batch shape (the full batches and the remainder batch) is warmed up first; each timed step
is bracketed by CUDA events with a 256 MiB L2 flush before it (outside the timed interval), and the spread of the timed steps is
reported.  A separate profiled step lists device time per kernel.  Finally one forward of sw_batch windows and one of a single
window are timed on each path: `net(x)` (tensor cores) and `net._forward_generic(x)` (the generic CUDA-core kernels), giving the
speed-up per window without running a whole volume on CUDA cores; for UNet and BasicUNet the tensor-core forward is also timed per
window in its other launch mode (eager or CUDA-graph replay), and with BatchNorm the activation-only norm_act_nc8 passes of one forward are timed on their own.
Prints one JSON line per workload, with the card name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import torch  # noqa: E402

OVERLAP = 0.5


def unetr_flops(net, roi) -> dict:
    """Multiply-add FLOPs (x2) of one window, from the layer shapes of UNETR.forward (ViT and decoder separately)."""
    hid, mlp, heads = net.hidden_size, net.mlp_dim, net.num_heads
    fs, cin = net.feature_size, net.in_channels
    v = [math.prod(s // 2**k for s in roi) for k in range(5)]   # voxels at 1, 1/2, 1/4, 1/8, 1/16 resolution
    S = v[4]
    vit = 2.0 * S * cin * 16**3 * hid
    vit += net.num_layers * (2.0 * S * hid * 3 * hid + 4.0 * heads * S * S * (hid // heads) + 2.0 * S * hid * hid + 4.0 * S * hid * mlp)

    def res(ci, co, n):      # UnetResBlock: two 3x3x3 convolutions and a 1x1x1 one when the channels change
        return 2.0 * n * 27 * (ci * co + co * co) + (2.0 * n * ci * co if ci != co else 0.0)

    def up(ci, co, n_in):    # ConvTranspose3d k2 s2
        return 2.0 * n_in * 8 * ci * co

    dec = res(cin, fs, v[0])
    dec += up(hid, 2 * fs, v[4]) + up(2 * fs, 2 * fs, v[3]) + res(2 * fs, 2 * fs, v[2]) + up(2 * fs, 2 * fs, v[2]) + res(2 * fs, 2 * fs, v[1])
    dec += up(hid, 4 * fs, v[4]) + up(4 * fs, 4 * fs, v[3]) + res(4 * fs, 4 * fs, v[2])
    dec += up(hid, 8 * fs, v[4])
    dec += up(hid, 8 * fs, v[4]) + res(16 * fs, 8 * fs, v[3])
    dec += up(8 * fs, 4 * fs, v[3]) + res(8 * fs, 4 * fs, v[2])
    dec += up(4 * fs, 2 * fs, v[2]) + res(4 * fs, 2 * fs, v[1])
    dec += up(2 * fs, fs, v[1]) + res(2 * fs, fs, v[0])
    dec += 2.0 * v[0] * fs * net.out.conv.conv.out_channels
    return {"vit": vit, "decoder": dec, "total": vit + dec}


def _per_axis(v) -> tuple[int, int, int]:
    return tuple(int(i) for i in v) if isinstance(v, (list, tuple)) else (int(v),) * 3


def dynunet_flops(net, roi) -> dict:
    """Multiply-add FLOPs (x2) of one window, from the layer shapes of DynUNet.forward: per-level kernel volumes and per-axis
    strides (the isotropic plan: 3x3x3 kernels, stride 2)."""
    f, cin, nl = net.filters, net.in_channels, len(net.filters)
    v, cum = [], (1, 1, 1)
    for s in net.strides:                               # voxels at level k: the roi over the cumulative strides
        cum = tuple(c * i for c, i in zip(cum, _per_axis(s)))
        v.append(math.prod(r // c for r, c in zip(roi, cum)))
    kv = [math.prod(_per_axis(k)) for k in net.kernel_size]   # kernel volume of level k
    res = net.conv_block.__name__ == "UnetResBlock"

    def block(ci, co, n, taps, skip_conv):   # two convolutions (+ the 1x1x1 one of a residual block when shape or channels change)
        return 2.0 * n * taps * (ci * co + co * co) + (2.0 * n * ci * co if res and skip_conv else 0.0)

    enc = block(cin, f[0], v[0], kv[0], cin != f[0])
    for k in range(1, nl):                              # down blocks and the bottleneck (output voxels v[k])
        enc += block(f[k - 1], f[k], v[k], kv[k], True)
    dec = 2.0 * v[0] * f[0] * net.out_channels
    for k in range(nl - 2, -1, -1):                     # up blocks: ConvTranspose3d (kernel = stride: one tap per output voxel), then
        # a basic block with the kernel of level k + 1 on the concat
        dec += 2.0 * v[k] * f[k + 1] * f[k] + 2.0 * v[k] * kv[k + 1] * (2 * f[k] * f[k] + f[k] * f[k])
    return {"encoder": enc, "decoder": dec, "total": enc + dec}


def segresnet_flops(net, roi) -> dict:
    """Multiply-add FLOPs (x2) of one window, from the layer shapes of SegResNet.forward."""
    f0, nd = net.init_filters, len(net.blocks_down)
    v = [math.prod(s // 2**k for s in roi) for k in range(nd)]     # voxels at level k
    c = [f0 * 2**k for k in range(nd)]                             # channels at level k
    conv3 = lambda n, ci, co: 2.0 * n * 27 * ci * co               # noqa: E731
    enc = conv3(v[0], net.in_channels, f0)                         # convInit
    for k, nb in enumerate(net.blocks_down):
        if k > 0:
            enc += conv3(v[k], c[k - 1], c[k])                     # stride-2 pre_conv (output voxels)
        enc += nb * 2 * conv3(v[k], c[k], c[k])                    # ResBlocks: two 3x3x3 convolutions each
    dec = 0.0
    for i, nb in enumerate(net.blocks_up):
        k = nd - 2 - i                                             # the level the decoder step lands on
        dec += 2.0 * v[k + 1] * c[k + 1] * c[k]                    # 1x1x1 at the low resolution
        if net.upsample_mode == "deconv":
            dec += 2.0 * v[k + 1] * c[k] * c[k] * 8                # ConvTranspose3d k2 s2
        dec += nb * 2 * conv3(v[k], c[k], c[k])
    if net.use_conv_final:
        dec += 2.0 * v[0] * f0 * net.conv_final[2].conv.out_channels
    return {"encoder": enc, "decoder": dec, "total": enc + dec}


def unet_flops(net, roi) -> dict:
    """Multiply-add FLOPs (x2) of one window, from the layer shapes of UNet with residual units: every convolution of the down
    ResidualUnits and the bottom one (encoder), and the transposed convolutions and up ResidualUnits (decoder)."""
    import torch.nn as nn

    from monai_b200.networks.blocks.convolutions import ResidualUnit

    def conv(m, v):                      # (FLOPs, output voxels) of a Conv3d / ConvTranspose3d on v input voxels
        k, s = math.prod(m.kernel_size), math.prod(m.stride)
        if isinstance(m, nn.ConvTranspose3d):
            return 2.0 * v * m.in_channels * m.out_channels * k, v * s
        return 2.0 * (v // s) * m.in_channels * m.out_channels * k, v // s

    def unit(mod, v):                    # a ResidualUnit or a Convolution block
        if not isinstance(mod, ResidualUnit):
            return conv(mod.conv, v)
        f, vo = 0.0, v
        for u in mod.conv:
            fu, vo = conv(u.conv, vo)
            f += fu
        if not isinstance(mod.residual, nn.Identity):
            f += conv(mod.residual, v)[0]
        return f, vo

    def level(block, v):                 # (encoder, decoder) FLOPs of Sequential(down, SkipConnection(sub), up)
        down, sub, up = block[0], block[1].submodule, block[2]
        enc, vd = unit(down, v)
        if isinstance(sub, ResidualUnit):
            e2, d2 = unit(sub, vd)[0], 0.0
        else:
            e2, d2 = level(sub, vd)
        dec, vu = 0.0, vd
        for m in (up if isinstance(up, nn.Sequential) else [up]):
            f, vu = unit(m, vu)
            dec += f
        return enc + e2, d2 + dec

    enc, dec = level(net.model, math.prod(roi))
    return {"encoder": enc, "decoder": dec, "total": enc + dec}


def basic_unet_flops(net, roi) -> dict:
    """Multiply-add FLOPs (x2) of one window, from the layer shapes of BasicUNet.forward: the two 3x3x3 convolutions of every TwoConv
    (encoder: conv_0 and down_1 ... down_4; decoder: upcat_4 ... upcat_1), the transposed convolutions k2 s2 and the 1x1x1 head."""
    v = [math.prod(s // 2**k for s in roi) for k in range(5)]   # voxels at level k

    def two(tc, n):
        return sum(2.0 * n * 27 * c.conv.in_channels * c.conv.out_channels for c in (tc.conv_0, tc.conv_1))

    enc = two(net.conv_0, v[0]) + sum(two(d.convs, v[k]) for k, d in enumerate((net.down_1, net.down_2, net.down_3, net.down_4), 1))
    dec = 2.0 * v[0] * net.final_conv.in_channels * net.final_conv.out_channels
    for k, uc in zip((3, 2, 1, 0), (net.upcat_4, net.upcat_3, net.upcat_2, net.upcat_1)):   # uc lands on level k
        dc = uc.upsample.deconv
        dec += 2.0 * v[k + 1] * 8 * dc.in_channels * dc.out_channels + two(uc.convs, v[k])
    return {"encoder": enc, "decoder": dec, "total": enc + dec}


def segresnet_ds_flops(net, roi) -> dict:
    """Multiply-add FLOPs (x2) of one window, from the module shapes of SegResNetDS: conv_init, both convolutions of every
    SegResBlock and the strided convolutions (encoder); the transposed convolutions or 1x1 preconvs, the up blocks and the head
    (decoder).  A transposed convolution costs every tap per input voxel."""
    scales = net.anisotropic_scales or [(2, 2, 2)] * len(net.blocks_down)
    sp = [tuple(roi)]
    for sc in scales[: len(net.blocks_down) - 1]:
        sp.append(tuple(s // int(f) for s, f in zip(sp[-1], sc)))
    v = [math.prod(s) for s in sp]                                   # voxels at level k

    def conv(n, m):
        return 2.0 * n * m.in_channels * m.out_channels * math.prod(m.kernel_size)

    def blocks(seq, n):
        return sum(conv(n, b.conv1) + conv(n, b.conv2) for b in seq)

    enc = conv(v[0], net.encoder.conv_init)
    for k, lvl in enumerate(net.encoder.layers):
        enc += blocks(lvl["blocks"], v[k])
        if k + 1 < len(v):
            enc += conv(v[k + 1], lvl["downsample"])               # output voxels
    dec, n_up = 0.0, len(net.blocks_down) - 1
    for i, lvl in enumerate(net.up_layers[:n_up]):
        k, up = n_up - 1 - i, lvl["upsample"]                      # the level the decoder step lands on
        dec += conv(v[k + 1], up.deconv if hasattr(up, "deconv") else up.preconv)
        dec += blocks(lvl["blocks"], v[k])
    dec += conv(v[0], net.up_layers[-1]["head"])
    return {"encoder": enc, "decoder": dec, "total": enc + dec}


def unet_act_passes(net, roi, batch) -> list:
    """(channels, spatial size) of each activation-only norm_act_nc8 pass of a BatchNorm residual UNet forward: the output of every
    unit of a down or bottom ResidualUnit but its last, activated before the next unit's convolution reads it."""
    from monai_b200.networks.blocks.convolutions import ResidualUnit

    out, block, sp = [], net.model, tuple(roi)
    while True:
        down, sub = block[0], block[1].submodule
        sp = tuple(v // down.conv.unit0.conv.stride[0] for v in sp)
        out += [(down.out_channels, sp)] * (len(down.conv) - 1)
        if isinstance(sub, ResidualUnit):
            return out + [(sub.out_channels, sp)] * (len(sub.conv) - 1)
        block = sub


def _nets():
    from monai_b200.networks.nets import UNETR, BasicUNet, DynUNet, SegResNet, SegResNetDS, UNet

    return {
        "unetr": {
            "unetr_sliding_window": dict(
                make=lambda: UNETR(in_channels=1, out_channels=14, img_size=(96, 96, 96)), seed=80, cin=1, volume=(256, 256, 256), roi=(96, 96, 96),
                flops=unetr_flops, desc="UNETR(in=1, out=14, img=96, hidden=768, heads=12, mlp=3072, fs=16)"),
        },
        "dynunet": {
            "dynunet_sliding_window": dict(
                make=lambda: DynUNet(3, 1, 14, kernel_size=[3] * 6, strides=[1, 2, 2, 2, 2, 2], upsample_kernel_size=[2] * 5), seed=30, cin=1,
                volume=(384, 384, 384), roi=(128, 128, 128), flops=dynunet_flops,
                desc="DynUNet(in=1, out=14, k=3x6, strides=[1,2,2,2,2,2], filters=32..320, affine IN)"),
            "dynunet_sliding_window_aniso_d": dict(
                make=lambda: DynUNet(3, 1, 14, **ANISO_D), seed=30, cin=1, volume=(64, 512, 512), roi=(32, 256, 256), flops=dynunet_flops,
                desc="DynUNet(in=1, out=14, k=[1,3,3]x2 + 3x4, strides=[1,1,1],[1,2,2],[1,2,2],[2,2,2],[2,2,2],[1,2,2], filters=32..320, affine IN)"),
            "dynunet_sliding_window_aniso_w": dict(
                make=lambda: DynUNet(3, 1, 14, **ANISO_W), seed=30, cin=1, volume=(384, 384, 64), roi=(192, 192, 32), flops=dynunet_flops,
                desc="DynUNet(in=1, out=14, k=[3,3,1]x2 + 3x3, strides=[1,1,1],[2,2,1],[2,2,1],[2,2,2],[2,2,2], res blocks, filters=32..320, affine IN)"),
        },
        "segresnet": {
            "segresnet_sliding_window_brats": dict(
                make=lambda: SegResNet(spatial_dims=3, init_filters=16, in_channels=4, out_channels=3, blocks_down=(1, 2, 2, 4), blocks_up=(1, 1, 1)),
                seed=30, cin=4, volume=(240, 240, 160), roi=(128, 128, 128), flops=segresnet_flops,
                desc="SegResNet(init=16, in=4, out=3, GroupNorm(8), blocks (1, 2, 2, 4)/(1, 1, 1), nontrainable)"),
            "segresnet_sliding_window_wholebody": dict(
                make=lambda: SegResNet(spatial_dims=3, init_filters=32, in_channels=1, out_channels=105, norm=("GROUP", {"num_groups": 8})),
                seed=30, cin=1, volume=(256, 256, 256), roi=(96, 96, 96), flops=segresnet_flops,
                desc="SegResNet(init=32, in=1, out=105, GroupNorm(8), blocks (1, 2, 2, 4)/(1, 1, 1), nontrainable)"),
        },
        "unet": {
            "unet_sliding_window_res_batch": dict(
                make=lambda: UNet(3, 1, 2, (16, 32, 64, 128, 256), (2, 2, 2, 2), num_res_units=2, norm="batch"), seed=20, cin=1,
                volume=(256, 256, 256), roi=(160, 160, 160), flops=unet_flops, eager_vs_replay=True, act_passes=unet_act_passes,
                desc="UNet(in=1, out=2, channels 16..256, strides 2, num_res_units=2, BatchNorm (eval), PReLU)"),
            "unet_sliding_window_res_instance": dict(
                make=lambda: UNet(3, 1, 2, (16, 32, 64, 128, 256), (2, 2, 2, 2), num_res_units=2), seed=20, cin=1,
                volume=(256, 256, 256), roi=(96, 96, 96), flops=unet_flops, eager_vs_replay=True,
                desc="UNet(in=1, out=2, channels 16..256, strides 2, num_res_units=2, InstanceNorm, PReLU)"),
        },
        "basic_unet": {
            "basic_unet_sliding_window": dict(
                make=lambda: BasicUNet(), seed=70, cin=1, volume=(256, 256, 256), roi=(96, 96, 96), flops=basic_unet_flops, eager_vs_replay=True,
                desc="BasicUNet(in=1, out=2, features (32, 32, 64, 128, 256, 32), affine IN, LeakyReLU 0.1)"),
        },
        "segresnet_ds": {
            "segresnet_ds_sliding_window_default": dict(
                make=lambda: SegResNetDS(), seed=110, cin=1, volume=(256, 256, 256), roi=(96, 96, 96), flops=segresnet_ds_flops,
                desc="SegResNetDS(init=32, in=1, out=2, BatchNorm (eval), ReLU, blocks (1, 2, 2, 4), deconv)"),
            "segresnet_ds_sliding_window_auto3dseg": dict(
                make=lambda: SegResNetDS(init_filters=32, in_channels=1, out_channels=14, blocks_down=(1, 2, 2, 4, 4), norm="instance_nvfuser",
                                         dsdepth=4, resolution=(0.8, 0.8, 2.5)),
                seed=111, cin=1, volume=(512, 512, 128), roi=(192, 192, 64), flops=segresnet_ds_flops,
                desc="SegResNetDS(init=32, in=1, out=14, instance norm, blocks (1, 2, 2, 4, 4), dsdepth 4, resolution (0.8, 0.8, 2.5), deconv)"),
        },
    }


# the anisotropic DynUNet plans of the aniso_d / aniso_w workloads (the shapes of tests/golden/dynunet_aniso_cases.py A and B)
ANISO_D = dict(kernel_size=[[1, 3, 3], [1, 3, 3], [3, 3, 3], [3, 3, 3], [3, 3, 3], [3, 3, 3]],
               strides=[[1, 1, 1], [1, 2, 2], [1, 2, 2], [2, 2, 2], [2, 2, 2], [1, 2, 2]],
               upsample_kernel_size=[[1, 2, 2], [1, 2, 2], [2, 2, 2], [2, 2, 2], [1, 2, 2]])
ANISO_W = dict(kernel_size=[[3, 3, 1], [3, 3, 1], [3, 3, 3], [3, 3, 3], [3, 3, 3]], strides=[[1, 1, 1], [2, 2, 1], [2, 2, 1], [2, 2, 2], [2, 2, 2]],
               upsample_kernel_size=[[2, 2, 1], [2, 2, 1], [2, 2, 2], [2, 2, 2]], filters=[32, 64, 128, 256, 320], res_block=True)
DYNUNET_WORKLOADS = {"iso": "dynunet_sliding_window", "aniso_d": "dynunet_sliding_window_aniso_d", "aniso_w": "dynunet_sliding_window_aniso_w"}


def _card() -> dict:
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_max_mhz": None}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        pl, mx = r.stdout.strip().splitlines()[0].split(", ")
        out["power_limit_w"], out["sm_max_mhz"] = float(pl), float(mx)
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        pass
    return out


def _windows(volume, roi) -> int:
    return math.prod(len(range(0, s - r + 1, int(r * (1 - OVERLAP)))) + ((s - r) % int(r * (1 - OVERLAP)) != 0) for s, r in zip(volume, roi))


def _timed(fn, x, reps: int) -> float:
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn(x)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def run(metric: str, wl: dict, args, card: dict) -> dict:
    from weights import fill_state_dict

    from monai_b200 import _kernels as K
    from monai_b200.inferers import sliding_window_inference

    volume, roi, cin = wl["volume"], wl["roi"], wl["cin"]
    dev = torch.device("cuda:0")
    net = wl["make"]()
    net.load_state_dict(fill_state_dict(net.state_dict(), wl["seed"]))
    net = net.half().eval().to(dev)
    assert net._tc_eligible() if hasattr(net, "_tc_eligible") else net._tc_ok
    vol = torch.randn((1, cin, *volume), generator=torch.Generator().manual_seed(0)).half().to(dev)
    windows = _windows(volume, roi)

    def step():
        return sliding_window_inference(vol, roi, args.sw_batch, net, OVERLAP, "gaussian")

    with torch.no_grad():
        for _ in range(max(1, args.warmup)):   # every batch shape, the remainder batch included
            step()
        torch.cuda.synchronize()
        flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
        times = []
        for _ in range(args.steps):
            flush.fill_(1)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        del flush

        K.profile_start()   # a separate, eager pass: the per-launch events slow the host down
        step()
        prof = K.profile_stop()
        prof_ms = sum(d["ms"] for d in prof.values())
        top = sorted(prof.items(), key=lambda kv: -kv[1]["ms"])[: args.top]

        per_window = {}
        for b in sorted({args.sw_batch, 1}):
            xb = torch.randn((b, cin, *roi), generator=torch.Generator().manual_seed(b)).half().to(dev)
            net(xb)
            tc_ms = _timed(net, xb, 5)
            net._forward_generic(xb)   # loads the generic kernels
            gen_ms = _timed(net._forward_generic, xb, 1)
            per_window[f"batch{b}"] = {"tensor_core": round(tc_ms / b, 3), "generic": round(gen_ms / b, 3), "speedup": round(gen_ms / tc_ms, 1)}
            if wl.get("eager_vs_replay"):   # the tensor-core forward once more with the other launch mode (CUDA-graph replay or eager)
                graph = net._graph_enabled
                net._graph_enabled = not graph
                net(xb)
                per_window[f"batch{b}"]["tensor_core_eager" if graph else "tensor_core_graph_replay"] = round(_timed(net, xb, 5) / b, 3)
                net._graph_enabled = graph
                net._graphs.clear()
        if wl.get("act_passes"):
            # the activation-only norm_act_nc8 passes that eval-mode BatchNorm adds (its units have no statistics to apply on the
            # next convolution's operand load), each timed over 20 launches at the step's batch
            passes = wl["act_passes"](net, roi, args.sw_batch)
            x8 = {sh: K.NC8(args.sw_batch, sh[0], sh[1], dev) for sh in set(passes)}
            for t in x8.values():
                t.buf.normal_()
            act_ms = sum(_timed(lambda t: K.norm_act_nc8(t, t.C, None, act=K.L.ACT_LEAKY, slope=0.25), x8[sh], 20) for sh in passes)
            per_window["bn_act_passes"] = {"n_per_forward": len(passes), "ms_per_forward": round(act_ms, 3),
                                           "ms_per_step": round(act_ms * -(-windows // args.sw_batch), 2)}

    fl = wl["flops"](net, roi)
    ms = sorted(times)[len(times) // 2]
    return {
        "metric": metric,
        "card": card,
        "config": {"volume": [cin, *volume], "roi": list(roi), "overlap": OVERLAP, "mode": "gaussian", "sw_batch": args.sw_batch,
                   "windows": windows, "dtype": "float16", "net": wl["desc"], "l2": "256 MiB flush write between timed steps", "steps": args.steps},
        "ms_per_step": round(ms, 2), "ms_per_step_min": round(min(times), 2), "ms_per_step_max": round(max(times), 2),
        "ms_per_step_all": [round(t, 2) for t in times],
        "voxels_per_s": math.prod(volume) / (ms / 1e3),
        "gflop_per_window": {k: round(v / 1e9, 2) for k, v in fl.items()},
        "model_tflops": fl["total"] * windows / (ms / 1e3) / 1e12,
        "profile_ms_total": round(prof_ms, 2),
        "top_kernels": [{"name": n, "ms": round(d["ms"], 3), "share": round(d["ms"] / prof_ms, 4), "n": d["n"],
                         "tflops": round(d["flops"] / (d["ms"] / 1e3) / 1e12, 1) if d["flops"] and d["ms"] else None,
                         "gbps": round(d["bytes"] / (d["ms"] / 1e3) / 1e9, 1) if d["bytes"] and d["ms"] else None} for n, d in top],
        "profile_gflop_per_window": round(sum(d["flops"] for d in prof.values()) / windows / 1e9, 2),
        "per_window_ms": per_window,
    }


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--net", required=True, choices=["unetr", "dynunet", "segresnet", "unet", "basic_unet", "segresnet_ds"])
    ap.add_argument("--workload", default=None, choices=["both", "brats", "wholebody", "all", "iso", "aniso_d", "aniso_w", "res_batch",
                                                          "res_instance", "res", "default", "auto3dseg", "ds"],
                    help="SegResNet: brats|wholebody|both (default both); DynUNet: iso|aniso_d|aniso_w|all (default iso); "
                         "UNet: res_batch|res_instance|res (default res: both); SegResNetDS: default|auto3dseg|ds (default ds: both)")
    ap.add_argument("--sw-batch", type=int, default=4)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--top", type=int, default=12)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sliding_window_tc.py measures on a CUDA device; none is available")
    workloads = _nets()[args.net]
    if args.net == "segresnet" and args.workload not in (None, "both"):
        workloads = {f"segresnet_sliding_window_{args.workload}": workloads[f"segresnet_sliding_window_{args.workload}"]}
    if args.net == "dynunet" and args.workload != "all":
        name = DYNUNET_WORKLOADS[args.workload or "iso"]
        workloads = {name: workloads[name]}
    if args.net == "unet" and args.workload not in (None, "res"):
        workloads = {f"unet_sliding_window_{args.workload}": workloads[f"unet_sliding_window_{args.workload}"]}
    if args.net == "segresnet_ds" and args.workload not in (None, "ds"):
        workloads = {f"segresnet_ds_sliding_window_{args.workload}": workloads[f"segresnet_ds_sliding_window_{args.workload}"]}
    card = _card()
    for metric, wl in workloads.items():
        print(json.dumps(run(metric, wl, args, card)), flush=True)


if __name__ == "__main__":
    main()
