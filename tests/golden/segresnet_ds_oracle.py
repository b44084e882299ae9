"""A torch-CPU restatement of SegResNetDS's eval-mode forward (monai/networks/nets/segresnet_ds.py) that the tests compare the
reference's fixtures and this package's forwards against.  It reads only a state_dict and the constructor arguments and uses the same
functional calls in the same order as the reference's modules, so in fp32 it reproduces the reference's outputs bit for bit."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F


def _scales(resolution, n_stages):
    """scales_for_resolution (segresnet_ds.py:44-55)."""
    res = np.array(resolution)
    nl = np.floor(np.log2(np.max(res) / res)).astype(np.int32)
    scales = [tuple(int(v) for v in np.where(2**i >= 2**nl, 1, 2)) for i in range(max(nl))]
    if n_stages > max(nl):
        return scales + [(2,) * len(resolution)] * (n_stages - max(nl))
    return scales[:n_stages]


def _norm(x, sd, p, norm, groups, eps):
    """norm1 / norm2 (segresnet_ds.py:99, 110; affine unless told otherwise, segresnet_ds.py:161-164)."""
    w, b = sd.get(p + ".weight"), sd.get(p + ".bias")
    if norm == "batch":   # eval mode: running statistics
        return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], w, b, False, 0.1, eps)
    if norm == "group":
        return F.group_norm(x, groups, w, b, eps)
    return F.instance_norm(x, None, None, w, b, True, 0.1, eps)


def _act(x, slope):
    return F.relu(x) if slope is None else F.leaky_relu(x, slope)


def _conv(x, w, b=None, stride=1, padding=0):
    return (F.conv1d, F.conv2d, F.conv3d)[x.dim() - 3](x, w, b, stride, padding)


def _block(x, sd, p, norm, groups, eps, slope):
    """SegResBlock.forward (segresnet_ds.py:121-125): x + conv2(act2(norm2(conv1(act1(norm1(x))))))."""
    pad1 = tuple(k // 2 for k in sd[p + ".conv1.weight"].shape[2:])
    y = _conv(_act(_norm(x, sd, p + ".norm1", norm, groups, eps), slope), sd[p + ".conv1.weight"], padding=pad1)
    y = _conv(_act(_norm(y, sd, p + ".norm2", norm, groups, eps), slope), sd[p + ".conv2.weight"], padding=pad1)
    y += x
    return y


def segresnet_ds_forward(sd: dict, x: torch.Tensor, blocks_down=(1, 2, 2, 4), norm: str = "batch", groups: int = 8, eps: float = 1e-5,
                         slope=None, upsample_mode: str = "deconv", resolution=None) -> torch.Tensor:
    """SegResNetDS._forward in eval mode (segresnet_ds.py:391-422): the encoder (segresnet_ds.py:217-229), then per up level
    upsample + skip, blocks; returns outputs[0], the head of the finest level.  `norm` is "batch", "instance" or "group"; `slope`
    None is ReLU, else LeakyReLU's negative slope."""
    nd = x.dim() - 2
    n = len(blocks_down)
    scales = _scales(resolution, n) if resolution else None
    kern = [[3 if s > 1 else 1 for s in sc] for sc in scales] if scales else [[3] * nd] * n
    stride = scales if scales else [(2,) * nd] * n
    x = _conv(x, sd["encoder.conv_init.weight"], padding=tuple(k // 2 for k in kern[0]))
    down = []
    for i, nb in enumerate(blocks_down):
        for j in range(nb):
            x = _block(x, sd, f"encoder.layers.{i}.blocks.{j}", norm, groups, eps, slope)
        down.append(x)
        if i < n - 1:
            x = _conv(x, sd[f"encoder.layers.{i}.downsample.weight"], stride=tuple(stride[i]), padding=tuple(k // 2 for k in kern[i]))
    down.reverse()
    x = down.pop(0)
    n_up = n - 1
    for i in range(n_up):
        lvl, p = n_up - i - 1, f"up_layers.{i}"
        s, k = tuple(stride[lvl]), kern[lvl]
        if upsample_mode == "deconv":   # UpSample with kernel_size (upsample.py:94-115)
            pad = tuple((kk - 1) // 2 for kk in k)
            op = tuple(ss - 1 - (kk - 1) % 2 for kk, ss in zip(k, s))
            x = (F.conv_transpose1d, F.conv_transpose2d, F.conv_transpose3d)[nd - 1](x, sd[p + ".upsample.deconv.weight"], None, s, pad, op)
        else:                           # preconv 1x1, then nn.Upsample(scale, linear, align_corners=False)
            x = _conv(x, sd[p + ".upsample.preconv.weight"])
            x = F.interpolate(x, scale_factor=tuple(float(v) for v in s), mode=("linear", "bilinear", "trilinear")[nd - 1], align_corners=False)
        x += down.pop(0)
        j = 0
        while f"{p}.blocks.{j}.conv1.weight" in sd:
            x = _block(x, sd, f"{p}.blocks.{j}", norm, groups, eps, slope)
            j += 1
    p = f"up_layers.{max(n_up - 1, 0)}.head"
    return _conv(x, sd[p + ".weight"], sd[p + ".bias"])
