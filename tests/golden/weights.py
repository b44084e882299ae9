"""Deterministic, name-keyed weights shared by make_golden.py (reference side) and the tests (monai_b200 side).

Filling a state_dict through this function makes the weights independent of module construction order and RNG
consumption, so the reference model and the H100 model are guaranteed to hold identical parameters.
"""
from __future__ import annotations

import zlib

import torch


def fill_state_dict(sd: dict, seed: int = 0) -> dict:
    out = {}
    for k in sorted(sd.keys()):
        v = sd[k]
        if not torch.is_floating_point(v):
            out[k] = v.clone()
            continue
        g = torch.Generator().manual_seed((zlib.crc32(k.encode()) + 7919 * seed) % (2**31))
        shape = tuple(v.shape)
        if "relative_position_bias_table" in k:
            t = torch.randn(shape, generator=g) * 0.5
        elif k.endswith("running_var"):
            t = torch.rand(shape, generator=g) + 0.5
        elif k.endswith("running_mean"):
            t = torch.randn(shape, generator=g) * 0.1
        elif v.dim() >= 2:
            fan_in = max(1, int(v[0].numel()))
            if "transp_conv" in k or "deconv" in k or (".2.conv.weight" in k and v.dim() == 5):
                fan_in = max(1, int(v.shape[0]) * int(v[0, 0].numel()) // 4)
            t = torch.randn(shape, generator=g) / (fan_in**0.5)
        elif ".A.weight" in k:
            t = torch.rand(shape, generator=g) * 0.3 + 0.1
        elif k.endswith("weight"):
            t = torch.rand(shape, generator=g) + 0.5
        else:
            t = torch.randn(shape, generator=g) * 0.1
        out[k] = t.to(v.dtype)
    return out
