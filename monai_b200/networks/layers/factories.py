"""Name -> torch.nn parameter-container lookup for activations and normalisations used on the hot path.

The reference resolves these through `LayerFactory` objects (monai/networks/layers/factories.py, utils.py:24-76).
Here the torch modules only *hold parameters / hyper-parameters* (so `state_dict` keys and initialisation match the
reference); the arithmetic is done by the CUDA kernels in monai_b200.networks.blocks.
"""
from __future__ import annotations

import torch.nn as nn

__all__ = ["split_args", "get_act_layer", "get_norm_layer", "get_dropout_layer"]


def split_args(args):
    """"name" or ("name", {kwargs}) -> (name, kwargs)."""
    if isinstance(args, str):
        return args, {}
    name, kw = args
    if not isinstance(kw, dict):
        raise TypeError("Layer specifiers must be single strings or pairs of the form (name/object-types, argument dict).")
    return name, kw


_ACTS = {
    "prelu": nn.PReLU, "leakyrelu": nn.LeakyReLU, "relu": nn.ReLU, "gelu": nn.GELU,
}


def get_act_layer(name):
    if name == "" or name is None:
        return nn.Identity()
    act_name, kw = split_args(name)
    key = str(act_name).lower()
    if key not in _ACTS:
        raise NotImplementedError(f"monai_b200 supports activations {sorted(_ACTS)}, got {act_name!r}.")
    return _ACTS[key](**kw)


def get_norm_layer(name, spatial_dims: int = 1, channels: int | None = 1):
    if name == "" or name is None:
        return nn.Identity()
    norm_name, kw = split_args(name)
    key = str(norm_name).lower()
    # "instance_nvfuser" is apex's InstanceNorm3dNVFuser; the reference's factory falls back to nn.InstanceNorm{1,2,3}d without apex
    # (monai/networks/layers/factories.py:258-281), the same arithmetic
    if key in ("instance", "instance_nvfuser"):
        return (nn.InstanceNorm1d, nn.InstanceNorm2d, nn.InstanceNorm3d)[spatial_dims - 1](channels, **kw)
    if key == "batch":
        return (nn.BatchNorm1d, nn.BatchNorm2d, nn.BatchNorm3d)[spatial_dims - 1](channels, **kw)
    if key == "group":   # Norm.GROUP (monai/networks/layers/factories.py): nn.GroupNorm(num_groups, num_channels, ...)
        return nn.GroupNorm(num_channels=channels, **kw)
    raise NotImplementedError(f"monai_b200 supports 'instance', 'instance_nvfuser', 'batch' and 'group' normalisation, got {norm_name!r}.")


def get_dropout_layer(name, dropout_dim: int = 1):
    if isinstance(name, (int, float)):
        return (nn.Dropout, nn.Dropout2d, nn.Dropout3d)[dropout_dim - 1](p=float(name))
    drop_name, kw = split_args(name)
    key = str(drop_name).lower()
    if key != "dropout":
        raise NotImplementedError(f"unsupported dropout type {drop_name!r}")
    return (nn.Dropout, nn.Dropout2d, nn.Dropout3d)[dropout_dim - 1](**kw)
