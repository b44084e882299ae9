"""Lazy resampling: consecutive spatial transforms are composed into ONE matrix and resampled ONCE (SURVEY.md §8 f1).

Restates monai/transforms/lazy/functional.py:195-296 (`apply_pending`), monai/transforms/lazy/utils.py:68-229 (matrix
composition, `resample`) and the pending-operation bookkeeping of monai/transforms/inverse.py:168-290.  A lazy transform does not
touch the voxels: it pushes {lazy_affine: output voxel index -> input voxel index, lazy_shape, ...} onto
`MetaTensor.pending_operations`; `apply_pending` multiplies the matrices in application order and hands the product to ONE
`SpatialResample` launch (dst_affine = affine @ cumulative) -- on the GPU one `b200_resample_affine` kernel whose
coordinates come from the composed matrix, so `Spacingd -> RandAffined` costs one pass over the volume instead of two.

As in the reference, the interpolation / padding mode of the single resample comes from the pending items' top-level
`lazy_interpolation_mode` / `lazy_padding_mode` entries (which the spatial transforms do not set: the defaults "bilinear" /
"border" apply) or from `overrides`.  Matrices that only permute / flip / shift by whole voxels still run through the
resampler here (the reference short-cuts them into array operations): same values, one launch.
"""
from __future__ import annotations

from collections.abc import Mapping
from typing import Any

import numpy as np
import torch

from ..data.meta_tensor import MetaTensor, is_meta

LAZY_SHAPE, LAZY_AFFINE = "lazy_shape", "lazy_affine"
LAZY_PADDING_MODE, LAZY_INTERP_MODE, LAZY_DTYPE, LAZY_ALIGN_CORNERS, LAZY_RESAMPLE_MODE = (
    "lazy_padding_mode", "lazy_interpolation_mode", "lazy_dtype", "lazy_align_corners", "lazy_resample_mode")
_OVERRIDE_KEYS = {"mode", "padding_mode", "dtype", "align_corners", "resample_mode", "device"}

__all__ = ["apply_pending", "apply_pending_transforms", "push_pending", "LAZY_SHAPE", "LAZY_AFFINE"]


def _affine3(m) -> np.ndarray:
    m = np.asarray(m.detach().cpu().numpy() if isinstance(m, torch.Tensor) else m, dtype=np.float64)
    if m.shape[0] == 3:   # 2-D matrix: lift to 3-D (to_affine_nd(3, .))
        full = np.eye(4)
        full[:2, :2], full[:2, -1] = m[:2, :2], m[:2, -1]
        return full
    return m


def _kwargs_from_pending(p) -> dict:
    if not isinstance(p, dict):
        return {}
    ret = {LAZY_INTERP_MODE: p.get(LAZY_INTERP_MODE, None), LAZY_PADDING_MODE: p.get(LAZY_PADDING_MODE, None)}
    if LAZY_SHAPE in p:
        ret[LAZY_SHAPE] = p[LAZY_SHAPE]
    if LAZY_DTYPE in p:
        ret[LAZY_DTYPE] = p[LAZY_DTYPE]
    return ret


def push_pending(img, info: dict, affine, shape) -> MetaTensor:
    """Record one lazy operation on `img` (wrapped into a MetaTensor if needed) without touching the voxels."""
    out = img if is_meta(img) else MetaTensor(img)
    if is_meta(img):
        out = type(img)(img.as_subclass(torch.Tensor))
        out.copy_meta_from(img, copy_attr=True)
    info = dict(info)
    info["lazy"] = True
    info[LAZY_SHAPE] = tuple(int(s) for s in shape)
    info[LAZY_AFFINE] = torch.as_tensor(np.asarray(affine, dtype=np.float64))
    out.push_pending_operation(info)
    return out


def _resample(data, matrix: np.ndarray, kwargs: dict):
    """lazy/utils.py:151-229 `resample`: one SpatialResample with dst_affine = affine @ matrix (always through the kernel)."""
    from .spatial import SpatialResample

    ndim = len(matrix) - 1
    img = data if is_meta(data) else MetaTensor(data)
    init_affine = np.asarray(img.affine, dtype=np.float64)
    k = min(ndim, init_affine.shape[0] - 1)
    aff_nd = np.eye(ndim + 1)
    aff_nd[:k, :k], aff_nd[:k, -1] = init_affine[:k, :k], init_affine[:k, -1]
    spatial_size = kwargs.get(LAZY_SHAPE, None)
    out_size = img.peek_pending_shape() if spatial_size is None else spatial_size
    rs = SpatialResample(dtype=kwargs.get(LAZY_DTYPE, torch.float64), align_corners=bool(kwargs.get(LAZY_ALIGN_CORNERS, False)))
    rs._trace = False   # the pending items themselves are pushed to applied_operations by apply_pending
    return rs(img, dst_affine=aff_nd @ matrix, spatial_size=[int(s) for s in out_size], mode=kwargs.get(LAZY_INTERP_MODE) or "bilinear",
              padding_mode=kwargs.get(LAZY_PADDING_MODE) or "border")


def apply_pending(data, pending: list | None = None, overrides: dict | None = None):
    """Compose and execute the pending operations of `data` (functional.py:195-296).  Returns (data, pending)."""
    overrides = dict(overrides or {})
    for k in overrides:
        if k not in _OVERRIDE_KEYS:
            raise ValueError(f"unsupported override {k!r}; options: {sorted(_OVERRIDE_KEYS)}")
    if is_meta(data) and pending is None:
        pending = list(data.pending_operations)
        data.clear_pending_operations()
    pending = [] if pending is None else pending
    if not pending:
        return data, []
    cumulative = _affine3(pending[0][LAZY_AFFINE] if isinstance(pending[0], dict) else pending[0])
    cur = _kwargs_from_pending(pending[0])
    over: dict[str, Any] = {}
    if "mode" in overrides:
        over[LAZY_INTERP_MODE] = overrides["mode"]
    if "padding_mode" in overrides:
        over[LAZY_PADDING_MODE] = overrides["padding_mode"]
    if "align_corners" in overrides:
        over[LAZY_ALIGN_CORNERS] = overrides["align_corners"]
    over[LAZY_DTYPE] = overrides.get("dtype", torch.float64)
    for p in pending[1:]:
        cumulative = cumulative @ _affine3(p[LAZY_AFFINE] if isinstance(p, dict) else p)   # is_compatible_apply_kwargs() is always True
        cur.update(_kwargs_from_pending(p))
    cur.update(over)
    out = _resample(data, cumulative, cur)
    if is_meta(out):
        for p in pending:
            out.push_applied_operation(p)
    return out, pending


def apply_pending_transforms(data, keys=None, overrides: dict | None = None):
    """Execute the pending operations of every MetaTensor in `data` (a tensor, or a mapping restricted to `keys`);
    `overrides` maps keys to override dictionaries for mappings (lazy/functional.py:84-140)."""
    if isinstance(data, Mapping):
        d = dict(data)
        for k in (d.keys() if keys is None else keys):
            if k in d and is_meta(d[k]) and d[k].pending_operations:
                ov = (overrides or {}).get(k, None) if overrides is not None else None
                d[k], _ = apply_pending(d[k], overrides=ov)
        return d
    if is_meta(data) and data.pending_operations:
        return apply_pending(data, overrides=overrides)[0]
    return data
