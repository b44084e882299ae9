"""H100-native `sliding_window_inference` (drop-in for monai/inferers/utils.py:42-321).

Same signature, argument meaning and error behaviour as the reference.  What differs is *how* the stitched
volume is produced: windows are gathered by `b200_sw_gather`, and the importance-weighted overlap blend
(reference: count-map build :264-275, `seg *= w` / `out[idx] += p` :286-288 + :351-360, `out /= count` :297-298)
is one gather-form CUDA kernel (`b200_sw_blend`) that evaluates the Gaussian importance map analytically,
accumulates in fp32 in the reference's window order and never stores a count map.

There is no CPU or eager-PyTorch fallback: CUDA inputs are required and the C-ABI library must be loadable.
1-D / 2-D inputs are handled by the same 3-D kernels through singleton axes; >3 spatial dims are not supported.
"""
from __future__ import annotations

import itertools
import math
from collections.abc import Callable, Mapping, Sequence
from typing import Any

import numpy as np
import torch
import torch.nn.functional as F

from .. import _kernels as K
from .. import _lib as L
from ..data.utils import compute_importance_map, dense_patch_starts, get_valid_patch_size, importance_factors

__all__ = ["sliding_window_inference", "sliding_window_inference_resampled", "resample_matrix"]

# keep at most this many bytes of window predictions resident before they are folded into the accumulators;
# when everything fits, the whole blend is ONE launch (mode 0) and the fp32 accumulators are never allocated.
_RESIDENT_BYTES = 24 << 30


def _resident_budget(device) -> int:
    """Bytes of window predictions kept resident: at most _RESIDENT_BYTES and at most 40 % of the memory currently free on `device`
    (the fp32 accumulators and the network's activations need the rest)."""
    try:
        free, _ = torch.cuda.mem_get_info(device)
        return int(max(1, min(_RESIDENT_BYTES, 0.4 * free)))
    except Exception:  # pragma: no cover - no CUDA context yet
        return _RESIDENT_BYTES

_PAD_MODES = {"constant", "reflect", "replicate", "circular"}


def _ensure_tuple_rep(v, n: int) -> tuple:
    if isinstance(v, torch.Tensor):
        v = v.detach().cpu().numpy()
    if isinstance(v, np.ndarray):
        v = v.tolist()
    if isinstance(v, (list, tuple)):
        if len(v) == n:
            return tuple(v)
        raise ValueError(f"Sequence must have length {n}, got {len(v)}.")
    return (v,) * n


def _fall_back_tuple(user, default: Sequence[int]) -> tuple[int, ...]:
    """`fall_back_tuple` (monai/utils/misc.py): non-positive / None entries take the default."""
    user = _ensure_tuple_rep(user, len(default))
    return tuple(int(u) if (u is not None and u > 0) else int(d) for u, d in zip(user, default))


def _get_scan_interval(image_size, roi_size, num_spatial_dims: int, overlap) -> tuple[int, ...]:
    """monai/inferers/utils.py:363-384 -- int(roi * (1 - overlap)) with float truncation, min 1; roi == image -> roi."""
    if len(image_size) != num_spatial_dims:
        raise ValueError(f"len(image_size) {len(image_size)} different from spatial dims {num_spatial_dims}.")
    if len(roi_size) != num_spatial_dims:
        raise ValueError(f"len(roi_size) {len(roi_size)} different from spatial dims {num_spatial_dims}.")
    out = []
    for i, o in zip(range(num_spatial_dims), overlap):
        if roi_size[i] == image_size[i]:
            out.append(int(roi_size[i]))
        else:
            interval = int(roi_size[i] * (1 - o))
            out.append(interval if interval > 0 else 1)
    return tuple(out)


def _flatten_struct(seg_out):
    dict_keys = None
    if isinstance(seg_out, torch.Tensor):
        seg = (seg_out,)
    elif isinstance(seg_out, Mapping):
        dict_keys = sorted(seg_out.keys())
        seg = tuple(seg_out[k] for k in dict_keys)
    elif isinstance(seg_out, (list, tuple)):
        seg = tuple(seg_out)
    else:
        seg = (seg_out,)
    return dict_keys, seg


def _pack_struct(seg_out, dict_keys=None):
    if dict_keys is not None:
        return dict(zip(dict_keys, seg_out))
    if isinstance(seg_out, (list, tuple)) and len(seg_out) == 1:
        return seg_out[0]
    return tuple(seg_out)


def _is_meta(x) -> bool:
    return hasattr(x, "copy_meta_from") and hasattr(x, "meta")


def _rewrap(out: torch.Tensor, like) -> torch.Tensor:
    """Reference: convert_to_dst_type(final_output, temp_meta) -- a MetaTensor input yields MetaTensor outputs."""
    if like is None:
        return out
    wrapped = type(like)(out)
    wrapped.copy_meta_from(like, copy_attr=False)
    return wrapped


class _OutputPlan:
    """Blend state of one predictor output (the reference's `ss` index)."""

    def __init__(self, seg: torch.Tensor, batch_size, image_size, roi_size, starts, total, device):
        self.chns = int(seg.shape[1])
        seg_shape = tuple(int(s) for s in seg.shape[2:])
        self.z_scale = None
        if seg_shape != tuple(roi_size):
            self.z_scale = [o / float(i) for o, i in zip(seg_shape, roi_size)]
        z = self.z_scale or [1.0, 1.0, 1.0]
        self.roi = seg_shape
        self.vol = tuple(int(i * s) for i, s in zip(image_size, z)) if self.z_scale else tuple(image_size)
        # window starts in output space: int(start * z) exactly as _compute_coords (utils.py:351-360)
        out_starts = [[int(s * zz) for s in ax] for ax, zz in zip(starts, z)]
        # the blend kernels keep at most 32 covering windows per axis in registers / shared tables (blend.cu): an overlap so
        # high that more windows cover one voxel along an axis would be truncated silently -- refuse it here instead
        max_cover = 1
        for ax, r in zip(out_starts, self.roi):
            cover = max((sum(1 for s in ax if s <= v < s + int(r)) for v in sorted(set(ax))), default=1)
            if cover > 32:
                raise ValueError(f"sliding_window_inference: {cover} windows overlap one voxel along an axis; monai_b200 blends at most 32 (lower the overlap)")
            max_cover = max(max_cover, cover)
        self.starts = [torch.tensor(ax, dtype=torch.int32, device=device) for ax in out_starts]
        self.starts[2]._align = math.gcd(8, *out_starts[2])  # 2 / 8 enable the vectorised blend paths
        self.starts[2]._max_cover = max_cover                # <= 3 enables the lean kernel
        self.batch_size = batch_size
        self.total = total
        per_win = self.chns * int(np.prod(seg_shape))
        self.cap = max(1, min(total, _resident_budget(device) // max(1, per_win * seg.element_size())))
        self.store = torch.empty((self.cap, self.chns, *seg_shape), device=device, dtype=seg.dtype)
        self.first = 0      # flat index of store[0]
        self.count = 0      # windows currently resident
        self.acc: torch.Tensor | None = None
        self.dtype = seg.dtype
        self.slot_ids: list[int] = []   # buffered mode: flat window ids of the resident predictions, in slot order
        self.result: torch.Tensor | None = None
        self.factors = None


def sliding_window_inference(
    inputs: torch.Tensor,
    roi_size: Sequence[int] | int,
    sw_batch_size: int,
    predictor: Callable[..., torch.Tensor | Sequence[torch.Tensor] | dict[Any, torch.Tensor]],
    overlap: Sequence[float] | float = 0.25,
    mode: str = "constant",
    sigma_scale: Sequence[float] | float = 0.125,
    padding_mode: str = "constant",
    cval: float = 0.0,
    sw_device: torch.device | str | None = None,
    device: torch.device | str | None = None,
    progress: bool = False,
    roi_weight_map: torch.Tensor | None = None,
    process_fn: Callable | None = None,
    buffer_steps: int | None = None,
    buffer_dim: int = -1,
    with_coord: bool = False,
    *args: Any,
    **kwargs: Any,
) -> torch.Tensor | tuple[torch.Tensor, ...] | dict[Any, torch.Tensor]:
    """Sliding-window inference on `inputs` with `predictor`; see the reference docstring for argument semantics.

    Differences that are improvements rather than incompatibilities: the weighted sum is accumulated in fp32 even
    for fp16 inputs (the reference accumulates in the input dtype, utils.py:148,269-270).  With `buffer_steps` the windows
    are visited in the reference's buffered order (sorted by their start along `buffer_dim`, batches never cross a buffer
    or a batch item, utils.py:182-191, 324-348) and each buffer is folded into the fp32 accumulators when it completes.
    """
    return _swi_core(inputs, roi_size, sw_batch_size, predictor, overlap, mode, sigma_scale, padding_mode, cval, sw_device, device, progress,
                     roi_weight_map, process_fn, buffer_steps, buffer_dim, with_coord, None, args, kwargs)


def sliding_window_inference_resampled(
    inputs: torch.Tensor,
    roi_size: Sequence[int] | int,
    sw_batch_size: int,
    predictor: Callable[..., torch.Tensor],
    matrix: Any,
    output_shape: Sequence[int],
    overlap: Sequence[float] | float = 0.25,
    mode: str = "constant",
    sigma_scale: Sequence[float] | float = 0.125,
    interp_mode: str = "bilinear",
    resample_padding_mode: str = "border",
    padding_mode: str = "constant",
    cval: float = 0.0,
    sw_device: torch.device | str | None = None,
    device: torch.device | str | None = None,
    *args: Any,
    **kwargs: Any,
) -> torch.Tensor:
    """Sliding-window inference whose overlap blend and the affine resampling that follows it run as ONE kernel.

    out[b, c, o] = sample(blend(windows)[b, c], M @ (o, 1)) for a 3x4 (or 4x4) `matrix` M that maps an OUTPUT voxel index to a
    coordinate in the inference grid -- what `sliding_window_inference` followed by `Spacing.inverse` / `SpatialResample`
    computes in the reference (monai/inferers/utils.py:286-298,351-360 then monai/transforms/spatial/functional.py:68-184),
    without ever writing the blended volume.  `interp_mode` "bilinear" | "nearest", `resample_padding_mode` "border" | "zeros".
    3-D volumes, single-tensor predictors.
    """
    m = np.asarray(matrix.detach().cpu().numpy() if isinstance(matrix, torch.Tensor) else matrix, dtype=np.float64)
    if m.shape not in ((3, 4), (4, 4)):
        raise ValueError(f"matrix must be 3x4 or 4x4 (output voxel index -> inference-grid coordinate), got {m.shape}")
    if len(inputs.shape) != 5 or len(tuple(output_shape)) != 3:
        raise NotImplementedError("sliding_window_inference_resampled handles 3-D volumes")
    interp = {"bilinear": 1, "trilinear": 1, "linear": 1, "nearest": 0}.get(str(getattr(interp_mode, "value", interp_mode)).lower())
    pad = {"border": 1, "zeros": 0}.get(str(getattr(resample_padding_mode, "value", resample_padding_mode)).lower())
    if interp is None or pad is None:
        raise ValueError(f"unsupported interp_mode / resample_padding_mode: {interp_mode}, {resample_padding_mode}")
    rs = ([float(v) for v in m[:3].reshape(-1)], tuple(int(v) for v in output_shape), interp, pad)
    return _swi_core(inputs, roi_size, sw_batch_size, predictor, overlap, mode, sigma_scale, padding_mode, cval, sw_device, device, False,
                     None, None, None, -1, False, rs, args, kwargs)


def resample_matrix(src_affine, dst_affine, in_shape: Sequence[int], out_shape: Sequence[int], align_corners: bool = False) -> np.ndarray:
    """3x4 matrix for `sliding_window_inference_resampled`: voxel index on the DESTINATION grid (affine `dst_affine`, shape
    `out_shape`) -> coordinate on the inference grid (affine `src_affine`, shape `in_shape`), with the conventions of
    SpatialResample (monai/transforms/spatial/functional.py:68-184) -- e.g. src = the Spacingd output the network ran on,
    dst = the original image grid: the inverse of Spacingd applied to the logits."""
    from ..transforms import utils as TU

    src = TU.to_affine_nd(3, np.asarray(src_affine, dtype=np.float64))
    dst = TU.to_affine_nd(3, np.asarray(dst_affine, dtype=np.float64))
    xform = TU.to_affine_nd(3, np.linalg.solve(src, dst))
    return TU.sample_matrix_from_xform(xform, tuple(int(v) for v in in_shape), np.asarray([int(v) for v in out_shape]), align_corners)


def _create_buffered_order(starts_nd, roi_size, batch_size: int, sw_batch_size: int, buffer_dim: int, buffer_steps: int):
    """Window order and buffer boundaries of the reference's buffered mode (monai/inferers/utils.py:324-348).

    Returns (order, groups): `order` = permutation of the canonical ("ij") window ids, stably sorted by the start along
    `buffer_dim`; `groups` = list of (first, last) positions IN THE SORTED LIST per buffer and batch item, expressed as flat
    indices b * num_win + position, in visiting order."""
    flat = list(itertools.product(*starts_nd))
    num_win = len(flat)
    key = np.asarray([f[buffer_dim] for f in flat])
    order = np.argsort(key, kind="mergesort")
    sorted_key = key[order]
    _, counts = np.unique(sorted_key, return_counts=True)
    b_ends = np.cumsum(counts).tolist()                      # possible buffer flush boundaries
    x = [0, *b_ends][:: min(len(b_ends), int(buffer_steps))]
    if x[-1] < b_ends[-1]:
        x.append(b_ends[-1])
    groups = [(b * num_win + x[i], b * num_win + x[i + 1]) for b in range(batch_size) for i in range(len(x) - 1)]
    return order, groups


def _swi_core(inputs, roi_size, sw_batch_size, predictor, overlap, mode, sigma_scale, padding_mode, cval, sw_device, device, progress,
              roi_weight_map, process_fn, buffer_steps, buffer_dim, with_coord, resample, args, kwargs):
    buffered = buffer_steps is not None and buffer_steps > 0
    num_spatial_dims = len(inputs.shape) - 2
    if buffered:
        if buffer_dim < -num_spatial_dims or buffer_dim > num_spatial_dims:
            raise ValueError(f"buffer_dim must be in [{-num_spatial_dims}, {num_spatial_dims}], got {buffer_dim}.")
        if buffer_dim < 0:
            buffer_dim += num_spatial_dims
    overlap = _ensure_tuple_rep(overlap, num_spatial_dims)
    for o in overlap:
        if o < 0 or o >= 1:
            raise ValueError(f"overlap must be >= 0 and < 1, got {overlap}.")
    if num_spatial_dims < 1 or num_spatial_dims > 3:
        raise NotImplementedError(f"monai_b200 sliding_window_inference supports 1-3 spatial dims, got {num_spatial_dims}.")
    mode_s = str(getattr(mode, "value", mode)).lower()
    pad_s = str(getattr(padding_mode, "value", padding_mode)).lower()
    if pad_s not in _PAD_MODES:
        raise ValueError(f"unsupported padding_mode {padding_mode}, available options are {sorted(_PAD_MODES)}.")
    if not inputs.is_cuda and sw_device is None:
        raise RuntimeError("monai_b200.sliding_window_inference needs CUDA inputs (or an explicit CUDA sw_device); there is no CPU path.")
    L.load()  # fail loudly when the CUDA library is missing

    compute_dtype = inputs.dtype
    batch_size, _, *image_size_ = inputs.shape
    out_device = torch.device(device) if device is not None else inputs.device
    sw_dev = torch.device(sw_device) if sw_device is not None else inputs.device
    if sw_dev.type != "cuda":
        raise RuntimeError(f"sw_device must be a CUDA device, got {sw_dev}.")

    temp_meta = inputs if _is_meta(inputs) else None
    x = inputs.as_subclass(torch.Tensor) if type(inputs) is not torch.Tensor else inputs
    x = x.detach()
    if x.dtype == torch.float64:   # float64 volumes are blended in fp32 and returned as float64 (the kernels take f16 / f32)
        x = x.float()
    roi_size = _fall_back_tuple(roi_size, image_size_)

    # pad when the image is smaller than the roi (utils.py:163-170): symmetric, half / diff-half
    image_size = tuple(max(image_size_[i], roi_size[i]) for i in range(num_spatial_dims))
    pad_size: list[int] = []
    for k in range(len(x.shape) - 1, 1, -1):
        diff = max(roi_size[k - 2] - x.shape[k], 0)
        half = diff // 2
        pad_size.extend([half, diff - half])
    if any(pad_size):
        x = F.pad(x, pad=pad_size, mode=pad_s, value=cval)
    x = x.to(sw_dev)

    # fused resample: the kernel samples the PADDED blended volume, so the matrix takes the leading pad of each axis
    rs_plan = None
    if resample is not None:
        mat, oshape, interp, rpad = resample
        mat = list(mat)
        for ax in range(3):
            mat[4 * ax + 3] += float(pad_size[2 * (2 - ax)]) if any(pad_size) else 0.0   # pad_size lists the LAST axis first
        rs_plan = (mat, oshape, interp, rpad)
    scan_interval = _get_scan_interval(image_size, roi_size, num_spatial_dims, overlap)
    starts_nd = dense_patch_starts(image_size, roi_size, scan_interval)
    valid_patch_size = get_valid_patch_size(image_size, roi_size)
    num_win = int(np.prod([len(s) for s in starts_nd]))
    total_slices = num_win * batch_size

    # lift to 3-D with leading singleton axes so one kernel family serves 1-D/2-D/3-D
    lift = 3 - num_spatial_dims
    x3 = x.reshape(x.shape[0], x.shape[1], *([1] * lift), *x.shape[2:])
    image3 = (1,) * lift + tuple(image_size)
    roi3 = (1,) * lift + tuple(roi_size)
    starts3 = [[0]] * lift + starts_nd
    flat_starts = list(itertools.product(*starts3))  # "ij" order, first axis slowest

    # importance map: separable factors for the kernel; a dense map only when the caller supplies / needs one
    dense_w: torch.Tensor | None = None
    factors = None
    clamp = 1.0
    if valid_patch_size == tuple(roi_size) and roi_weight_map is not None:
        dense_w = torch.as_tensor(roi_weight_map).to(device=sw_dev, dtype=torch.float32)
    else:
        try:
            f_nd, clamp = importance_factors(valid_patch_size, mode_s, sigma_scale)
        except ValueError:
            raise
        except Exception as e:  # pragma: no cover
            raise RuntimeError(
                f"patch size {valid_patch_size}, mode={mode}, sigma_scale={sigma_scale}, device={device}\n"
                "Seems to be OOM. Please try smaller patch size or mode='constant' instead of mode='gaussian'."
            ) from e
        factors = [torch.ones(1)] * lift + f_nd
        factors = [f.to(sw_dev) for f in factors]
    importance_map_for_fn = None
    if process_fn is not None:
        importance_map_for_fn = (
            dense_w.to(compute_dtype) if dense_w is not None
            else compute_importance_map(valid_patch_size, mode_s, sigma_scale, sw_dev, compute_dtype)
        )

    w_align = math.gcd(16, *[int(v) for v in starts3[2]])   # the gather copies 16-byte vectors when the W starts allow it
    win_tab_all = torch.tensor(
        [(b, *s) for b in range(batch_size) for s in flat_starts], dtype=torch.int32, device=sw_dev
    ).reshape(-1, 4)

    plans: list[_OutputPlan] = []
    dict_keys = None
    first_wmaps: list[torch.Tensor | None] = []

    def _dense3(w: torch.Tensor, shape3) -> torch.Tensor:
        return w.to(device=sw_dev, dtype=torch.float32).reshape(shape3).contiguous()

    def _out_shape(pl: _OutputPlan):
        return (batch_size, pl.chns, *(rs_plan[1] if rs_plan is not None else pl.vol))

    def _flush(pl: _OutputPlan, wmap_now: torch.Tensor | None, final: bool) -> None:
        """Fold the resident predictions into the result (mode 0 when they are ALL resident, else mode 1)."""
        if pl.count == 0:
            return
        vol_shape = (batch_size, pl.chns, *pl.vol)
        preds = pl.store[: pl.count]
        if buffered:
            # the resident predictions are the windows `pl.slot_ids` (visiting order != id order): look them up through a slot map
            if pl.acc is None:
                pl.acc = torch.zeros(vol_shape, device=sw_dev, dtype=torch.float32)
            slot_map = torch.full((total_slices,), -1, dtype=torch.int32, device=sw_dev)
            slot_map[torch.tensor(pl.slot_ids, dtype=torch.int64, device=sw_dev)] = torch.arange(pl.count, dtype=torch.int32, device=sw_dev)
            K.sw_blend(1, preds, 0, 0, vol_shape, pl.roi, pl.starts, pl.factors, clamp, wmap_now, pl.acc, slot_map=slot_map, n_slots=pl.count)
            pl.slot_ids = []
        elif final and pl.acc is None and pl.count == pl.total:
            pl.result = torch.empty(_out_shape(pl), device=sw_dev, dtype=pl.dtype)
            K.sw_blend(0, preds, 0, pl.total, vol_shape, pl.roi, pl.starts, pl.factors, clamp, wmap_now, pl.result, resample=rs_plan)
        else:
            if pl.acc is None:
                pl.acc = torch.zeros(vol_shape, device=sw_dev, dtype=torch.float32)
            K.sw_blend(1, preds, pl.first, pl.first + pl.count, vol_shape, pl.roi, pl.starts, pl.factors, clamp, wmap_now, pl.acc)
        pl.first += pl.count
        pl.count = 0

    # batches of flat window ids (b * num_win + canonical "ij" id) in visiting order; `ends` = batches after which a buffer is complete
    if not buffered:
        batches: list = [range(g, min(g + sw_batch_size, total_slices)) for g in range(0, total_slices, sw_batch_size)]
        ends: set = set()
    else:
        order, groups = _create_buffered_order(starts_nd, roi_size, batch_size, sw_batch_size, buffer_dim, int(buffer_steps))
        batches, ends = [], set()
        for first, last in groups:
            b_off = (first // num_win) * num_win
            for g in range(first, last, sw_batch_size):
                batches.append([b_off + int(order[pos - b_off]) for pos in range(g, min(g + sw_batch_size, last))])
            ends.add(len(batches) - 1)
    it = batches
    if progress:
        try:
            from tqdm import tqdm

            it = tqdm(batches)
        except ImportError:  # pragma: no cover
            pass
    nd_slices = [tuple(slice(s, s + r) for s, r in zip(st[lift:], roi_size)) for st in flat_starts]
    for bi, slice_range in enumerate(it):
        if isinstance(slice_range, range):
            tab = win_tab_all[slice_range.start : slice_range.stop]
        else:
            tab = win_tab_all[torch.tensor(slice_range, dtype=torch.int64, device=sw_dev)]
        win_data3 = K.sw_gather(x3, tab, roi3, w_align=w_align)
        win_data = win_data3.reshape(win_data3.shape[0], win_data3.shape[1], *roi_size)
        if with_coord:
            unravel_slice = [
                [slice(idx // num_win, idx // num_win + 1), slice(None)] + list(nd_slices[idx % num_win]) for idx in slice_range
            ]
            seg_prob_out = predictor(win_data, unravel_slice, *args, **kwargs)
        else:
            seg_prob_out = predictor(win_data, *args, **kwargs)
        dict_keys, seg_tuple = _flatten_struct(seg_prob_out)
        if buffered:
            seg_tuple = tuple(seg_tuple[:1])   # the reference's buffered mode blends the first output only (utils.py:241)
        w_t = None
        if process_fn is not None:
            seg_tuple, w_t = process_fn(seg_tuple, win_data, importance_map_for_fn)
            seg_tuple = tuple(seg_tuple)
        for ss, seg in enumerate(seg_tuple):
            if not isinstance(seg, torch.Tensor) or seg.dim() != num_spatial_dims + 2:
                raise ValueError(f"predictor output {ss} must be a tensor with {num_spatial_dims} spatial dims, got {type(seg)}.")
            seg = seg.detach()
            if seg.device != sw_dev:
                seg = seg.to(sw_dev)
            if seg.dtype not in (torch.float16, torch.float32):
                seg = seg.float()
            seg3 = seg.reshape(seg.shape[0], seg.shape[1], *([1] * lift), *seg.shape[2:])
            if len(plans) <= ss:
                pl = _OutputPlan(seg3, batch_size, image3, roi3, starts3, total_slices, sw_dev)
                # weight map in output space: separable factors unless a dense map / other resolution is involved
                wsrc = w_t if w_t is not None else dense_w
                if wsrc is None and pl.z_scale is None:
                    pl.factors, wm = factors, None
                else:
                    if wsrc is None:
                        wsrc = compute_importance_map(valid_patch_size, mode_s, sigma_scale, sw_dev, torch.float32)
                    wm = _dense3(wsrc, roi3)
                    if pl.z_scale is not None:  # nearest-exact resize of the weight map (utils.py:263)
                        wm = F.interpolate(wm[None, None], size=pl.roi, mode="nearest-exact")[0, 0].contiguous()
                    pl.factors = None
                first_wmaps.append(wm)
                plans.append(pl)
            pl = plans[ss]
            if tuple(seg3.shape[1:]) != (pl.chns, *pl.roi):
                raise ValueError(f"predictor output {ss} changed shape between windows: {tuple(seg3.shape)}")
            wm_now = first_wmaps[ss]
            if w_t is not None and pl.factors is None:
                wm_now = _dense3(w_t, roi3)
                if pl.z_scale is not None:
                    wm_now = F.interpolate(wm_now[None, None], size=pl.roi, mode="nearest-exact")[0, 0].contiguous()
            n = seg3.shape[0]
            if pl.count + n > pl.cap:
                _flush(pl, wm_now, final=False)
            pl.store[pl.count : pl.count + n].copy_(seg3)
            pl.count += n
            if buffered:
                pl.slot_ids.extend(int(i) for i in slice_range)
            if process_fn is not None:  # the weight map may change from batch to batch: fold immediately
                _flush(pl, wm_now, final=(pl.first + pl.count == pl.total and pl.acc is None))
            elif buffered and bi in ends:   # this buffer is complete: fold it into the accumulators
                _flush(pl, wm_now, final=False)

    outputs = []
    for ss, pl in enumerate(plans):
        _flush(pl, first_wmaps[ss], final=True)
        if pl.result is None:
            vol_shape = (batch_size, pl.chns, *pl.vol)
            pl.result = torch.empty(_out_shape(pl), device=sw_dev, dtype=pl.dtype)
            # count map is analytic: sum of the (first) weight map over all windows (utils.py:272-275)
            K.sw_blend(2, None, 0, pl.total, vol_shape, pl.roi, pl.starts, pl.factors, clamp, first_wmaps[ss], pl.result, acc=pl.acc, resample=rs_plan)
            pl.acc = None
        if rs_plan is not None:
            if pl.z_scale is not None:
                raise NotImplementedError("sliding_window_inference_resampled needs predictor outputs at the window resolution")
            outputs.append(pl.result)
            pl.store = None
            continue
        out = pl.result.reshape(batch_size, pl.chns, *pl.vol[lift:])
        pl.store = None
        outputs.append(out)

    # remove padding if the image was smaller than the roi (utils.py:301-313)
    if any(pad_size) and rs_plan is None:
        for ss, out in enumerate(outputs):
            zoom_scale = [s / r for s, r in zip(out.shape[2:], roi_size)]
            final_slicing: list[slice] = []
            for sp in range(num_spatial_dims):
                si = num_spatial_dims - sp - 1
                final_slicing.insert(
                    0,
                    slice(
                        int(round(pad_size[sp * 2] * zoom_scale[si])),
                        int(round((pad_size[sp * 2] + image_size_[si]) * zoom_scale[si])),
                    ),
                )
            outputs[ss] = out[(slice(None), slice(None), *final_slicing)]

    outputs = [o.to(device=out_device, dtype=compute_dtype if compute_dtype in (torch.float16, torch.float32, torch.float64) else o.dtype) for o in outputs]
    outputs = [_rewrap(o, temp_meta) for o in outputs]
    return _pack_struct(outputs, dict_keys)
