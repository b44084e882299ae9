"""Inferer classes with the reference's constructor / call signatures (monai/inferers/inferer.py:62-97, 399-552).

`SlidingWindowInferer` stores its arguments and calls the H100-native `sliding_window_inference` positionally,
exactly as the reference does (inferer.py:532-552).  `SlidingWindowInfererAdapt` keeps its name and signature; the
OOM ladder of the reference (inferer.py:565-641) degrades gracefully here because the resident-prediction budget
already bounds memory, so it only adds the `cpu_thresh` bookkeeping.
"""
from __future__ import annotations

import warnings
from abc import ABC, abstractmethod
from collections.abc import Callable, Mapping, Sequence
from typing import Any

import torch

from ..data.utils import compute_importance_map
from .merger import AvgMerger, Merger
from .splitter import Splitter
from .utils import sliding_window_inference

__all__ = ["Inferer", "SimpleInferer", "PatchInferer", "SlidingWindowInferer", "SlidingWindowInfererAdapt", "SliceInferer"]


class Inferer(ABC):
    """Base class: `inferer(inputs, network, *args, **kwargs)` (inferer.py:62-97)."""

    @abstractmethod
    def __call__(self, inputs: torch.Tensor, network: Callable, *args: Any, **kwargs: Any) -> Any:
        raise NotImplementedError(f"Subclass {self.__class__.__name__} must implement this method.")


class SimpleInferer(Inferer):
    """Runs `network(inputs, *args, **kwargs)` (inferer.py:373-396)."""

    def __call__(self, inputs: torch.Tensor, network: Callable, *args: Any, **kwargs: Any):
        return network(inputs, *args, **kwargs)


class SlidingWindowInferer(Inferer):
    def __init__(
        self,
        roi_size: Sequence[int] | int,
        sw_batch_size: int = 1,
        overlap: Sequence[float] | float = 0.25,
        mode: str = "constant",
        sigma_scale: Sequence[float] | float = 0.125,
        padding_mode: str = "constant",
        cval: float = 0.0,
        sw_device: torch.device | str | None = None,
        device: torch.device | str | None = None,
        progress: bool = False,
        cache_roi_weight_map: bool = False,
        cpu_thresh: int | None = None,
        buffer_steps: int | None = None,
        buffer_dim: int = -1,
        with_coord: bool = False,
    ) -> None:
        super().__init__()
        mode_s = str(getattr(mode, "value", mode)).lower()
        if mode_s not in ("constant", "gaussian"):
            raise ValueError(f"'{mode}' is not a valid BlendMode")
        self.roi_size = roi_size
        self.sw_batch_size = sw_batch_size
        self.overlap = overlap
        self.mode = mode_s
        self.sigma_scale = sigma_scale
        self.padding_mode = padding_mode
        self.cval = cval
        self.sw_device = sw_device
        self.device = device
        self.progress = progress
        self.cpu_thresh = cpu_thresh
        self.buffer_steps = buffer_steps
        self.buffer_dim = buffer_dim
        self.with_coord = with_coord
        # the reference precomputes the dense map to avoid recomputing it per call; the CUDA blend only needs the
        # separable factors, which cost nothing -- the cached map is kept for attribute compatibility.
        self.roi_weight_map = None
        try:
            if cache_roi_weight_map and isinstance(roi_size, Sequence) and min(roi_size) > 0:
                self.roi_weight_map = compute_importance_map(
                    tuple(self.roi_size), mode=mode_s, sigma_scale=sigma_scale, device=device if device is not None else "cpu"
                )
            if cache_roi_weight_map and self.roi_weight_map is None:
                warnings.warn("cache_roi_weight_map=True, but cache is not created. (dynamic roi_size?)")
        except BaseException as e:
            raise RuntimeError(
                f"roi size {self.roi_size}, mode={mode}, sigma_scale={sigma_scale}, device={device}\n"
                "Seems to be OOM. Please try smaller patch size or mode='constant' instead of mode='gaussian'."
            ) from e

    def __call__(self, inputs: torch.Tensor, network: Callable, *args: Any, **kwargs: Any):
        device = kwargs.pop("device", self.device)
        buffer_steps = kwargs.pop("buffer_steps", self.buffer_steps)
        buffer_dim = kwargs.pop("buffer_dim", self.buffer_dim)
        if device is None and self.cpu_thresh is not None and inputs.shape[2:].numel() > self.cpu_thresh:
            device = "cpu"  # stitched result is handed back in host memory for very large images
        return sliding_window_inference(
            inputs,
            self.roi_size,
            self.sw_batch_size,
            network,
            self.overlap,
            self.mode,
            self.sigma_scale,
            self.padding_mode,
            self.cval,
            self.sw_device,
            device,
            self.progress,
            self.roi_weight_map,
            None,
            buffer_steps,
            buffer_dim,
            self.with_coord,
            *args,
            **kwargs,
        )


class SlidingWindowInfererAdapt(SlidingWindowInferer):
    """The reference's adaptive policy (monai/inferers/inferer.py:555-641) with the same call contract: stitch on the GPU; after a
    CUDA out-of-memory error switch to buffered stitching (halving `buffer_steps` on further failures) and finally to a result
    held in host memory; `cpu_thresh` remembers the size from which GPU stitching is not attempted again.  With an explicit
    stitching `device` no adaptation takes place.  The buffer axis is the longest one when it is at least twice the last axis."""

    def __call__(self, inputs: torch.Tensor, network: Callable, *args: Any, **kwargs: Any):
        if self.device is not None:
            return super().__call__(inputs, network, *args, **kwargs)
        skip_buffer = self.buffer_steps is not None and self.buffer_steps <= 0
        cpu_cond = self.cpu_thresh is not None and inputs.shape[2:].numel() > self.cpu_thresh
        gpu_stitching = inputs.is_cuda and not cpu_cond
        buffered_stitching = inputs.is_cuda and cpu_cond and not skip_buffer
        buffer_steps = max(1, self.buffer_steps) if self.buffer_steps is not None else 1
        buffer_dim = -1
        sh = list(inputs.shape[2:])
        max_dim = sh.index(max(sh))
        if inputs.shape[max_dim + 2] / inputs.shape[-1] >= 2:
            buffer_dim = max_dim
        for _ in range(10):  # at most 10 trials
            try:
                return super().__call__(
                    inputs, network, *args, device=inputs.device if gpu_stitching else torch.device("cpu"),
                    buffer_steps=buffer_steps if buffered_stitching else None, buffer_dim=buffer_dim, **kwargs,
                )
            except RuntimeError as e:
                if (not gpu_stitching and not buffered_stitching) or "OutOfMemoryError" not in type(e).__name__:
                    raise
                torch.cuda.empty_cache()
                if gpu_stitching:  # GPU stitching failed: remember the size, go buffered (or straight to the host)
                    gpu_stitching = False
                    self.cpu_thresh = inputs.shape[2:].numel() - 1
                    if skip_buffer:
                        buffered_stitching = False
                        warnings.warn(f"GPU stitching failed, attempting on CPU, image dim {tuple(inputs.shape)}.")
                    else:
                        buffered_stitching = True
                        self.buffer_steps = buffer_steps
                        warnings.warn(f"GPU stitching failed, buffer {buffer_steps} dim {buffer_dim}, image dim {tuple(inputs.shape)}.")
                elif buffer_steps > 1:
                    buffer_steps = max(1, buffer_steps // 2)
                    self.buffer_steps = buffer_steps
                    warnings.warn(f"GPU buffered stitching failed, image dim {tuple(inputs.shape)} reducing buffer to {buffer_steps}.")
                else:
                    buffered_stitching = False
                    warnings.warn(f"GPU buffered stitching failed, attempting on CPU, image dim {tuple(inputs.shape)}.")
        raise RuntimeError(f"SlidingWindowInfererAdapt {skip_buffer} {cpu_cond} {gpu_stitching} {buffered_stitching} {buffer_steps}")


class SliceInferer(SlidingWindowInferer):
    """Slice-by-slice (2-D network) inference over a 3-D volume with the same contract as the reference class
    (monai/inferers/inferer.py:691-771): `roi_size` is 2-D, a singleton is inserted at `spatial_dim`, the window batch is
    squeezed before the 2-D network runs and its outputs (tensor, sequence or mapping) are unsqueezed again.  Gather and
    blend run in the CUDA kernels of `sliding_window_inference`; the 2-D predictor is any callable."""

    def __init__(self, spatial_dim: int = 0, *args: Any, **kwargs: Any) -> None:
        self.spatial_dim = spatial_dim
        super().__init__(*args, **kwargs)
        roi = self.roi_size
        self.orig_roi_size = tuple(roi) if isinstance(roi, (list, tuple)) else (roi,)

    def __call__(self, inputs: torch.Tensor, network: Callable, *args: Any, **kwargs: Any):
        if self.spatial_dim > 2:
            raise ValueError("`spatial_dim` can only be `0, 1, 2` with `[H, W, D]` respectively.")
        if len(self.orig_roi_size) == 2 and len(inputs.shape[2:]) == 3:
            roi = list(self.orig_roi_size)
            roi.insert(self.spatial_dim, 1)
            self.roi_size = roi
        else:
            raise RuntimeError(
                f"Currently, only 2D `roi_size` ({self.orig_roi_size}) with 3D `inputs` tensor (shape={inputs.shape}) is supported."
            )
        return super().__call__(inputs, lambda x: self.network_wrapper(network, x, *args, **kwargs))

    def network_wrapper(self, network: Callable, x: torch.Tensor, *args: Any, **kwargs: Any):
        dim = self.spatial_dim + 2
        out = network(x.squeeze(dim=dim), *args, **kwargs)
        if isinstance(out, torch.Tensor):
            return out.unsqueeze(dim=dim)
        if isinstance(out, Mapping):
            return {k: v.unsqueeze(dim=dim) for k, v in out.items()}
        return tuple(o.unsqueeze(dim=dim) for o in out)


class PatchInferer(Inferer):
    """Inference on patches from a `Splitter`, merged by a `Merger` (reference: monai/inferers/inferer.py:100-370).  Same
    constructor / call contract: `batch_size` patches are concatenated per network call, `preprocessing` / `postprocessing`
    wrap the network, tuple / dict outputs get one merger each (`output_keys` selects and orders dict entries), output
    patches may be resized with respect to the input patches (the location is scaled by the size ratio), and
    `match_spatial_shape` crops the padded merge back to the (scaled) input shape.  `buffer_size` (a background sampling
    thread in the reference) is accepted and ignored: splitting here is a view of a device tensor."""

    def __init__(self, splitter: Splitter | None = None, merger_cls: type[Merger] | str = AvgMerger, batch_size: int = 1,
                 preprocessing: Callable | None = None, postprocessing: Callable | None = None, output_keys: Sequence | None = None,
                 match_spatial_shape: bool = True, buffer_size: int = 0, **merger_kwargs: Any) -> None:
        Inferer.__init__(self)
        if not isinstance(splitter, (Splitter, type(None))):
            raise TypeError(
                f"'splitter' should be a `Splitter` object that returns: "
                "an iterable of pairs of (patch, location) or a MetaTensor that has `PatchKeys.LOCATION` metadata)."
                f"{type(splitter)} is given."
            )
        self.splitter = splitter
        if isinstance(merger_cls, str):
            from . import merger as _merger_mod

            found = getattr(_merger_mod, merger_cls, None)
            if found is None:
                from pydoc import locate

                found = locate(merger_cls)
            if found is None:
                raise ValueError(f"The requested `merger_cls` ['{merger_cls}'] does not exist.")
            merger_cls = found
        if not (isinstance(merger_cls, type) and issubclass(merger_cls, Merger)):
            raise TypeError(f"'merger' should be a subclass of `Merger`, {merger_cls} is given.")
        self.merger_cls = merger_cls
        self.merger_kwargs = merger_kwargs
        if preprocessing is not None and not callable(preprocessing):
            raise TypeError(f"'preprocessing' should be a callable object, {type(preprocessing)} is given.")
        self.preprocessing = preprocessing
        if postprocessing is not None and not callable(postprocessing):
            raise TypeError(f"'postprocessing' should be a callable object, {type(postprocessing)} is given.")
        self.postprocessing = postprocessing
        if batch_size < 1:
            raise ValueError(f"`batch_size` must be a positive number, {batch_size} is given.")
        self.batch_size = batch_size
        self.output_keys = output_keys
        self.match_spatial_shape = match_spatial_shape
        self.buffer_size = buffer_size

    def _batches(self, patches):
        batch, locs = [], []
        for patch, loc in patches:
            batch.append(patch)
            locs.append(loc)
            if len(batch) == self.batch_size:
                yield torch.cat(batch), locs, len(batch)
                batch, locs = [], []
        if batch:
            yield torch.cat(batch), locs, len(batch)

    def _as_tuple(self, outputs: Any) -> tuple:
        if isinstance(outputs, dict):
            if self.output_keys is None:
                self.output_keys = list(outputs.keys())
            return tuple(outputs[k] for k in self.output_keys)
        return tuple(outputs) if isinstance(outputs, (list, tuple)) else (outputs,)

    def _merged_shapes(self, inputs, out_patch, ratio):
        if self.splitter is None:
            return None, None
        original = self.splitter.get_input_shape(inputs)
        padded = self.splitter.get_padded_shape(inputs)
        cropped_shape = tuple(out_patch.shape[:2]) + tuple(round(s * r) for s, r in zip(original, ratio))
        merged_shape = tuple(out_patch.shape[:2]) + tuple(round(s * r) for s, r in zip(padded, ratio))
        if not self.match_spatial_shape:
            cropped_shape = merged_shape
        return cropped_shape, merged_shape

    def __call__(self, inputs: torch.Tensor, network: Callable, *args: Any, **kwargs: Any) -> Any:
        if self.splitter is None:
            if isinstance(inputs, torch.Tensor):
                raise ValueError(
                    "`splitter` should be set if the input is not already split into patches. "
                    "For inputs that are split, the location of patches needs to be provided as "
                    "(image, location) pairs, or as `PatchKey.LOCATION` metadata in a MetaTensor. "
                    f"The provided inputs type is {type(inputs)}."
                )
            patches_locations = inputs
        else:
            patches_locations = self.splitter(inputs)
        mergers: list[Merger] = []
        ratios: list[tuple] = []
        for patches, locations, nb in self._batches(patches_locations):
            if self.preprocessing:
                patches = self.preprocessing(patches)
            outputs = network(patches, *args, **kwargs)
            if self.postprocessing:
                outputs = self.postprocessing(outputs)
            outputs = self._as_tuple(outputs)
            if not mergers:
                in_patch = torch.chunk(patches, nb)[0]
                for out_batch in outputs:
                    out_patch = torch.chunk(out_batch, nb)[0]
                    ratio = tuple(op / ip for ip, op in zip(in_patch.shape[2:], out_patch.shape[2:]))
                    mk = dict(self.merger_kwargs)
                    cropped_shape, merged_shape = self._merged_shapes(inputs, out_patch, ratio)
                    if "merged_shape" not in mk:
                        mk["merged_shape"] = merged_shape
                        if mk["merged_shape"] is None:
                            raise ValueError("`merged_shape` cannot be `None`.")
                    if "cropped_shape" not in mk:
                        mk["cropped_shape"] = cropped_shape
                    if "device" not in mk and issubclass(self.merger_cls, AvgMerger):
                        mk["device"] = out_patch.device
                    mergers.append(self.merger_cls(**mk))
                    ratios.append(ratio)
            for out_batch, merger, ratio in zip(outputs, mergers, ratios):
                for in_loc, out_patch in zip(locations, torch.chunk(out_batch, nb)):
                    merger.aggregate(out_patch, [round(l * r) for l, r in zip(in_loc, ratio)])
        merged = [m.finalize() for m in mergers]
        if self.output_keys:
            return dict(zip(self.output_keys, merged))
        return merged[0] if len(merged) == 1 else merged
