"""CPU-only checks of the host side: planner arithmetic (bit-exact vs the reference fixtures), the C-ABI library
loads and exports every symbol include/monai_b200.h declares, and argument validation of the drop-in API."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest
import torch

from monai_b200 import _lib
from monai_b200.data import utils as du
from monai_b200.inferers import SlidingWindowInferer, sliding_window_inference
from monai_b200.inferers.utils import _get_scan_interval

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_planner_bit_exact(golden_dir):
    g = np.load(os.path.join(golden_dir, "planner.npz"))
    for i in range(int(g["n"])):
        image, roi, ov = tuple(g[f"c{i}.image"]), tuple(g[f"c{i}.roi"]), tuple(g[f"c{i}.overlap"])
        image_p = tuple(int(max(a, b)) for a, b in zip(image, roi))
        interval = _get_scan_interval(image_p, roi, len(image), ov)
        assert interval == tuple(g[f"c{i}.interval"])
        sl = du.dense_patch_slices(image_p, roi, interval)
        np.testing.assert_array_equal(np.array([[s.start for s in w] for w in sl]), g[f"c{i}.starts"])
        assert all(w[d].stop - w[d].start == min(roi[d], image_p[d]) for w in sl for d in range(len(roi)))


def test_importance_factors_reproduce_the_dense_map(golden_dir):
    g = np.load(os.path.join(golden_dir, "planner.npz"))
    for j in range(int(g["n_imp"])):
        sig = g[f"imp{j}.sigma"].tolist()
        sig = sig[0] if len(sig) == 1 else tuple(sig)
        patch, mode = tuple(int(v) for v in g[f"imp{j}.patch"]), str(g[f"imp{j}.mode"])
        dense = du.compute_importance_map(patch, mode, sig).numpy()
        np.testing.assert_array_equal(dense, g[f"imp{j}.map"])
        f, clamp = du.importance_factors(patch, mode, sig)
        m = f[0].numpy()
        for i, v in enumerate(f[1:], start=1):
            m = (m[..., None] * v.numpy()[(None,) * i]).astype(np.float32)
        np.testing.assert_array_equal(np.maximum(m, np.float32(clamp)), g[f"imp{j}.map"])


def test_get_valid_patch_size_follows_reference_code():
    assert du.get_valid_patch_size((10, 20, 30), 5) == (5, 20, 30)
    assert du.get_valid_patch_size((10, 20, 30), (5, 0)) == (5, 20, 30)
    assert du.get_valid_patch_size((10, 20, 30), (50, None, 7)) == (10, 20, 7)


def test_abi_exports_every_declared_symbol():
    header = open(os.path.join(ROOT, "include", "monai_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    assert os.path.exists(_lib.LIB_PATH), f"{_lib.LIB_PATH} missing: run python -m monai_b200._build"
    lib = ctypes.CDLL(str(_lib.LIB_PATH))
    missing = [s for s in sorted(declared) if not hasattr(lib, s)]
    assert not missing, f"symbols declared in include/monai_b200.h but not exported: {missing}"
    assert declared == set(_lib.SIGNATURES), (declared ^ set(_lib.SIGNATURES))
    assert _lib.load().b200_abi_version() == _lib.ABI_VERSION


def test_struct_layouts_match_abi3_header():
    # sanity: ctypes mirrors must be at least as large as the packed field sum and 8-byte aligned
    assert ctypes.sizeof(_lib.BlendDesc) % 8 == 0
    assert ctypes.sizeof(_lib.ConvDesc) == 21 * 4 + 4 + 16
    # 10 ints, in_stats (offset 40), eps, act, slope, pad; res_w, res_y, res_ctot, res_coff, res_stats; in_gamma, in_beta, add, add_ctot, add_coff
    assert ctypes.sizeof(_lib.ConvTcDesc) == 128
    assert (_lib.ConvTcDesc.in_stats.offset, _lib.ConvTcDesc.res_w.offset, _lib.ConvTcDesc.in_gamma.offset, _lib.ConvTcDesc.add.offset,
            _lib.ConvTcDesc.add_coff.offset) == (40, 64, 96, 112, 124)


def test_argument_validation_matches_reference():
    x = torch.zeros(1, 1, 8, 8, 8)
    with pytest.raises(ValueError, match="overlap must be >= 0 and < 1"):
        sliding_window_inference(x, (4, 4, 4), 1, lambda t: t, overlap=1.0)
    with pytest.raises(ValueError, match="overlap must be >= 0 and < 1"):
        sliding_window_inference(x, (4, 4, 4), 1, lambda t: t, overlap=(0.5, -0.1, 0.5))
    with pytest.raises(ValueError, match="buffer_dim must be in"):
        sliding_window_inference(x, (4, 4, 4), 1, lambda t: t, buffer_steps=2, buffer_dim=7)
    with pytest.raises(RuntimeError, match="CUDA"):
        sliding_window_inference(x, (4, 4, 4), 1, lambda t: t)  # CPU tensors: no silent fallback
    with pytest.raises(ValueError):
        SlidingWindowInferer((4, 4, 4), mode="nonsense")


def test_kernels_refuse_cpu_tensors():
    from monai_b200 import _kernels as K

    with pytest.raises(RuntimeError, match="CUDA"):
        K.instnorm_stats(torch.zeros(1, 2, 4, 4, 4))
    with pytest.raises(RuntimeError, match="CUDA"):
        K.conv3d_direct(torch.zeros(1, 1, 4, 4, 4), torch.zeros(2, 1, 3, 3, 3))


def test_slice_inferer_argument_errors_match_reference():
    """SliceInferer (monai/inferers/inferer.py:691-771): bad `spatial_dim` -> ValueError, non-2D roi or non-3D input -> RuntimeError,
    both raised before any device work."""
    import pytest
    import torch

    from monai_b200.inferers import SliceInferer

    x = torch.zeros(1, 1, 4, 8, 8)
    with pytest.raises(ValueError, match="spatial_dim"):
        SliceInferer(roi_size=(8, 8), spatial_dim=3, sw_batch_size=1)(x, lambda t: t)
    with pytest.raises(RuntimeError, match="only 2D `roi_size`"):
        SliceInferer(roi_size=(4, 8, 8), spatial_dim=0, sw_batch_size=1)(x, lambda t: t)
    with pytest.raises(RuntimeError, match="only 2D `roi_size`"):
        SliceInferer(roi_size=(8, 8), spatial_dim=0, sw_batch_size=1)(torch.zeros(1, 1, 8, 8), lambda t: t)
    inf = SliceInferer(roi_size=(8, 8), spatial_dim=1, sw_batch_size=2, cval=-1)
    assert inf.orig_roi_size == (8, 8) and inf.cval == -1 and inf.sw_batch_size == 2


def test_sliding_window_splitter_matches_reference_fixture(golden_dir):
    """Patch grid, padding (constant / replicate / none), negative offsets, int and float overlaps and filter_fn of
    SlidingWindowSplitter vs the real reference (tests/golden/make_golden.py patch); splitting is indexing, so CPU tensors work."""
    import os

    import numpy as np
    import pytest
    import torch

    sys.path.insert(0, golden_dir)
    from make_golden_cases import PATCH_CASES  # noqa: F401  (kept in a tiny module so the tests do not import the reference)

    from monai_b200.inferers import SlidingWindowSplitter

    g = np.load(os.path.join(golden_dir, "patch.npz"))
    for name, (shape, kw) in PATCH_CASES.items():
        x = torch.from_numpy(g[f"{name}.x"])
        assert tuple(x.shape) == shape
        s = SlidingWindowSplitter(**kw)
        pl = list(s(x))
        np.testing.assert_array_equal(np.array([l for _, l in pl], dtype=np.int64), g[f"{name}.loc"], err_msg=name)
        np.testing.assert_array_equal(torch.stack([p for p, _ in pl]).numpy(), g[f"{name}.patches"], err_msg=name)
        assert tuple(s.get_padded_shape(x)) == tuple(g[f"{name}.padded_shape"]), name
    x = torch.from_numpy(g["p2d.x"])
    s = SlidingWindowSplitter(filter_fn=lambda patch, loc: loc[0] >= 1 and float(patch.mean()) > 0.4, **PATCH_CASES["p2d"][1])
    np.testing.assert_array_equal(np.array([l for _, l in s(x)], dtype=np.int64), g["p2d.filtered_loc"])
    # argument validation of the reference
    with pytest.raises(ValueError, match="Relative overlap must be between"):
        SlidingWindowSplitter(4, overlap=1.0)
    with pytest.raises(ValueError, match="cannot be negative"):
        SlidingWindowSplitter(4, overlap=-1)
    with pytest.raises(ValueError, match="requires a valid padding mode"):
        SlidingWindowSplitter(4, offset=-1, pad_mode=None)
    with pytest.raises(ValueError, match="at least two parameters"):
        SlidingWindowSplitter(4, filter_fn=lambda p: True)
    with pytest.raises(ValueError, match="cannot be larger than patch size"):
        list(SlidingWindowSplitter(4, overlap=5)(torch.zeros(1, 1, 8, 8)))
    with pytest.raises(ValueError, match="cannot be larger than inputs size"):
        list(SlidingWindowSplitter(4, offset=9)(torch.zeros(1, 1, 8, 8)))


def test_patch_inferer_argument_errors():
    import pytest
    import torch

    from monai_b200.inferers import AvgMerger, PatchInferer, SlidingWindowSplitter

    with pytest.raises(TypeError, match="'splitter' should be a `Splitter`"):
        PatchInferer(splitter=lambda x: x)
    with pytest.raises(ValueError, match="does not exist"):
        PatchInferer(merger_cls="NoSuchMerger")
    with pytest.raises(TypeError, match="subclass of `Merger`"):
        PatchInferer(merger_cls=dict)
    with pytest.raises(ValueError, match="positive number"):
        PatchInferer(batch_size=0)
    with pytest.raises(TypeError, match="'preprocessing' should be a callable"):
        PatchInferer(preprocessing=3)
    with pytest.raises(ValueError, match="`splitter` should be set"):
        PatchInferer()(torch.zeros(1, 1, 4, 4), lambda p: p)
    assert PatchInferer(merger_cls="AvgMerger").merger_cls is AvgMerger
    with pytest.raises(RuntimeError, match="CUDA device"):
        AvgMerger(merged_shape=(1, 1, 4, 4), device="cpu")
    assert isinstance(PatchInferer(splitter=SlidingWindowSplitter(4)).splitter, SlidingWindowSplitter)


def test_buffered_window_order_matches_the_reference(golden_dir):
    """buffer_steps / buffer_dim: the order and batching in which the predictor sees the windows is the reference's
    (monai/inferers/utils.py:324-348), checked against coordinates recorded from the real reference (with_coord=True)."""
    import itertools

    import numpy as np

    from monai_b200.data.utils import dense_patch_starts
    from monai_b200.inferers.utils import _create_buffered_order, _get_scan_interval

    g = np.load(os.path.join(golden_dir, "buffered.npz"))
    for ci in range(int(g["n"])):
        x, cfg = g[f"c{ci}.x"], g[f"c{ci}.cfg"]
        nd = x.ndim - 2
        roi, swb, steps, dim = tuple(int(v) for v in cfg[:nd]), int(cfg[nd]), int(cfg[nd + 1]), int(cfg[nd + 2])
        dim = dim + nd if dim < 0 else dim
        image = tuple(max(i, r) for i, r in zip(x.shape[2:], roi))
        interval = _get_scan_interval(image, roi, nd, (float(g[f"c{ci}.ov"]),) * nd)
        starts = dense_patch_starts(image, roi, interval)
        flat = list(itertools.product(*starts))
        order, groups = _create_buffered_order(starts, roi, x.shape[0], swb, dim, steps)
        coords, sizes = [], []
        for first, last in groups:
            b = first // len(flat)
            for g0 in range(first, last, swb):
                ids = [int(order[pos - b * len(flat)]) for pos in range(g0, min(g0 + swb, last))]
                sizes.append(len(ids))
                coords.extend([b, *flat[i]] for i in ids)
        np.testing.assert_array_equal(np.asarray(sizes), g[f"c{ci}.batch_sizes"], err_msg=f"case {ci}")
        np.testing.assert_array_equal(np.asarray(coords), g[f"c{ci}.coords"], err_msg=f"case {ci}")
