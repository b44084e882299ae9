"""GPU parity: monai_b200.sliding_window_inference (CUDA gather + blend kernels through the C ABI) vs the reference
fixtures and the numpy oracle.  fp32 blend is bit-exact by construction (same op order); asserted at 1e-6."""
import os

import numpy as np
import pytest
import torch

from monai_b200.inferers import SlidingWindowInferer, sliding_window_inference
from oracle import sliding_window as osw
from test_oracle_golden import SIGMA_CONSTANT, SIGMA_GAUSSIAN, SigmaPred

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _cheap_predictor(x):
    ramp = torch.arange(x.shape[-1], dtype=x.dtype, device=x.device) * 0.01
    return torch.cat([x.mean(dim=1, keepdim=True) * 1.5 + ramp, torch.tanh(x[:, :1]) - 0.25], dim=1)


def test_matches_reference_fixtures(golden_dir):
    g = np.load(os.path.join(golden_dir, "sliding_window.npz"))
    for name in g["names"]:
        ov = g[f"{name}.overlap"].tolist()
        ov = ov[0] if len(ov) == 1 else tuple(ov)
        x = torch.from_numpy(g[f"{name}.x"]).to(DEV)
        y = sliding_window_inference(
            x, tuple(int(v) for v in g[f"{name}.roi"]), int(g[f"{name}.bs"]), _cheap_predictor, ov, str(g[f"{name}.mode"]),
            0.125, str(g[f"{name}.pad"]), float(g[f"{name}.cval"]),
        )
        assert y.device.type == "cuda" and y.dtype == torch.float32
        np.testing.assert_allclose(y.cpu().numpy(), g[f"{name}.y"], rtol=1e-5, atol=1e-5, err_msg=f"case {name}")


def test_multi_resolution_dict_outputs(golden_dir):
    g = np.load(os.path.join(golden_dir, "sliding_window.npz"))

    def multi(x):
        return {"1": x + 1.0, "2": torch.nn.functional.avg_pool3d(x, 2) * 2.0, "3": x[..., ::4, ::4, ::4] - 3.0}

    r = sliding_window_inference(torch.from_numpy(g["multi.x"]).to(DEV), (16, 16, 16), 3, multi, 0.5, "gaussian")
    assert sorted(r.keys()) == ["1", "2", "3"]
    for k in ("1", "2", "3"):
        np.testing.assert_allclose(r[k].cpu().numpy(), g[f"multi.y{k}"], rtol=1e-5, atol=1e-5)


def test_sigma_and_cval_goldens_of_the_reference_unit_tests():
    x = torch.ones((1, 1, 7, 7), device=DEV)

    def pred():
        p = SigmaPred()
        return lambda d: p(d)

    r = sliding_window_inference(x, (3, 3), 10, pred(), overlap=0.5, padding_mode="constant", cval=-1, mode="constant", sigma_scale=1.0)
    np.testing.assert_allclose(r.cpu().numpy(), SIGMA_CONSTANT, rtol=1e-4)
    r = sliding_window_inference(x, (3, 3), 10, pred(), overlap=0.5, padding_mode="constant", cval=-1, mode="gaussian", sigma_scale=1.0)
    np.testing.assert_allclose(r.cpu().numpy(), SIGMA_GAUSSIAN, rtol=1e-4)
    for kw in (dict(sigma_scale=1.0), dict(sigma_scale=[1.0, 1.0]), dict(sigma_scale=[1.0, 1.0], cache_roi_weight_map=True)):
        r = SlidingWindowInferer((3, 3), 10, overlap=0.5, mode="gaussian", **kw)(x, pred())
        np.testing.assert_allclose(r.cpu().numpy(), SIGMA_GAUSSIAN, rtol=1e-4)
    # test_cval
    x = torch.ones((1, 1, 3, 3), device=DEV)
    r = sliding_window_inference(x, (5, 5), 10, lambda d: d + d.sum(), overlap=0.5, padding_mode="constant", cval=-1, mode="constant", sigma_scale=1.0)
    np.testing.assert_allclose(r.cpu().numpy(), np.ones((1, 1, 3, 3)) * -6.0, rtol=1e-4)
    r = SlidingWindowInferer((5, 5), 10, overlap=0.5, mode="constant", cval=-1)(x, lambda d: d + d.sum())
    np.testing.assert_allclose(r.cpu().numpy(), np.ones((1, 1, 3, 3)) * -6.0, rtol=1e-4)


TEST_CASES = [
    [(2, 3, 16), (4,), 3, 0.25, "constant"], [(2, 3, 16, 15, 7, 9), 4, 3, 0.25, "constant"], [(1, 3, 16, 15, 7), (4, -1, 7), 3, 0.25, "constant"],
    [(2, 3, 16, 15, 7), (4, -1, 7), 3, 0.25, "constant"], [(3, 3, 16, 15, 7), (4, -1, 7), 3, 0.25, "constant"],
    [(2, 3, 16, 15, 7), (4, -1, 7), 3, 0.25, "constant"], [(1, 3, 16, 15, 7), (4, 10, 7), 3, 0.25, "constant"],
    [(1, 3, 16, 15, 7), (20, 22, 23), 10, 0.25, "constant"], [(2, 3, 15, 7), (2, 6), 1000, 0.25, "constant"],
    [(1, 3, 16, 7), (80, 50), 7, 0.25, "constant"], [(1, 3, 16, 15, 7), (20, 22, 23), 10, 0.5, "constant"],
    [(1, 3, 16, 15, 7), (20, 22, 23), 10, 0.5, "gaussian"], [(1, 3, 16, 15, 7), (4, 10, 7), 3, 0.25, "gaussian"],
    [(3, 3, 16, 15, 7), (4, -1, 7), 3, 0.25, "gaussian"], [(1, 3, 16, 15, 7), (4, 10, 7), 3, 0.25, "gaussian"],
    [(1, 3, 16, 15, 7), (4, 10, 7), 1, 0.25, "gaussian"], [(1, 3, 16, 15, 7), (4, 10, 7), 1, (0.25, 0.5, 0.75), "gaussian"],
]


@pytest.mark.parametrize("shape,roi,bs,ov,mode", TEST_CASES)
def test_sliding_window_default_cases(shape, roi, bs, ov, mode):
    """The shape / roi / overlap / mode matrix of tests/inferers/test_sliding_window_inference.py:28-46,98-121
    (compute = x + 1 on an arange ramp, so the expected result is exact)."""
    n = int(np.prod(shape))
    x = torch.arange(n, dtype=torch.float, device=DEV).reshape(shape)
    if len(shape) - 2 > 3:
        with pytest.raises(NotImplementedError):
            sliding_window_inference(x, roi, bs, lambda d: d + 1, overlap=ov, mode=mode)
        return
    r = sliding_window_inference(x, roi, bs, lambda d: d + 1, overlap=ov, mode=mode)
    np.testing.assert_allclose(r.cpu().numpy(), (x + 1).cpu().numpy(), rtol=1e-6)
    r = SlidingWindowInferer(roi, bs, overlap=ov, mode=mode)(x, lambda d: d + 1)
    np.testing.assert_allclose(r.cpu().numpy(), (x + 1).cpu().numpy(), rtol=1e-6)


def test_matches_oracle_on_fresh_random_inputs_fp32_and_fp16():
    rng = np.random.default_rng(5)
    x = rng.standard_normal((2, 2, 50, 37, 45)).astype(np.float32)
    want = osw.sliding_window_inference(x, (24, 16, 20), 5, lambda a: _cheap_predictor(torch.from_numpy(a)).numpy(), 0.5, "gaussian")
    got = sliding_window_inference(torch.from_numpy(x).to(DEV), (24, 16, 20), 5, _cheap_predictor, 0.5, "gaussian")
    np.testing.assert_allclose(got.cpu().numpy(), want, rtol=1e-5, atol=1e-6)
    # fp16 volume: fp32 accumulation inside the kernel, compare with the fp32 oracle at fp16 resolution
    got16 = sliding_window_inference(torch.from_numpy(x).to(DEV).half(), (24, 16, 20), 5, _cheap_predictor, 0.5, "gaussian")
    assert got16.dtype == torch.float16
    np.testing.assert_allclose(got16.float().cpu().numpy(), want, rtol=4e-3, atol=4e-3)


def test_streaming_path_equals_one_shot(monkeypatch):
    """Force the resident-prediction budget down so the accumulate (mode 1) + finalize (mode 2) path runs."""
    import monai_b200.inferers.utils as U

    x = torch.randn(1, 1, 40, 40, 40, device=DEV)
    a = sliding_window_inference(x, (16, 16, 16), 4, _cheap_predictor, 0.5, "gaussian")
    monkeypatch.setattr(U, "_RESIDENT_BYTES", 6 * 2 * 16**3 * 4)
    b = sliding_window_inference(x, (16, 16, 16), 4, _cheap_predictor, 0.5, "gaussian")
    torch.testing.assert_close(a, b, rtol=0, atol=0)  # same fp32 op order -> identical


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_eight_voxel_blend_path_is_bit_identical_to_the_scalar_path(monkeypatch, dtype):
    """W, roi and all W starts are multiples of 8 -> the 8-voxels-per-thread kernel runs; forcing the alignment hint
    to 1 sends the same data through the scalar kernel.  Same op order, so one-shot and streaming results are identical."""
    import monai_b200.inferers.utils as U

    x = torch.randn(2, 1, 40, 48, 64, device=DEV).to(dtype)
    roi = (16, 24, 32)
    a = sliding_window_inference(x, roi, 4, _cheap_predictor, 0.5, "gaussian")
    with monkeypatch.context() as m:
        m.setattr(U, "_RESIDENT_BYTES", 7 * 2 * 16 * 24 * 32 * x.element_size())
        a_stream = sliding_window_inference(x, roi, 4, _cheap_predictor, 0.5, "gaussian")
    orig = U.K.sw_blend

    def scalar(mode, preds, wb, we, vol_shape, roi_, starts, *rest, **kw):
        assert starts[2]._align == 8
        starts[2]._align = 1
        return orig(mode, preds, wb, we, vol_shape, roi_, starts, *rest, **kw)

    monkeypatch.setattr(U.K, "sw_blend", scalar)
    b = sliding_window_inference(x, roi, 4, _cheap_predictor, 0.5, "gaussian")
    torch.testing.assert_close(a, b, rtol=0, atol=0)
    torch.testing.assert_close(a_stream, b, rtol=0, atol=0)
    want = osw.sliding_window_inference(x.float().cpu().numpy(), roi, 4, lambda v: _cheap_predictor(torch.from_numpy(v)).numpy(), 0.5, "gaussian")
    tol = 1e-5 if dtype == torch.float32 else 4e-3
    np.testing.assert_allclose(a.float().cpu().numpy(), want, rtol=tol, atol=tol)


@pytest.mark.parametrize("spatial_dim", [0, 1, 2])
def test_slice_inferer_equals_per_slice_prediction(spatial_dim):
    """A 2-D predictor slid over a 3-D volume (reference tests/inferers/test_slice_inferer.py): with the roi covering whole
    slices every voxel is predicted exactly once, so the stitched volume equals the per-slice predictions; tensor, tuple
    and dict outputs; the inferer can be called repeatedly."""
    from monai_b200.inferers import SliceInferer

    def pred2d(t):   # [N, C, A, B] -> 2 channels
        assert t.dim() == 4
        ramp = torch.arange(t.shape[-1], dtype=t.dtype, device=t.device) * 0.01
        return torch.cat([t * 2.0 + ramp, torch.tanh(t) - 0.5], dim=1)

    x = torch.randn(2, 1, 6, 16, 24, device=DEV)
    roi = list(x.shape[2:])
    roi.pop(spatial_dim)
    want = torch.stack([pred2d(s) for s in x.unbind(dim=spatial_dim + 2)], dim=spatial_dim + 2)
    inf = SliceInferer(roi_size=roi, spatial_dim=spatial_dim, sw_batch_size=3, cval=-1)
    for _ in range(2):
        got = inf(x, pred2d)
        assert got.shape == (2, 2, 6, 16, 24)
        torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-6)
    got_t = inf(x, lambda t: (pred2d(t), pred2d(t)[:, :1] + 1))
    torch.testing.assert_close(got_t[1], want[:, :1] + 1, rtol=1e-6, atol=1e-6)
    got_d = inf(x, lambda t: {"a": pred2d(t)})
    torch.testing.assert_close(got_d["a"], want, rtol=1e-6, atol=1e-6)


def test_patch_inferer_matches_reference_fixture(golden_dir):
    """PatchInferer(SlidingWindowSplitter, AvgMerger) vs the real reference (tests/golden/make_golden.py patch): tuple output
    with a half-resolution head (location scaled by the size ratio), batches of 3, cropping of the padded merge; dict output
    with selected keys, pre / post processing and `match_spatial_shape=False`; merger bookkeeping of AvgMerger."""
    from monai_b200.inferers import AvgMerger, PatchInferer, SlidingWindowSplitter

    def net(p):
        return p * 2.0 + 1.0, torch.nn.functional.avg_pool3d(p, 2) - 0.5

    g = np.load(os.path.join(golden_dir, "patch.npz"))
    x = torch.from_numpy(g["pi.x"]).to(DEV)
    inf = PatchInferer(splitter=SlidingWindowSplitter(patch_size=4, overlap=0.5, pad_mode="constant"), merger_cls=AvgMerger, batch_size=3)
    a, b = inf(x, net)
    assert a.dtype == torch.float32 and tuple(a.shape) == g["pi.same"].shape and tuple(b.shape) == g["pi.half"].shape
    np.testing.assert_allclose(a.cpu().numpy(), g["pi.same"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(b.cpu().numpy(), g["pi.half"], rtol=1e-6, atol=1e-6)
    inf = PatchInferer(splitter=SlidingWindowSplitter(patch_size=(4, 5, 4), overlap=(2, 0, 1), pad_mode="constant", pad_value=0.25),
                       batch_size=2, preprocessing=lambda p: p + 1.0, postprocessing=lambda o: {"a": o[0], "b": o[1], "c": o[0] * 0},
                       output_keys=["b", "a"], match_spatial_shape=False)
    d = inf(x, net)
    assert list(d.keys()) == ["b", "a"]
    np.testing.assert_allclose(d["b"].cpu().numpy(), g["pi.dict_b"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(d["a"].cpu().numpy(), g["pi.dict_a"], rtol=1e-6, atol=1e-6)
    # AvgMerger on its own: counts, fp16 patches, finalisation guard, never-covered elements are NaN as in the reference
    m = AvgMerger(merged_shape=(1, 2, 6, 6), device=DEV)
    p = torch.ones((1, 2, 4, 4), device=DEV).half()
    m.aggregate(p, (0, 0))
    m.aggregate(p * 3, (2, 2))
    assert m.get_counts().dtype == torch.uint8 and int(m.get_counts()[0, 0, 2, 2]) == 2 and int(m.get_counts()[0, 1, 5, 0]) == 0
    out = m.finalize()
    assert float(out[0, 0, 0, 0]) == 1.0 and float(out[0, 1, 3, 3]) == 2.0 and float(out[0, 0, 5, 5]) == 3.0 and bool(torch.isnan(out[0, 0, 5, 0]))
    assert m.finalize() is out
    with pytest.raises(ValueError, match="already finalized"):
        m.aggregate(p, (0, 0))
    with pytest.raises(ValueError, match="leaves the merged volume"):
        AvgMerger(merged_shape=(1, 2, 6, 6), device=DEV).aggregate(p, (3, 3))


def test_fp16_predictions_one_shot_equals_streaming(monkeypatch):
    """fp16 predictions: the one-shot blend (all windows resident) and the streaming accumulate + finalize path give the same
    bits."""
    import monai_b200.inferers.utils as U

    x = torch.randn(2, 1, 40, 72, 128, generator=torch.Generator().manual_seed(7)).half().to(DEV)
    a = sliding_window_inference(x, (16, 24, 64), 4, _cheap_predictor, 0.5, "gaussian")
    monkeypatch.setattr(U, "_RESIDENT_BYTES", 9 * 2 * 16 * 24 * 64 * 2)
    b = sliding_window_inference(x, (16, 24, 64), 4, _cheap_predictor, 0.5, "gaussian")
    np.testing.assert_array_equal(a.float().cpu().numpy(), b.float().cpu().numpy())


def test_args_kwargs_process_fn_with_coord_and_device():
    x = torch.rand((1, 1, 12, 12, 12), device=DEV)
    t1, t2 = torch.ones(1, device=DEV), torch.ones(1, device=DEV)

    def compute(data, test1, test2):
        return data + test1 + test2

    r = sliding_window_inference(x, (4, 4, 4), 10, compute, 0.5, "constant", 0.125, "constant", 0.0, DEV, DEV, False, None, None, None, 0, False, t1, test2=t2)
    np.testing.assert_allclose(r.cpu().numpy(), (x + 2).cpu().numpy(), rtol=1e-6)

    seen = []

    def with_coord(data, coords):
        seen.append(coords)
        return data * 2

    r = sliding_window_inference(x, (8, 8, 8), 2, with_coord, 0.5, "gaussian", with_coord=True)
    np.testing.assert_allclose(r.cpu().numpy(), (x * 2).cpu().numpy(), rtol=1e-5)
    assert len(seen[0]) == 2 and len(seen[0][0]) == 5 and seen[0][0][2] == slice(0, 8)

    def process_fn(seg_tuple, win, imp):
        return tuple(s * 3 for s in seg_tuple), imp

    r = sliding_window_inference(x, (8, 8, 8), 2, lambda d: d + 1, 0.5, "gaussian", process_fn=process_fn)
    np.testing.assert_allclose(r.cpu().numpy(), ((x + 1) * 3).cpu().numpy(), rtol=1e-5)

    r = sliding_window_inference(x, (8, 8, 8), 2, lambda d: d + 1, 0.25, device="cpu")
    assert r.device.type == "cpu"
    np.testing.assert_allclose(r.numpy(), (x + 1).cpu().numpy(), rtol=1e-6)
