"""The fp16 tensor-core forward of UNet with residual units (InstanceNorm or eval-mode BatchNorm) and the post-activation residual
add of b200_norm_act_nc8 (res_mode 1), against float64, the generic CUDA-core forward and fixtures of the real reference
(tests/golden/unet_res_tc.npz, configurations in unet_res_cases.py)."""
import os

import numpy as np
import pytest
import torch

from monai_b200 import _kernels as K
from monai_b200 import _lib as L
from monai_b200.inferers import sliding_window_inference
from monai_b200.networks.nets import UNet
from unet_res_cases import FIXTURE, RES_CASES, load_input
from weights import fill_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
TAGS = ["A", "B", "C"]


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(1e-6, np.abs(b).max()))


def _build(kw, seed):
    net = UNet(**kw)
    net.load_state_dict(fill_state_dict(net.state_dict(), seed))
    return net.eval().to(DEV)


def _bar(y, ref):
    """The project's fp16 bar: 3e-2 of the output scale and 98 % arg-max agreement."""
    err = _rel(y, ref)
    assert err <= 3e-2, f"rel err {err}"
    agree = float((y.argmax(1) == ref.argmax(1)).mean())
    assert agree >= 0.98, agree


# ------------------------------------------------------------------------------------------- norm_act_nc8, res_mode 1
SENT = 7.25   # fp16 sentinel of the output allocation


def _slice_nc8(x, ctot, coff, fill):
    """x [N, C, *sp] fp16 as channels [coff, coff + C) of an NC8 buffer with ctot channels whose other channels hold `fill`."""
    N, C_ = x.shape[:2]
    full = torch.full((N, ctot, *x.shape[2:]), fill, dtype=torch.float16)
    full[:, coff:coff + C_] = x
    return K.pack_nc8(full.to(DEV))


ACTS = [(L.ACT_NONE, 0.0), (L.ACT_RELU, 0.0), (L.ACT_LEAKY, 0.01), (L.ACT_LEAKY, 0.25), (L.ACT_LEAKY, -0.2), (L.ACT_LEAKY, 1.5)]


@pytest.mark.parametrize("act,slope", ACTS, ids=[f"act{a}_{s}" for a, s in ACTS])
@pytest.mark.parametrize("norm", ["stats", "stats_affine", "none"])
def test_norm_act_nc8_post_add_vs_float64(norm, act, slope):
    N, C_, sp, eps = 2, 16, (5, 6, 7), 1e-5
    S = sp[0] * sp[1] * sp[2]
    x = (torch.randn(N, C_, *sp, generator=_gen(1)) * 1.5 + torch.linspace(-1, 1, C_).reshape(1, C_, 1, 1, 1)).half()
    r = torch.randn(N, C_, *sp, generator=_gen(2)).half()
    f = x.double().flatten(2)
    st = torch.stack([f.sum(-1), (f * f).sum(-1)], -1).reshape(-1, 2).float().contiguous()
    g = (torch.rand(C_, generator=_gen(3)) + 0.5) if norm == "stats_affine" else None
    b = (torch.randn(C_, generator=_gen(4)) * 0.3) if norm == "stats_affine" else None
    # float64 reference from the same statistics
    v = x.double()
    if norm != "none":
        mean = (st[:, 0].double() / S).reshape(N, C_, 1, 1, 1)
        var = (st[:, 1].double() / S).reshape(N, C_, 1, 1, 1) - mean * mean
        v = (v - mean) / torch.sqrt(var + eps)
        if g is not None:
            v = v * g.double().reshape(1, C_, 1, 1, 1) + b.double().reshape(1, C_, 1, 1, 1)
    if act == L.ACT_LEAKY:
        v = torch.where(v >= 0, v, v * slope)
    elif act == L.ACT_RELU:
        v = v.clamp_min(0)
    ref = v + r.double()
    # x, res and y are channel slices of wider buffers; x's and res's neighbours are NaN, y's allocation holds a sentinel
    xb = _slice_nc8(x, 32, 8, float("nan"))
    rb = _slice_nc8(r, 48, 24, float("nan"))
    out = K.NC8(N, 40, sp, DEV)
    out.buf.fill_(SENT)
    kw = dict(x_coff=8, res=rb, res_coff=24, act=act, slope=slope, out=out, out_coff=16, eps=eps, res_after_act=True)
    stats = st.to(DEV) if norm != "none" else None
    gb = dict(gamma=g.to(DEV), beta=b.to(DEV)) if g is not None else {}
    K.norm_act_nc8(xb, C_, stats, **kw, **gb)
    y = K.unpack_nc8(out, dtype=torch.float32).cpu()
    got = y[:, 16:32].double()
    bound = 2.0**-10 * ref.abs() + 1e-3
    assert bool(((got - ref).abs() <= bound).all()), float(((got - ref).abs() / bound).max())
    assert bool((y[:, :16] == SENT).all()) and bool((y[:, 32:] == SENT).all()), "channels outside the output slice changed"
    first = out.buf.clone()
    K.norm_act_nc8(xb, C_, stats, **kw, **gb)
    assert torch.equal(out.buf, first), "reruns differ"


def test_norm_act_nc8_post_add_rejects_normalised_residual():
    N, C_, sp = 1, 16, (4, 4, 4)
    x = K.pack_nc8(torch.randn(N, C_, *sp, generator=_gen(5)).half().to(DEV))
    st = torch.ones(N * C_, 2, device=DEV)
    g = torch.ones(C_, device=DEV)
    with pytest.raises(ValueError, match="res_mode 1"):
        K.norm_act_nc8(x, C_, st, res=x, res_stats=st, res_after_act=True)
    with pytest.raises(ValueError, match="res_mode 1"):
        K.norm_act_nc8(x, C_, st, res=x, res_stats=st, res_gamma=g, res_beta=g, res_after_act=True)
    with pytest.raises(ValueError):   # residual affine parameters need residual statistics in either mode
        K.norm_act_nc8(x, C_, st, res=x, res_gamma=g, res_after_act=True)
    out = K.NC8(N, C_, sp, DEV)
    rc = L.load().b200_norm_act_nc8(L.ptr(x.buf), C_, 0, N, C_, x.S, L.ptr(st), 1e-5, L.ptr(x.buf), C_, 0, None, 0, 0.0, L.ptr(out.buf),
                                    C_, 0, None, None, None, None, 2, L.stream_ptr(x.buf.device))
    assert rc != 0, "res_mode 2 must be rejected"


# ------------------------------------------------------------------------------------------------------------- network
@pytest.mark.parametrize("tag", TAGS)
def test_unet_res_tc_matches_reference_fixture(golden_dir, tag):
    kw, shape, seed = RES_CASES[tag][:3]
    g = np.load(os.path.join(golden_dir, FIXTURE))
    net = _build(kw, seed)
    x = load_input(tag, g).to(DEV)
    assert net._use_tc(x)
    y = net(x)
    assert y.dtype == torch.float16 and y.is_contiguous() and tuple(y.shape) == (shape[0], kw["out_channels"], *shape[2:])
    y = y.float().cpu().numpy()
    s = int(g[f"{tag}.y_stride"])
    sub, ref = y[..., ::s, ::s, ::s], g[f"{tag}.y_sub"]
    _bar(sub, ref)
    ysum = float(g[f"{tag}.y_sum"])
    assert abs(float(y.astype(np.float64).sum()) - ysum) <= 3e-2 * np.abs(ref).max() * y.size   # the whole output
    # the same net on the generic CUDA-core forward
    _bar(y, net._forward_generic(x.float()).cpu().numpy())


@pytest.mark.parametrize("tag", TAGS)
def test_unet_res_tc_dispatch_is_measured(tag):
    kw, _, seed = RES_CASES[tag][:3]
    net = _build(kw, seed)
    x = load_input(tag)[:1].to(DEV)
    net(x)   # packs the weights
    K.profile_start()
    net(x)
    prof = K.profile_stop()
    assert {"conv3x3x3_tc", "conv_gather_tc", "norm_act_nc8" if tag != "C" else "norm_act_affine_nc8"} <= set(prof), sorted(prof)
    assert "conv_cin1_nc8" in prof if kw["in_channels"] == 1 else "pack_nc8" in prof
    assert not ({"conv3d_direct", "norm_act", "instnorm_stats"} & set(prof)), sorted(prof)
    assert set(prof) <= {"conv3x3x3_tc", "conv3x3x3_tc_affine", "conv3x3x3_tc_affine_add", "conv_gather_tc", "conv_cin1_nc8", "conv_cin1_tc",
                         "gemm_tc", "norm_act_nc8", "norm_act_affine_nc8", "pack_nc8", "unpack_nc8", "copy_channels"}, sorted(prof)
    if tag == "C":
        assert "gemm_tc" in prof   # the 1x1x1 residual of a stride-1 level


@pytest.mark.parametrize("w", [-0.2, 1.5])
def test_unet_res_tc_prelu_slope_outside_unit_interval_materialises(w):
    kw, _, seed = RES_CASES["B"][:3]
    net = _build(kw, seed)
    x = load_input("B").to(DEV)
    net(x)
    K.profile_start()
    net(x)
    n_fused = K.profile_stop()["norm_act_nc8"]["n"]
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, torch.nn.PReLU):
                m.weight.fill_(w)
    K.profile_start()
    y = net(x)
    n_mat = K.profile_stop()["norm_act_nc8"]["n"]
    assert n_mat > n_fused, (n_mat, n_fused)   # act(norm(y)) materialised where the operand load would have applied it
    _bar(y.float().cpu().numpy(), net._forward_generic(x.float()).cpu().numpy())


def test_unet_res_tc_follows_batchnorm_running_statistics():
    kw, _, seed = RES_CASES["A"][:3]
    net = _build(kw, seed)
    x = load_input("A")[:1].to(DEV)
    y1 = net(x)
    assert torch.equal(net(x), y1)
    sd = net.state_dict()
    new = {k: (v * 1.3 + 0.05 if k.endswith(("running_mean", "running_var")) else v) for k, v in sd.items()}
    net.load_state_dict(new)   # only buffers change
    y2 = net(x)
    assert not torch.equal(y2, y1)
    fresh = UNet(**kw)
    fresh.load_state_dict({k: v.cpu() for k, v in new.items()})
    fresh = fresh.eval().to(DEV)
    assert torch.equal(y2, fresh(x))
    _bar(y2.float().cpu().numpy(), net._forward_generic(x.float()).cpu().numpy())


@pytest.mark.parametrize("tag", ["A", "C"])
def test_unet_res_tc_graph_replay_equals_eager(tag):
    kw, _, seed = RES_CASES[tag][:3]
    net = _build(kw, seed)
    assert net._graph_enabled
    x = load_input(tag).to(DEV)
    y1 = net(x)        # captures the graph
    y2 = net(x)        # replays it
    assert len(net._graphs) == 1 and y1.is_contiguous()
    assert torch.equal(y1, y2)
    assert torch.equal(net._forward_tc(x), y1)
    x2 = x.flip(-1).contiguous()   # same shape, new values: the replay reads the new input
    assert torch.equal(net(x2), net._forward_tc(x2))


def test_unet_plain_tc_stays_eager():
    net = _build(dict(spatial_dims=3, in_channels=1, out_channels=2, channels=(16, 32, 64), strides=(2, 2)), 3)
    assert not net._graph_enabled


def test_unet_res_tc_rejects_non_divisible_input_before_any_launch():
    kw, _, seed = RES_CASES["A"][:3]
    net = _build(kw, seed)
    n0 = L.launch_count()
    with pytest.raises(ValueError, match="divisible by 16"):
        net(torch.zeros(1, 1, 64, 64, 40, device=DEV, dtype=torch.float16))
    with pytest.raises(ValueError, match="input"):
        net(torch.zeros(1, 2, 64, 64, 64, device=DEV, dtype=torch.float16))
    assert L.launch_count() == n0


def test_unet_res_tc_sliding_window_fp16():
    kw, _, seed = RES_CASES["B"][:3]
    net = _build(kw, seed)
    vol = torch.randn(1, 4, 80, 64, 48, generator=_gen(95)).half()
    # 3 x 1 x 1 windows of 48 x 64 x 48 at overlap 0.5 in batches of 2: one full batch and a remainder batch of 1
    got = sliding_window_inference(vol.to(DEV), (48, 64, 48), 2, net, 0.5, "gaussian")
    ref = sliding_window_inference(vol.float().to(DEV), (48, 64, 48), 2, net, 0.5, "gaussian")
    assert got.dtype == torch.float16 and got.shape == ref.shape
    _bar(got.float().cpu().numpy(), ref.cpu().numpy())
