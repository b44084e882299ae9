"""The fp16 tensor-core forward of BasicUNet and its 2x max pool on NC8 buffers (b200_maxpool2_nc8), against torch, the generic
CUDA-core forward and fixtures of the real reference (tests/golden/basic_unet_tc.npz, configurations in basic_unet_cases.py)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from monai_b200 import _kernels as K
from monai_b200 import _lib as L
from monai_b200.inferers import sliding_window_inference
from monai_b200.networks.nets import BasicUNet
from basic_unet_cases import BASIC_CASES, FIXTURE, load_input
from weights import fill_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
CASES = BASIC_CASES
TAGS = ["A", "B", "C"]
TC_KERNELS = {"conv3x3x3_tc", "conv3x3x3_tc_affine", "conv_cin1_tc", "conv_cin1_nc8", "gemm_tc", "norm_act_nc8", "norm_act_affine_nc8",
              "head_conv_norm_nc8", "head_conv_norm_affine_nc8", "maxpool2_nc8", "pack_nc8", "unpack_nc8", "copy_channels"}
GENERIC_ONLY = {"conv3d_direct", "maxpool3d_2", "norm_act", "instnorm_stats"}


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(1e-6, np.abs(b).max()))


def _build(kw, seed):
    net = BasicUNet(**kw)
    net.load_state_dict(fill_state_dict(net.state_dict(), seed))
    return net.eval().to(DEV)


def _bar(y, ref):
    """The project's fp16 bar: 3e-2 of the output scale and 98 % arg-max agreement."""
    err = _rel(y, ref)
    assert err <= 3e-2, f"rel err {err}"
    agree = float((y.argmax(1) == ref.argmax(1)).mean())
    assert agree >= 0.98, agree


# ------------------------------------------------------------------------------------------------------- maxpool2_nc8
SENT = 7.25   # fp16 sentinel of the output allocation


def _slice_nc8(x, ctot, coff, fill):
    """x [N, C, *sp] fp16 as channels [coff, coff + C) of an NC8 buffer with ctot channels whose other channels hold `fill`."""
    N, C_ = x.shape[:2]
    full = torch.full((N, ctot, *x.shape[2:]), fill, dtype=torch.float16)
    full[:, coff:coff + C_] = x
    return K.pack_nc8(full.to(DEV))


@pytest.mark.parametrize("sp", [(4, 6, 8), (5, 7, 9), (2, 2, 2), (3, 3, 67)], ids=["even", "odd", "one_cell", "odd_long"])
@pytest.mark.parametrize("sl", [(16, 16, 0, 16, 0), (16, 32, 8, 40, 16), (8, 48, 40, 24, 8)], ids=["whole", "slices", "last_chunk"])
def test_maxpool2_nc8_equals_torch(sp, sl):
    C_, x_ctot, x_coff, y_ctot, y_coff = sl
    N = 2
    x = (torch.randn(N, C_, *sp, generator=_gen(sum(sp) + C_)) * 3).half()
    # x's neighbouring channels are NaN (a read outside the slice would show); the output allocation holds a sentinel
    xb = _slice_nc8(x, x_ctot, x_coff, float("nan"))
    osp = tuple(s // 2 for s in sp)
    out = K.NC8(N, y_ctot, osp, DEV)
    out.buf.fill_(SENT)
    K.maxpool2_nc8(xb, C_, x_coff=x_coff, out=out, out_coff=y_coff)
    y = K.unpack_nc8(out).cpu()
    ref = F.max_pool3d(x.to(DEV), 2).cpu()
    assert torch.equal(y[:, y_coff:y_coff + C_], ref)
    outside = torch.cat([y[:, :y_coff], y[:, y_coff + C_:]], 1)
    assert bool((outside == SENT).all()), "channels outside the output slice changed"


def test_maxpool2_nc8_propagates_nan():
    x = torch.randn(1, 16, 6, 6, 6, generator=_gen(7)).half()
    x[0, 3, 1, 2, 3] = float("nan")   # in the cell of output voxel (0, 1, 1)
    x[0, 9, 5, 5, 5] = float("nan")   # in the cell of output voxel (2, 2, 2)
    y = K.unpack_nc8(K.maxpool2_nc8(K.pack_nc8(x.to(DEV)), 16)).cpu()
    ref = F.max_pool3d(x.to(DEV), 2).cpu()
    assert bool(ref[0, 3, 0, 1, 1].isnan()) and bool(ref[0, 9, 2, 2, 2].isnan())
    assert torch.equal(y.isnan(), ref.isnan()) and int(y.isnan().sum()) == 2
    assert torch.equal(y.nan_to_num(), ref.nan_to_num())


def test_maxpool2_nc8_rejects_misaligned_slice():
    xb = K.NC8(1, 32, (4, 4, 4), DEV)
    n0 = L.launch_count()
    with pytest.raises(ValueError, match="maxpool2_nc8"):
        K.maxpool2_nc8(xb, 16, x_coff=4)
    assert L.launch_count() == n0


# ------------------------------------------------------------------------------------------------------------- network
@pytest.mark.parametrize("tag", TAGS)
def test_basic_unet_tc_matches_reference_fixture(golden_dir, tag):
    kw, shape, seed = CASES[tag][:3]
    g = np.load(os.path.join(golden_dir, FIXTURE))
    net = _build(kw, seed)
    x = load_input(tag, g).to(DEV)
    assert net._use_tc(x)
    y = net(x)
    assert y.dtype == torch.float16 and y.is_contiguous() and tuple(y.shape) == (shape[0], kw.get("out_channels", 2), *shape[2:])
    y = y.float().cpu().numpy()
    s = int(g[f"{tag}.y_stride"])
    sub, ref = y[..., ::s, ::s, ::s], g[f"{tag}.y_sub"]
    _bar(sub, ref)
    ysum = float(g[f"{tag}.y_sum"])
    assert abs(float(y.astype(np.float64).sum()) - ysum) <= 3e-2 * np.abs(ref).max() * y.size   # the whole output
    # the same net on the generic CUDA-core forward
    _bar(y, net._forward_generic(x.float()).cpu().numpy())


@pytest.mark.parametrize("tag", TAGS)
def test_basic_unet_tc_dispatch_is_measured(tag):
    kw, _, seed = CASES[tag][:3]
    net = _build(kw, seed)
    x = load_input(tag)[:1].to(DEV)
    net(x)   # packs the weights
    K.profile_start()
    net(x)
    prof = K.profile_stop()
    names = set(prof)
    assert {"maxpool2_nc8", "gemm_tc"} <= names, sorted(names)
    assert any(n.startswith("conv3x3x3_tc") for n in names) and names & {"norm_act_nc8", "norm_act_affine_nc8"}, sorted(names)
    assert not (GENERIC_ONLY & names), sorted(names)
    assert names <= TC_KERNELS, sorted(names)
    assert prof["maxpool2_nc8"]["n"] == 4 and prof["maxpool2_nc8"]["bytes"] > 0
    assert prof["gemm_tc"]["n"] == (5 if kw.get("out_channels", 2) > 16 else 4)   # the transposed convolutions (+ the wide head)


@pytest.mark.parametrize("tag", ["A", "C"])
def test_basic_unet_tc_graph_replay_equals_eager(tag):
    kw, _, seed = CASES[tag][:3]
    net = _build(kw, seed)
    x = load_input(tag).to(DEV)
    y1 = net(x)        # captures the graph (or runs eager when replay is off for this net)
    y2 = net(x)
    assert y1.is_contiguous() and torch.equal(y1, y2)
    assert torch.equal(net._forward_tc(x), y1)
    x2 = x.flip(-1).contiguous()   # same shape, new values: a replay reads the new input
    assert torch.equal(net(x2), net._forward_tc(x2))
    if net._graph_enabled:
        assert len(net._graphs) == 1


def test_basic_unet_fp16_of_other_sizes_takes_the_generic_path():
    kw, _, seed = CASES["A"][:3]
    net = _build(kw, seed)
    x = torch.randn(1, 1, 40, 48, 48, generator=_gen(3)).half().to(DEV)
    assert not net._use_tc(x)
    K.profile_start()
    y = net(x)
    prof = K.profile_stop()
    assert {"conv3d_direct", "maxpool3d_2"} <= set(prof) and "maxpool2_nc8" not in prof, sorted(prof)
    assert y.dtype == torch.float16 and tuple(y.shape) == (1, 2, 40, 48, 48) and bool(y.isfinite().all())


def test_basic_unet_tc_active_dropout_takes_the_generic_path():
    kw, _, seed = CASES["C"][:3]
    net = _build(kw, seed).train()
    x = load_input("C").to(DEV)
    assert not net._use_tc(x)
    with pytest.raises(RuntimeError, match="eval mode"):
        net(x)


def test_basic_unet_tc_rejects_bad_input_before_any_launch():
    kw, _, seed = CASES["A"][:3]
    net = _build(kw, seed)
    n0 = L.launch_count()
    with pytest.raises(ValueError, match="input"):
        net(torch.zeros(1, 2, 32, 32, 32, device=DEV, dtype=torch.float16))
    with pytest.raises(ValueError, match="input"):
        net(torch.zeros(1, 32, 32, 32, device=DEV, dtype=torch.float16))
    assert L.launch_count() == n0


def test_basic_unet_tc_sliding_window_fp16():
    kw, _, seed = CASES["B"][:3]
    net = _build(kw, seed)
    vol = torch.randn(1, 4, 80, 64, 48, generator=_gen(96)).half()
    # 3 x 1 x 1 windows of 48 x 64 x 48 at overlap 0.5 in batches of 2: one full batch and a remainder batch of 1
    got = sliding_window_inference(vol.to(DEV), (48, 64, 48), 2, net, 0.5, "gaussian")
    ref = sliding_window_inference(vol.float().to(DEV), (48, 64, 48), 2, net, 0.5, "gaussian")
    assert got.dtype == torch.float16 and got.shape == ref.shape
    _bar(got.float().cpu().numpy(), ref.cpu().numpy())
