"""The fp16 tensor-core forward of SegResNet and its kernels (b200_group_stats, the epilogue add of b200_conv3x3x3_tc,
b200_upsample_add_nc8), against torch and against fixtures of the real reference (tests/golden/segresnet_tc.npz, configurations in
tc_cases.py)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from monai_b200 import _kernels as K
from monai_b200 import _lib as L
from monai_b200.inferers import sliding_window_inference
from monai_b200.networks.nets import SegResNet
from tc_cases import TC_CASES, load_input
from weights import fill_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
TC_KERNELS = {"gemm_tc", "conv3x3x3_tc", "conv3x3x3_tc_affine", "conv3x3x3_tc_affine_add", "conv_cin1_tc", "conv_gather_tc", "norm_act_nc8",
              "norm_act_affine_nc8", "head_conv_norm_nc8", "head_conv_norm_affine_nc8", "group_stats", "upsample_add_nc8"}
GENERIC_ONLY = {"conv3d_direct", "norm_act", "resample_affine", "instnorm_stats"}


def _build(kw, seed):
    net = SegResNet(**kw)
    net.load_state_dict(fill_state_dict(net.state_dict(), seed))
    return net.eval().to(DEV)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(1e-6, np.abs(b).max()))


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _stats(t):
    """{sum, sumsq} per (n, c) of an fp32 [N, C, ...] tensor, as the kernels' statistics."""
    f = t.flatten(2).double()
    return torch.stack([f.sum(-1), (f * f).sum(-1)], -1).reshape(-1, 2).float().contiguous()


def _check_stats(got, ref_t):
    """Kernel statistics against float64 sums of the fp32 reference: the kernels add fp32 values in another order."""
    f = ref_t.flatten(2).double()
    ref = torch.stack([f.sum(-1), (f * f).sum(-1)], -1).reshape(-1, 2)
    scale = torch.stack([f.abs().sum(-1), (f * f).sum(-1)], -1).reshape(-1, 2)
    err = float(((got.double() - ref).abs() / (scale + 1e-6)).max())
    assert err <= 2e-3, err


# ---------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("groups", [48, 24, 16, 12, 6])   # 1, 2, 3, 4 and 8 channels per group; 3 straddles the 8-channel chunks
def test_group_stats_vs_torch(groups):
    N, C, sp, eps = 2, 48, (5, 6, 7), 1e-5
    x = (torch.randn(N, C, *sp, generator=_gen(groups)) * 2 + torch.arange(C).reshape(1, C, 1, 1, 1) * 0.1).half().to(DEV)
    st = _stats(x.float())
    cpg = C // groups
    out = torch.empty_like(st)
    K._call("group_stats", L.ptr(st), N, C, groups, L.ptr(out), L.stream_ptr(torch.device(DEV)))
    want = st.double().reshape(N, groups, cpg, 2).sum(2, keepdim=True).expand(N, groups, cpg, 2).reshape(-1, 2) / cpg
    assert torch.allclose(out.double(), want, rtol=1e-6, atol=1e-6)
    if cpg == 1:
        assert torch.equal(out, st)
    # fed the folded statistics, the NC8 normalisation is torch's GroupNorm
    gamma = (torch.rand(C, generator=_gen(1)) + 0.5).to(DEV)
    beta = (torch.randn(C, generator=_gen(2)) * 0.3).to(DEV)
    y = K.norm_act_nc8(K.pack_nc8(x), C, K.group_stats(st, N, C, groups), act=L.ACT_RELU, eps=eps, gamma=gamma, beta=beta)
    ref = F.relu(F.group_norm(x.float(), groups, gamma, beta, eps))
    err = float((K.unpack_nc8(y, dtype=torch.float32) - ref).abs().max())
    assert err <= 2.0**-10 * float(ref.abs().max()) + 1e-3, err


def _add_case(Cin, Cout, N, D, groups, add_ctot, add_coff, act, slope, seed):
    sp = (D, 20, 24)
    raw = K.pack_nc8((torch.randn(N, Cin, *sp, generator=_gen(seed)) * 2 + 0.3).half().to(DEV))
    addt = (torch.randn(N, add_ctot, *sp, generator=_gen(seed + 1))).half().to(DEV)
    add = K.pack_nc8(addt)
    st = K.group_stats(_stats(K.unpack_nc8(raw, dtype=torch.float32)), N, Cin, groups)
    g = (torch.rand(Cin, generator=_gen(seed + 2)) + 0.5).to(DEV)
    b = (torch.randn(Cin, generator=_gen(seed + 3)) * 0.3).to(DEV)
    wt = (torch.randn(Cout, Cin, 3, 3, 3, generator=_gen(seed + 4)) / (27 * Cin) ** 0.5).to(DEV)
    w = K.conv3x3x3_tc_pack_weight(wt)
    kw = dict(want_stats=True, in_norm=(st, 1e-5, act, slope), in_affine=(g, b))
    y, yst = K.conv3x3x3_tc(raw, w, Cin, Cout, add=(add, add_coff), **kw)
    # reference: the unfused normalised operand (bit-identical to the fused one) through an fp32 convolution, plus the slice
    normed = K.norm_act_nc8(raw, Cin, st, act=act, slope=slope, gamma=g, beta=b)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        ref = F.conv3d(K.unpack_nc8(normed, dtype=torch.float32), wt.half().float(), padding=1) + addt[:, add_coff:add_coff + Cout].float()
    return raw, w, add, kw, y, yst, ref


@pytest.mark.parametrize("Cout,N,D", [(16, 1, 16), (32, 1, 8), (48, 1, 4), (64, 1, 6), (80, 1, 2), (96, 1, 3), (112, 1, 2), (128, 1, 5),
                                      (16, 2, 1), (64, 3, 24)])
def test_conv_tc_affine_add_vs_torch(Cout, N, D):
    """Every N tile width 16-128 at depths that select BD = 4 (D % 4 == 0 or D >= 16), 2 and 1; the batch-3 launch has more tiles
    than SMs.  Output at the fp16 storage tolerance, statistics of the fp32 sum, bit-identical reruns."""
    Cin = 32
    raw, w, add, kw, y, yst, ref = _add_case(Cin, Cout, N, D, 8, Cout, 0, L.ACT_RELU, 0.0, Cout + D)
    got = K.unpack_nc8(y, dtype=torch.float32)
    err = float((got - ref).abs().max())
    assert err <= 2.0**-10 * float(ref.abs().max()) + 1e-3, err
    _check_stats(yst, ref)
    y2, yst2 = K.conv3x3x3_tc(raw, w, Cin, Cout, add=(add, 0), **kw)
    assert torch.equal(y2.buf, y.buf) and torch.equal(yst2, yst)


def test_conv_tc_workspace_query_sizes_the_epilogue_add():
    """At 128 channels the add runs BD = 1 tiles where the plain kernel runs BD = 2: on a small volume (fewer tiles than SMs) its
    statistics need more partial rows, which the workspace query sizes from the descriptor's add."""
    d = L.ConvTcDesc(N=1, Cin=32, Cout=128, D=5, H=20, W=24, in_ctot=32, out_ctot=128, in_stats=16, in_eps=1e-5, in_act=L.ACT_RELU,
                     add_ctot=128)   # in_stats, add: any non-NULL 16-byte-aligned value
    lib = L.load()
    plain = lib.b200_conv3x3x3_tc_workspace_bytes(C.byref(d))
    d.add = 16
    with_add = lib.b200_conv3x3x3_tc_workspace_bytes(C.byref(d))
    assert with_add > plain > 0, (plain, with_add)
    d.in_stats = None
    assert lib.b200_conv3x3x3_tc_workspace_bytes(C.byref(d)) == -1   # the add needs the operand normalisation


def test_conv_tc_affine_add_channel_slice():
    """The added tensor is channels [16, 48) of a 64-channel buffer; LeakyReLU on the load, groups of 3 channels."""
    raw, w, add, kw, y, yst, ref = _add_case(48, 32, 2, 8, 16, 64, 16, L.ACT_LEAKY, 0.1, 7)
    err = float((K.unpack_nc8(y, dtype=torch.float32) - ref).abs().max())
    assert err <= 2.0**-10 * float(ref.abs().max()) + 1e-3, err
    _check_stats(yst, ref)
    with pytest.raises(ValueError):
        K.conv3x3x3_tc(raw, w, 48, 32, add=(add, 40), **kw)   # slice beyond the buffer


@pytest.mark.parametrize("scale,sp", [(2, (3, 5, 1)), (2, (1, 4, 7)), (2, (8, 6, 10)), (1, (5, 7, 9))])
def test_upsample_add_nc8_vs_torch(scale, sp):
    N = 2
    x = torch.randn(N, 40, *sp, generator=_gen(sum(sp))).half().to(DEV)
    osp = tuple(scale * s for s in sp)
    skip = torch.randn(N, 24, *osp, generator=_gen(sum(sp) + 1)).half().to(DEV)
    xs, ss = x[:, 8:24].float(), skip[:, 8:24].float()   # channel slices of x, skip and the output
    out = K.NC8(N, 32, osp, DEV)
    out.buf.zero_()
    y, st = K.upsample_add_nc8(K.pack_nc8(x), 16, scale, K.pack_nc8(skip), x_coff=8, skip_coff=8, out=out, out_coff=16, want_stats=True)
    up = F.interpolate(xs, scale_factor=2, mode="trilinear", align_corners=False) if scale == 2 else xs
    ref = up + ss
    got = K.unpack_nc8(y, dtype=torch.float32)
    assert torch.count_nonzero(got[:, :16]) == 0
    err = float((got[:, 16:] - ref).abs().max())
    assert err <= 2.0**-10 * float(ref.abs().max()) + 1e-4, err
    _check_stats(st, ref)
    y2, st2 = K.upsample_add_nc8(K.pack_nc8(x), 16, scale, K.pack_nc8(skip), x_coff=8, skip_coff=8, want_stats=True)
    assert torch.equal(y2.buf, y.buf[:, 2:]) and torch.equal(st2, st)


# ---------------------------------------------------------------------------------------------------- network
@pytest.mark.parametrize("tag", ["A", "B", "C"])
def test_segresnet_tc_matches_reference_fixture(golden_dir, tag):
    kw, shape, seed = TC_CASES["segresnet"][tag][:3]
    g = np.load(os.path.join(golden_dir, "segresnet_tc.npz"))
    net = _build(kw, seed)
    assert net._tc_ok
    x = load_input("segresnet", tag, g).to(DEV)
    y = net(x)
    assert y.dtype == torch.float16 and tuple(y.shape) == (shape[0], kw["out_channels"], *shape[2:])
    y = y.float().cpu().numpy()
    s = int(g[f"{tag}.y_stride"])
    sub, ref = y[..., ::s, ::s, ::s], g[f"{tag}.y_sub"]
    err = _rel(sub, ref)
    assert err <= 3e-2, f"rel err {err}"   # the project's fp16 bar (DESIGN.md §2)
    agree = float((sub.argmax(1) == ref.argmax(1)).mean())
    assert agree >= 0.98, agree
    ysum = float(g[f"{tag}.y_sum"])
    assert abs(float(y.astype(np.float64).sum()) - ysum) <= 3e-2 * np.abs(ref).max() * y.size   # the whole output, not only the subsample


@pytest.mark.parametrize("tag", ["A", "B", "C"])
def test_segresnet_dispatch_is_measured(tag):
    kw, _, seed = TC_CASES["segresnet"][tag][:3]
    net = _build(kw, seed)
    x = load_input("segresnet", tag)[:1].to(DEV)
    K.profile_start()
    net(x)
    fp16 = K.profile_stop()
    want = {"conv3x3x3_tc_affine_add", "upsample_add_nc8", "gemm_tc"}
    want |= {"conv_gather_tc"} if len(kw.get("blocks_down", (1, 2, 2, 4))) > 1 else set()
    want |= {"group_stats"} if tag != "C" else set()
    assert want <= set(fp16), sorted(fp16)
    assert not (GENERIC_ONLY & set(fp16)), sorted(fp16)
    ran = {k for k in fp16 if not k.endswith("_pack_weight")}   # the first call also packs the weights
    assert ran <= TC_KERNELS | {"pack_nc8", "unpack_nc8", "copy_channels"}, sorted(fp16)
    K.profile_start()
    y32 = net(x.float())
    fp32 = K.profile_stop()
    assert y32.dtype == torch.float32
    assert not (TC_KERNELS & set(fp32)), sorted(fp32)
    assert "conv3d_direct" in fp32


@pytest.mark.parametrize("kw", [dict(), dict(init_filters=16, norm="batch")], ids=["init8", "batchnorm"])
def test_segresnet_ineligible_configs_take_the_generic_path(kw):
    net = _build(kw, 70).half()
    assert not net._tc_ok
    x = torch.randn((1, 1, 16, 16, 16), generator=_gen(71)).half().to(DEV)
    K.profile_start()
    y = net(x)
    prof = K.profile_stop()
    assert not (TC_KERNELS & set(prof)) and "conv3d_direct" in prof, sorted(prof)
    assert torch.equal(y, net._forward_generic(x))


def test_segresnet_tc_deterministic_graphed_and_follows_new_weights():
    kw, _, seed = TC_CASES["segresnet"]["A"][:3]
    net = _build(kw, seed)
    x = load_input("segresnet", "A").to(DEV)
    y1 = net(x)        # captures the graph
    y2 = net(x)        # replays it
    assert torch.equal(y1, y2)
    assert torch.equal(net._forward_tc(x), y1)
    net.load_state_dict(fill_state_dict(net.state_dict(), seed + 100))
    y3 = net(x)
    assert not torch.equal(y3, y1)
    fresh = _build(kw, seed + 100)
    assert torch.equal(y3, fresh._forward_tc(x))


def test_segresnet_tc_wide_head_graphed_equals_eager():
    kw, _, seed = TC_CASES["segresnet"]["B"][:3]
    net = _build(kw, seed)
    x = load_input("segresnet", "B").to(DEV)
    y1, y2 = net(x), net(x)
    assert y1.is_contiguous() and torch.equal(y1, y2)
    assert torch.equal(net._forward_tc(x), y1)


def test_segresnet_tc_rejects_bad_shapes():
    kw, _, seed = TC_CASES["segresnet"]["A"][:3]
    net = _build(kw, seed)
    with pytest.raises(ValueError, match="divisible by 8"):
        net(torch.zeros(1, 4, 32, 32, 20, device=DEV, dtype=torch.float16))
    with pytest.raises(ValueError, match="input"):
        net(torch.zeros(1, 2, 32, 32, 32, device=DEV, dtype=torch.float16))


def test_segresnet_tc_sliding_window_vs_generic_fp32():
    kw, _, seed = TC_CASES["segresnet"]["A"][:3]
    net = _build(kw, seed)
    vol = torch.randn(1, 4, 96, 80, 64, generator=_gen(95)).half()
    # 4 windows of 64^3 at overlap 0.5: one batch of 3 and a remainder batch of 1
    got = sliding_window_inference(vol.to(DEV), (64, 64, 64), 3, net, 0.5, "gaussian")
    ref = sliding_window_inference(vol.float().to(DEV), (64, 64, 64), 3, net, 0.5, "gaussian")
    assert got.shape == ref.shape
    g, r = got.float().cpu().numpy(), ref.cpu().numpy()
    err = _rel(g, r)
    assert err <= 3e-2, f"rel err {err}"
    agree = float((g.argmax(1) == r.argmax(1)).mean())
    assert agree >= 0.98, agree
