"""SegResNetDS on the GPU: the given operand normalisation of the 3x3x3 / one-plane tensor-core convolutions (`in_scale_shift`, an
eval-mode BatchNorm) and the epilogue add of b200_conv3x3_tc, against float64 references and the zero-padded 3x3x3 kernel; the
network's generic fp32 path against fixtures of the real reference (segresnet_ds.npz) and its fp16 tensor-core forward against
segresnet_ds_tc.npz (configurations in segresnet_ds_cases.py)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from monai_b200 import _kernels as K
from monai_b200 import _lib as L
from monai_b200.inferers import sliding_window_inference
from monai_b200.networks.nets import SegResNetDS
from segresnet_ds_cases import FIXTURE, FP32_CASES, TC_CASES, TC_FIXTURE, load_input
from weights import fill_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
TAGS = ["A", "B", "C", "D"]
GENERIC_ONLY = {"conv3d_direct", "norm_act", "instnorm_stats", "resample_affine"}
SENT = 7.25   # fp16 sentinel of output allocations


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(1e-6, np.abs(b).max()))


def _build(kw, seed):
    net = SegResNetDS(**kw)
    net.load_state_dict(fill_state_dict(net.state_dict(), seed))
    return net.eval().to(DEV)


def _bar(y, ref):
    """The project's fp16 bar: 3e-2 of the output scale and 98 % arg-max agreement."""
    err = _rel(y, ref)
    assert err <= 3e-2, f"rel err {err}"
    agree = float((y.argmax(1) == ref.argmax(1)).mean())
    assert agree >= 0.98, agree


def _slice_nc8(x, ctot, coff, fill):
    """x [N, C, *sp] fp16 as channels [coff, coff + C) of an NC8 buffer with ctot channels whose other channels hold `fill`."""
    N, C_ = x.shape[:2]
    full = torch.full((N, ctot, *x.shape[2:]), fill, dtype=torch.float16)
    full[:, coff:coff + C_] = x
    return K.pack_nc8(full.to(DEV))


def _kernel_shape(axis):
    return tuple(1 if a == axis else 3 for a in range(3))


def _conv(x, w, axis, add, **kw):
    """conv3x3x3_tc (axis -1) or conv3x3_tc (axis 0..2) of NC8 x with the Conv3d weight w."""
    if axis < 0:
        return K.conv3x3x3_tc(x, K.conv3x3x3_tc_pack_weight(w), w.shape[1], w.shape[0], add=add, **kw)
    return K.conv3x3_tc(x, K.conv3x3_tc_pack_weight(w, axis), w.shape[1], w.shape[0], axis, add=add, **kw)


# ------------------------------------------------------------------------------------------ in_scale_shift and the add
@pytest.mark.parametrize("axis", [-1, 0, 1, 2], ids=["333", "d1", "h1", "w1"])
@pytest.mark.parametrize("add", [False, True], ids=["plain", "add"])
@pytest.mark.parametrize("cout,sp", [(32, (5, 9, 20)), (64, (8, 16, 8)), (128, (3, 17, 9))])
def test_in_scale_shift_matches_float64(axis, add, cout, sp):
    """act(x * s + t) on the operand load from a given table, with and without the epilogue add, on channel slices of two batch
    items, against float64 on the same fp16 operands; channels outside the output slice keep the sentinel; reruns give the same bits."""
    N, cin, x_ctot, x_coff, y_ctot, y_coff = 2, 32, 64, 16, cout + 16, 8
    g = _gen(cout + sum(sp) + axis)
    x = (torch.randn(N, cin, *sp, generator=g) * 2).half()
    w = torch.randn(cout, cin, *_kernel_shape(axis), generator=g) / (cin * 9) ** 0.5
    tab = torch.stack((torch.rand(cin, generator=g) + 0.5, torch.randn(cin, generator=g) * 0.5), 1).contiguous()
    slope = 0.1
    r = (torch.randn(N, cout, *sp, generator=g)).half()
    xb = _slice_nc8(x, x_ctot, x_coff, float("nan"))
    ab = (_slice_nc8(r, cout + 24, 24, float("nan")), 24) if add else None
    outs = []
    for _ in range(2):
        out = K.NC8(N, y_ctot, sp, DEV)
        out.buf.fill_(SENT)
        _, st = _conv(xb, w.to(DEV), axis, ab, in_coff=x_coff, out=out, out_coff=y_coff, want_stats=True,
                      in_scale_shift=(tab.to(DEV), L.ACT_LEAKY, slope))
        outs.append((K.unpack_nc8(out).cpu(), st.cpu()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), "reruns differ"
    y, st = outs[0]
    # the operand the tensor cores see: act(x * s + t) in fp32, rounded once to fp16
    a = x.float() * tab[:, 0].view(1, -1, 1, 1, 1) + tab[:, 1].view(1, -1, 1, 1, 1)
    a = torch.where(a >= 0, a, a * slope).half().double()
    pad = tuple(k // 2 for k in _kernel_shape(axis))
    ref = F.conv3d(a, w.half().double(), padding=pad)
    if add:
        ref = ref + r.double()
    got = y[:, y_coff:y_coff + cout].double()
    err = (got - ref).abs().max().item()
    assert err <= 2e-3 * ref.abs().max().item() + 1e-3, err
    outside = torch.cat([y[:, :y_coff], y[:, y_coff + cout:]], 1)
    assert bool((outside == SENT).all()), "channels outside the output slice changed"
    s_ref = torch.stack((ref.sum((2, 3, 4)), (ref * ref).sum((2, 3, 4))), -1).reshape(-1, 2)
    assert torch.allclose(st.double(), s_ref, rtol=2e-3, atol=2e-3 * float(s_ref.abs().max())), "statistics"


def test_in_scale_shift_equals_the_statistics_form_on_the_same_table():
    """A table equal to the one InstanceNorm statistics give yields the same bits as the statistics form: the transform is shared."""
    N, C_, sp = 2, 32, (6, 10, 12)
    x = torch.randn(N, C_, *sp, generator=_gen(5)).half().to(DEV)
    w = (torch.randn(C_, C_, 3, 3, 3, generator=_gen(6)) / 16).to(DEV)
    xb = K.pack_nc8(x)
    st = K.instnorm_stats(x)
    y_st, _ = _conv(xb, w, -1, None, in_norm=(st, 1e-5, L.ACT_RELU, 0.0))
    # batch item 0's (scale, shift) as a given table, applied to both items: item 0 must match the statistics form
    s0 = st.view(N, C_, 2)[0].double()
    S = float(np.prod(sp))
    mean = s0[:, 0] / S
    var = (s0[:, 1] / S - mean * mean).clamp_min(0)
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    tab = torch.stack((rstd, -mean * rstd), 1).float().contiguous()
    y_tab, _ = _conv(xb, w, -1, None, in_scale_shift=(tab, L.ACT_RELU, 0.0))
    a, b = K.unpack_nc8(y_st)[0].float(), K.unpack_nc8(y_tab)[0].float()
    assert float((a - b).abs().max()) <= 2e-3 * float(a.abs().max())


def _desc(x, cout, **kw):
    d = L.ConvTcDesc(N=x.N, Cin=32, Cout=cout, D=x.sp[0], H=x.sp[1], W=x.sp[2], in_ctot=x.C, in_coff=0, out_ctot=cout, out_coff=0)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_in_scale_shift_descriptor_errors():
    """The C ABI rejects a given table (in_table = 1) without in_stats or together with in_gamma / in_beta, a misaligned table, an
    in_table other than 0 / 1, a bad activation and the folded residual; the workspace query rejects the same descriptors (-1), and
    nothing is launched."""
    x = K.NC8(1, 32, (4, 8, 8), DEV)
    y = K.NC8(1, 32, (4, 8, 8), DEV)
    w3, w33 = K.conv3x3x3_tc_pack_weight(torch.zeros(32, 32, 3, 3, 3, device=DEV)), K.conv3x3_tc_pack_weight(torch.zeros(32, 32, 1, 3, 3, device=DEV), 0)
    tab = torch.zeros(64, device=DEV)
    st = torch.zeros(64, device=DEV)
    lib = L.load()
    bad = {
        "without in_stats": dict(in_table=1),
        "with in_gamma": dict(in_table=1, in_stats=L.ptr(tab), in_gamma=L.ptr(st)),
        "with in_beta": dict(in_table=1, in_stats=L.ptr(tab), in_beta=L.ptr(st)),
        "misaligned": dict(in_table=1, in_stats=L.ptr(tab) + 4),
        "in_table 2": dict(in_table=2, in_stats=L.ptr(tab)),
        "prelu": dict(in_table=1, in_stats=L.ptr(tab), in_act=2),
        "slope": dict(in_table=1, in_stats=L.ptr(tab), in_act=1, in_slope=1.5),
        "with res_w": dict(in_table=1, in_stats=L.ptr(tab), res_w=L.ptr(w3), res_y=L.ptr(y.buf), res_ctot=32),
    }
    torch.cuda.synchronize()
    n0 = L.launch_count()
    for name, kw in bad.items():
        d = _desc(x, 32, **kw)
        assert lib.b200_conv3x3x3_tc_workspace_bytes(C.byref(d)) == -1, name
        assert lib.b200_conv3x3x3_tc(C.byref(d), L.ptr(x.buf), L.ptr(w3), None, L.ptr(y.buf), None, None, L.stream_ptr(x.buf.device)) != 0, name
        assert "in_table" in lib.b200_last_error().decode() or name in ("prelu", "slope", "with res_w"), (name, lib.b200_last_error())
        if name != "with res_w":
            assert lib.b200_conv3x3_tc_workspace_bytes(C.byref(d), 0) == -1, name
    # the add without any operand normalisation is rejected for both kernels
    d = _desc(x, 32, add=L.ptr(y.buf), add_ctot=32)
    assert lib.b200_conv3x3x3_tc_workspace_bytes(C.byref(d)) == -1 and lib.b200_conv3x3_tc_workspace_bytes(C.byref(d), 1) == -1
    assert lib.b200_conv3x3_tc(C.byref(d), 1, L.ptr(x.buf), L.ptr(w33), None, L.ptr(y.buf), None, None, L.stream_ptr(x.buf.device)) != 0
    # a valid descriptor passes both queries
    d = _desc(x, 32, in_table=1, in_stats=L.ptr(tab), add=L.ptr(y.buf), add_ctot=32)
    assert lib.b200_conv3x3x3_tc_workspace_bytes(C.byref(d)) >= 0 and lib.b200_conv3x3_tc_workspace_bytes(C.byref(d), 2) >= 0
    assert L.launch_count() == n0
    with pytest.raises(ValueError, match="in_scale_shift excludes"):
        K.conv3x3_tc(x, w33, 32, 32, 0, in_norm=(st, 1e-5, 0, 0.0), in_scale_shift=(tab.view(32, 2), 0, 0.0))
    with pytest.raises(ValueError, match="add needs"):
        K.conv3x3_tc(x, w33, 32, 32, 0, add=(y, 0))
    assert L.launch_count() == n0


@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("cout,D", [(16, 8), (48, 5), (64, 16), (96, 2), (128, 3)])
@pytest.mark.parametrize("given", [False, True], ids=["stats", "table"])
def test_conv3x3_tc_add_equals_zero_padded_333(axis, cout, D, given):
    """conv3x3_tc with the epilogue add gives the bits (output and statistics) of conv3x3x3_tc with the add and the weight
    zero-padded to 3x3x3."""
    N, cin, sp = 2, 32, (D, 12, 20)
    g = _gen(cout * 7 + D + axis)
    x = torch.randn(N, cin, *sp, generator=g).half().to(DEV)
    w = (torch.randn(cout, cin, *_kernel_shape(axis), generator=g) / (cin * 9) ** 0.5).to(DEV)
    w333 = torch.zeros(cout, cin, 3, 3, 3, device=DEV)
    sl = [slice(None), slice(None)] + [slice(1, 2) if a == axis else slice(None) for a in range(3)]
    w333[tuple(sl)] = w
    xb = K.pack_nc8(x)
    r = K.pack_nc8(torch.randn(N, cout, *sp, generator=g).half().to(DEV))
    if given:
        tab = torch.stack((torch.rand(cin, generator=g) + 0.5, torch.randn(cin, generator=g)), 1).contiguous().to(DEV)
        kw = dict(in_scale_shift=(tab, L.ACT_RELU, 0.0))
    else:
        st = K.instnorm_stats(x)
        kw = dict(in_norm=(st, 1e-5, L.ACT_LEAKY, 0.01), in_affine=(torch.rand(cin, device=DEV) + 0.5, torch.randn(cin, device=DEV)))
    y1, s1 = _conv(xb, w, axis, (r, 0), want_stats=True, **kw)
    y3, s3 = _conv(xb, w333, -1, (r, 0), want_stats=True, **kw)
    assert torch.equal(y1.buf, y3.buf) and torch.equal(s1, s3)


def test_conv_gather_transposed_331_matches_float64():
    """The deconv of an anisotropic SegResNetDS level: ConvTranspose3d k (3,3,1), s (2,2,1), p (1,1,0), op (1,1,0) on conv_gather_tc."""
    N, cin, cout, sp = 2, 64, 32, (5, 6, 7)
    g = _gen(11)
    x = torch.randn(N, cin, *sp, generator=g).half()
    w = torch.randn(cin, cout, 3, 3, 1, generator=g) / (cin * 9 / 4) ** 0.5
    k, s, p, op = (3, 3, 1), (2, 2, 1), (1, 1, 0), (1, 1, 0)
    y, _ = K.conv_gather_tc(K.pack_nc8(x.to(DEV)), K.conv_gather_tc_pack_weight(w.to(DEV), k, s, p, True), cin, cout, k, s, p, transposed=True,
                            output_padding=op)
    ref = F.conv_transpose3d(x.double(), w.half().double(), None, s, p, op)
    got = K.unpack_nc8(y).cpu().double()
    assert got.shape == ref.shape == (N, cout, 10, 12, 7)
    assert float((got - ref).abs().max()) <= 2e-3 * float(ref.abs().max())


# ------------------------------------------------------------------------------------------------------------- network
@pytest.mark.parametrize("i", range(len(FP32_CASES)))
def test_segresnet_ds_generic_fp32_matches_reference(golden_dir, i):
    kw, shape, seed = FP32_CASES[i]
    g = np.load(os.path.join(golden_dir, FIXTURE))
    net = _build(kw, seed)
    x = torch.from_numpy(g[f"c{i}.x"]).to(DEV)
    assert not net._use_tc(x)
    y = net(x).cpu().numpy()
    assert y.shape == g[f"c{i}.y"].shape
    assert _rel(y, g[f"c{i}.y"]) <= 1e-3


@pytest.mark.parametrize("tag", TAGS)
def test_segresnet_ds_tc_matches_reference_fixture(golden_dir, tag):
    kw, shape, seed = TC_CASES[tag][:3]
    g = np.load(os.path.join(golden_dir, TC_FIXTURE))
    net = _build(kw, seed)
    x = load_input(tag, g).to(DEV)
    assert net._tc_ok and net._use_tc(x)
    y = net(x)
    assert y.dtype == torch.float16 and y.is_contiguous() and tuple(y.shape) == (shape[0], kw.get("out_channels", 2), *shape[2:])
    y = y.float().cpu().numpy()
    s = int(g[f"{tag}.y_stride"])
    sub, ref = y[..., ::s, ::s, ::s], g[f"{tag}.y_sub"]
    _bar(sub, ref)
    ysum = float(g[f"{tag}.y_sum"])
    assert abs(float(y.astype(np.float64).sum()) - ysum) <= 3e-2 * np.abs(ref).max() * y.size   # the whole output
    # the same net on the generic forward
    _bar(y, net._forward_generic(x.float()).cpu().numpy())


@pytest.mark.parametrize("tag", TAGS)
def test_segresnet_ds_tc_dispatch(tag):
    """Only tensor-core / NC8 kernels run; statistics exist only for instance norms, the BatchNorm nets read given tables."""
    kw, _, seed = TC_CASES[tag][:3]
    net = _build(kw, seed)
    x = load_input(tag)[:1].to(DEV)
    net(x)   # packs the weights
    K.profile_start()
    net(x)
    prof = K.profile_stop()
    names = set(prof)
    assert not (GENERIC_ONLY & names), sorted(names)
    allowed = {"conv_cin1_tc", "conv_cin1_nc8", "conv_gather_tc", "gemm_tc", "upsample_add_nc8", "group_stats", "head_conv_nc8",
               "pack_nc8", "unpack_nc8", "copy_channels"}
    assert all(n in allowed or n.startswith("conv3x3x3_tc") or n.startswith("conv3x3_tc") for n in names), sorted(names)
    convs = sum(v["n"] for n, v in prof.items() if n.startswith("conv3x3"))
    blocks = sum(kw.get("blocks_down", (1, 2, 2, 4))) + len(kw.get("blocks_down", (1, 2, 2, 4))) - 1
    stem = 0 if "conv_cin1_tc" in names or "conv_cin1_nc8" in names else 1
    assert convs == 2 * blocks + stem, (convs, blocks, sorted(names))
    if kw.get("resolution"):
        assert any(n.startswith("conv3x3_tc") for n in names), sorted(names)


@pytest.mark.parametrize("tag", ["A", "B"])
def test_segresnet_ds_tc_graph_replay_equals_eager(tag):
    kw, _, seed = TC_CASES[tag][:3]
    net = _build(kw, seed)
    x = load_input(tag).to(DEV)
    y1 = net(x)
    y2 = net(x)
    assert y1.is_contiguous() and torch.equal(y1, y2)
    assert torch.equal(net._forward_tc(x), y1)
    x2 = x.flip(-1).contiguous()   # same shape, new values: a replay reads the new input
    assert torch.equal(net(x2), net._forward_tc(x2))
    if net._graph_enabled:
        assert len(net._graphs) == 1


def test_segresnet_ds_tc_follows_load_state_dict():
    """New weights and new BatchNorm running statistics (nothing else) take effect, in eager and replayed forwards."""
    kw, _, seed = TC_CASES["C"][:3]
    net = _build(kw, seed)
    x = load_input("C").to(DEV)
    y0 = net(x)
    sd = net.state_dict()
    sd2 = {k: (v * 1.5 + 0.05 if k.endswith("running_var") else v.clone()) for k, v in sd.items()}
    net.load_state_dict(sd2)
    y1 = net(x)
    fresh = SegResNetDS(**kw)
    fresh.load_state_dict({k: v.cpu() for k, v in sd2.items()})
    fresh = fresh.eval().to(DEV)
    assert not torch.equal(y0, y1)
    assert torch.equal(y1, fresh._forward_tc(x))
    net.load_state_dict(fill_state_dict(net.state_dict(), seed + 1))
    ref = _build(kw, seed + 1)
    assert torch.equal(net(x), ref._forward_tc(x))


def test_segresnet_ds_tc_training_batchnorm_takes_the_generic_path():
    kw, _, seed = TC_CASES["A"][:3]
    net = _build(kw, seed).train()
    x = load_input("A")[:1].to(DEV)
    assert not net._use_tc(x)
    with pytest.raises(RuntimeError, match="eval"):
        net(x)


def test_segresnet_ds_tc_rejects_bad_input_before_any_launch():
    net = _build(TC_CASES["B"].kw, TC_CASES["B"].seed)
    torch.cuda.synchronize()
    n0 = L.launch_count()
    with pytest.raises(ValueError, match="must be divisible by"):
        net(torch.zeros(1, 4, 64, 64, 36, device=DEV, dtype=torch.float16))   # D, H need 16, W needs 8
    with pytest.raises(ValueError, match="expects an"):
        net(torch.zeros(1, 2, 64, 64, 32, device=DEV, dtype=torch.float16))
    with pytest.raises(ValueError, match="expects an"):
        net(torch.zeros(4, 64, 64, 32, device=DEV, dtype=torch.float16))
    assert L.launch_count() == n0


def test_segresnet_ds_tc_sliding_window_fp16():
    kw, _, seed = TC_CASES["C"][:3]
    net = _build(kw, seed)
    vol = torch.randn(1, 1, 20, 48, 40, generator=_gen(97)).half()
    # windows of 12 x 32 x 32 at overlap 0.5 in batches of 3
    got = sliding_window_inference(vol.to(DEV), (12, 32, 32), 3, net, 0.5, "gaussian")
    ref = sliding_window_inference(vol.float().to(DEV), (12, 32, 32), 3, net, 0.5, "gaussian")
    assert got.dtype == torch.float16 and got.shape == ref.shape
    _bar(got.float().cpu().numpy(), ref.cpu().numpy())
