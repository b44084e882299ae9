"""Anisotropic DynUNet plans on the tensor cores: the one-plane 3x3 convolution (b200_conv3x3_tc), the per-axis kernel / stride /
padding of b200_conv_gather_tc (ABI 4), and the network against fixtures of the real reference (tests/golden/dynunet_aniso_tc.npz,
configurations in dynunet_aniso_cases.py).

The kernel checks use the float64 references, bounds, guarded buffers and rerun checks of test_gpu_tc_gemm_sweep.py."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from monai_b200 import _kernels as K
from monai_b200 import _lib as L
from monai_b200.inferers import sliding_window_inference
from monai_b200.networks.nets import DynUNet
from dynunet_aniso_cases import ANISO_CASES, FIXTURE, load_input
from test_gpu_tc_gemm_sweep import MAX_K16_STEPS, assert_regime, check, check_stats, from_nc8, nc8_input, nc8_output, twice
from weights import fill_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
TC_KERNELS = {"gemm_tc", "conv3x3x3_tc", "conv3x3x3_tc_affine", "conv3x3_tc", "conv3x3_tc_affine", "conv_cin1_tc", "conv_gather_tc",
              "norm_act_nc8", "norm_act_affine_nc8", "head_conv_norm_nc8", "head_conv_norm_affine_nc8"}


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _kernel(axis):
    return tuple(1 if a == axis else 3 for a in range(3))


def _cdiv(a, b):
    return -(-a // b)


def conv_tc_tile(Cout, D):
    """conv_tc.cu conv_tc_nt / dispatch_bd, plain and operand-normalising forms: (NT, BD)."""
    nt = Cout if Cout <= 128 else (64 if Cout >= 384 and Cout % 64 == 0 else next(n for n in range(128, 15, -16) if Cout % n == 0))
    if 4 * nt <= 256 and (D % 4 == 0 or D >= 16):
        return nt, 4
    return (nt, 2) if D >= 2 and 2 * nt <= 256 else (nt, 1)


def conv_tc_tiles(N, Cout, sp):
    """(tiles per (batch item, N tile) group, total tiles): 16 x 8 patches of BD planes (conv_epi.cuh)."""
    nt, bd = conv_tc_tile(Cout, sp[0])
    tpg = _cdiv(sp[2], 8) * _cdiv(sp[1], 16) * _cdiv(sp[0], bd)
    return tpg, tpg * N * (Cout // nt)


def _stats(t):
    f = t.flatten(2).double()
    return torch.stack([f.sum(-1), (f * f).sum(-1)], -1).reshape(-1, 2).float().contiguous()


# ---------------------------------------------------------------------------------------------- conv3x3_tc vs float64
D_FOR_BD = {4: 8, 2: 3, 1: 1}
WIDTH_COUTS = (16, 32, 48, 64, 80, 96, 112, 128, 320)       # every N tile width; 320 runs on 80-wide tiles


def _c33_cases():
    out = []
    for axis in range(3):
        for cout in WIDTH_COUTS:
            for bd, D in D_FOR_BD.items():
                if conv_tc_tile(cout, D)[1] == bd:
                    out.append((axis, 2, 32, cout, (D, 19, 13), 8, 8, "i"))
        out.append((axis, 3, 16, 32, (16, 64, 64), 0, 8, "ii"))
        out.append((axis, 2, 16, 16, (16, 64, 96), 8, 0, "iii"))
    return out


def _c33_id(c):
    axis, N, cin, cout, sp = c[:5]
    return f"ax{axis}-N{N}-Cin{cin}-Cout{cout}-BD{conv_tc_tile(cout, sp[0])[1]}-{'x'.join(map(str, sp))}"


@pytest.mark.parametrize("case", _c33_cases(), ids=_c33_id)
def test_conv3x3_tc_vs_float64(case):
    """Plain and with the affine operand normalisation: every output element within the sweep's bound of a float64 conv3d on the
    fp16-rounded operands (for the fused form: the fp16 operand norm_act_nc8 stores), statistics within theirs, outputs confined
    to their channel slice, and both bit-identical on a rerun."""
    axis, N, Cin, Cout, sp, in_coff, out_coff, reg = case
    k = _kernel(axis)
    pad = tuple((i - 1) // 2 for i in k)
    assert Cin // 16 * 9 <= MAX_K16_STEPS
    assert_regime(reg, *conv_tc_tiles(N, Cout, sp))
    g = _gen(1000 + 7 * Cout + axis + sp[0])
    x = (torch.randn((N, Cin, *sp), generator=g) * 1.5 + 0.25).half()
    w = (torch.randn((Cout, Cin, *k), generator=g) / (9 * Cin) ** 0.5).half()
    b = torch.randn(Cout, generator=g)
    gam, bet = torch.randn(Cin, generator=g), torch.randn(Cin, generator=g) * 0.5
    _, xin = nc8_input(x, in_coff)
    pw = K.conv3x3_tc_pack_weight(w.float().to(DEV), axis)
    st = _stats(x.float()).to(DEV)
    in_norm, in_aff = (st, 1e-5, L.ACT_LEAKY, 0.01), (gam.to(DEV), bet.to(DEV))
    # the operand the fused form feeds the tensor core: norm_act_nc8's fp16 output (its bits are pinned by the test below)
    _, xc = nc8_input(x, 0, extra=0)
    normed = K.unpack_nc8(K.norm_act_nc8(xc, Cin, st, act=L.ACT_LEAKY, slope=0.01, eps=1e-5, gamma=gam.to(DEV), beta=bet.to(DEV))).cpu()
    for fused in (False, True):
        def launch():
            go, out = nc8_output(N, Cout, out_coff, sp)
            kw = dict(in_norm=in_norm, in_affine=in_aff) if fused else {}
            _, s = K.conv3x3_tc(xin, pw, Cin, Cout, axis, in_coff=in_coff, bias=b.to(DEV), out=out, out_coff=out_coff, want_stats=True, **kw)
            return go, s

        go, s, same_bits = twice(launch)
        xo = (normed if fused else x).double()
        r = F.conv3d(xo, w.double(), b.double(), padding=pad)
        A = F.conv3d(xo.abs(), w.double().abs(), b.double().abs(), padding=pad)
        what = f"conv3x3_tc axis {axis} {'fused' if fused else 'plain'} N={N} Cin={Cin} Cout={Cout} sp={sp}"
        go.assert_untouched_outside((slice(None), slice(out_coff // 8, (out_coff + Cout) // 8)), what)
        check("conv3x3_tc", what, from_nc8(go.view, out_coff, Cout).cpu(), r, A)
        check_stats("conv3x3_tc", what, s.cpu(), r.reshape(N, Cout, -1), A.reshape(N, Cout, -1))
        same_bits()


# ---------------------------------------------------------------------------------------------- conv3x3_tc bit for bit
@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("Cout,D", [(32, 16), (64, 6), (128, 3), (320, 1), (48, 5)])
def test_conv3x3_tc_equals_conv3x3x3_tc_with_zero_padded_weights(axis, Cout, D):
    """Same bits as the 3x3x3 kernel with the weight zero-padded to 3x3x3, plain and with the fused affine operand norm; and the
    fused operand norm equals norm_act_nc8 followed by a plain launch."""
    Cin, N, sp = 32, 2, (D, 40, 24)
    k = _kernel(axis)
    g = _gen(77 + axis + Cout + D)
    raw = K.pack_nc8((torch.randn((N, Cin, *sp), generator=g) * 2 + 0.3).half().to(DEV))
    w = (torch.randn((Cout, Cin, *k), generator=g) / (9 * Cin) ** 0.5).to(DEV)
    w27 = torch.zeros((Cout, Cin, 3, 3, 3), device=DEV)
    w27[:, :, slice(1, 2) if axis == 0 else slice(None), slice(1, 2) if axis == 1 else slice(None), slice(1, 2) if axis == 2 else slice(None)] = w
    bias = torch.randn(Cout, generator=g).to(DEV)
    p33, p27 = K.conv3x3_tc_pack_weight(w, axis), K.conv3x3x3_tc_pack_weight(w27)
    st = _stats(K.unpack_nc8(raw, dtype=torch.float32))
    gam, bet = (torch.randn(Cin, generator=g) * 1.5).to(DEV), (torch.randn(Cin, generator=g) * 0.5).to(DEV)
    norm = dict(in_norm=(st, 1e-4, L.ACT_LEAKY, 0.1), in_affine=(gam, bet))
    for kw in ({}, norm):
        y33, s33 = K.conv3x3_tc(raw, p33, Cin, Cout, axis, bias=bias, want_stats=True, **kw)
        y27, s27 = K.conv3x3x3_tc(raw, p27, Cin, Cout, bias=bias, want_stats=True, **kw)
        assert torch.equal(y33.buf, y27.buf), sorted(kw)
        assert torch.equal(s33, s27), sorted(kw)
    fused, fst = K.conv3x3_tc(raw, p33, Cin, Cout, axis, bias=bias, want_stats=True, **norm)
    normed = K.norm_act_nc8(raw, Cin, st, act=L.ACT_LEAKY, slope=0.1, eps=1e-4, gamma=gam, beta=bet)
    plain, pst = K.conv3x3_tc(normed, p33, Cin, Cout, axis, bias=bias, want_stats=True)
    assert torch.equal(fused.buf, plain.buf) and torch.equal(fst, pst)


def test_conv3x3_tc_rejects_the_3x3x3_only_forms():
    d = L.ConvTcDesc(N=1, Cin=16, Cout=16, D=4, H=8, W=8, in_ctot=16, in_coff=0, out_ctot=16, out_coff=0)
    assert L.load().b200_conv3x3_tc_workspace_bytes(d, 0) > 0
    d.res_w, d.res_y, d.res_ctot = 16, 16, 16
    assert L.load().b200_conv3x3_tc_workspace_bytes(d, 0) == -1
    d.res_w = d.res_y = None
    d.add, d.add_ctot = 16, 16
    assert L.load().b200_conv3x3_tc_workspace_bytes(d, 1) == -1
    d.add = None
    assert L.load().b200_conv3x3_tc_workspace_bytes(d, 3) == -1


# ---------------------------------------------------------------------------------------------- per-axis conv_gather_tc
# (k, stride, pad, transposed, N, Cin, Cout, input spatial, in_coff, out_coff)
CG_ANISO = [
    ((1, 3, 3), (1, 2, 2), (0, 1, 1), False, 2, 32, 64, (5, 14, 18), 8, 8),
    ((3, 3, 3), (1, 2, 2), (1, 1, 1), False, 2, 16, 32, (4, 9, 12), 0, 16),
    ((3, 3, 1), (2, 2, 1), (1, 1, 0), False, 2, 32, 48, (9, 10, 5), 8, 8),
    ((1, 1, 1), (2, 1, 2), (0, 0, 0), False, 2, 16, 96, (6, 5, 9), 8, 8),
    ((1, 2, 2), (1, 2, 2), (0, 0, 0), True, 2, 64, 32, (3, 5, 4), 8, 32),
    ((2, 2, 1), (2, 2, 1), (0, 0, 0), True, 2, 32, 16, (4, 3, 7), 0, 16),
    ((2, 1, 2), (2, 1, 2), (0, 0, 0), True, 1, 48, 128, (3, 6, 4), 16, 128),
]


def _cg_id(c):
    return f"{'T' if c[3] else ''}k{''.join(map(str, c[0]))}-s{''.join(map(str, c[1]))}-p{''.join(map(str, c[2]))}-Cout{c[6]}"


@pytest.mark.parametrize("case", CG_ANISO, ids=_cg_id)
def test_conv_gather_tc_per_axis_vs_float64(case):
    """Per-axis kernel, stride and padding; the transposed ones write into the upper or lower half of a concat buffer with bias."""
    k, s, p, t, N, Cin, Cout, sp, in_coff, out_coff = case
    taps = math.prod(_cdiv(kk, ss) for kk, ss in zip(k, s)) if t else math.prod(k)
    assert Cin // 16 * taps <= MAX_K16_STEPS
    g = _gen(500 + Cout + sum(k))
    x = torch.randn((N, Cin, *sp), generator=g).half()
    w = (torch.randn((Cin, Cout, *k) if t else (Cout, Cin, *k), generator=g) / (Cin * math.prod(k)) ** 0.5).half()
    b = torch.randn(Cout, generator=g)
    conv = (lambda a, ww, bb: F.conv_transpose3d(a, ww, bb, stride=s, padding=p)) if t else (lambda a, ww, bb: F.conv3d(a, ww, bb, stride=s, padding=p))
    r = conv(x.double(), w.double(), b.double())
    A = conv(x.double().abs(), w.double().abs(), b.double().abs())
    osp = tuple(r.shape[2:])
    _, xin = nc8_input(x, in_coff)
    pw = K.conv_gather_tc_pack_weight(w.float().to(DEV), k, s, p, t)

    def launch():
        go, out = nc8_output(N, Cout, out_coff, osp)
        _, st = K.conv_gather_tc(xin, pw, Cin, Cout, k, s, p, transposed=t, in_coff=in_coff, bias=b.to(DEV), out=out, out_coff=out_coff,
                                 want_stats=True)
        return go, st

    go, st, same_bits = twice(launch)
    what = f"conv_gather_tc k{k} s{s} p{p} {'transposed ' if t else ''}Cout={Cout} sp={sp}"
    go.assert_untouched_outside((slice(None), slice(out_coff // 8, (out_coff + Cout) // 8)), what)
    check("conv_gather_tc", what, from_nc8(go.view, out_coff, Cout).cpu(), r, A)
    check_stats("conv_gather_tc", what, st.cpu(), r.reshape(N, Cout, -1), A.reshape(N, Cout, -1))
    same_bits()


# ---------------------------------------------------------------------------------------------------- network
def _build(kw, seed):
    net = DynUNet(**kw)
    net.load_state_dict(fill_state_dict(net.state_dict(), seed))
    return net.eval().to(DEV)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(1e-6, np.abs(b).max()))


CASES = ["A", "B", "C"]


@pytest.mark.parametrize("tag", CASES)
@pytest.mark.parametrize("half", [False, True])
def test_dynunet_aniso_tc_matches_reference_fixture(golden_dir, tag, half):
    kw, shape, seed = ANISO_CASES[tag][:3]
    g = np.load(os.path.join(golden_dir, FIXTURE))
    net = _build(kw, seed)
    assert net._tc_ok
    if half:
        net = net.half()
    x = load_input(tag, g).to(DEV)
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
    assert abs(float(y.astype(np.float64).sum()) - ysum) <= 3e-2 * np.abs(ref).max() * y.size


@pytest.mark.parametrize("tag", CASES)
def test_dynunet_aniso_dispatch_is_measured(tag):
    kw, _, seed = ANISO_CASES[tag][:3]
    net = _build(kw, seed)
    x = load_input(tag)[:1].to(DEV)
    K.profile_start()
    net(x)
    fp16 = K.profile_stop()
    assert any(k.startswith("conv3x3_tc") for k in fp16), sorted(fp16)
    assert "conv_gather_tc" in fp16 and "conv3d_direct" not in fp16, sorted(fp16)
    K.profile_start()
    y32 = net(x.float())
    fp32 = K.profile_stop()
    assert y32.dtype == torch.float32
    assert not (TC_KERNELS & set(fp32)) and "conv3d_direct" in fp32, sorted(fp32)


@pytest.mark.parametrize("tag", CASES)
def test_dynunet_aniso_graphed_deterministic_and_follows_new_weights(tag):
    kw, _, seed = ANISO_CASES[tag][:3]
    net = _build(kw, seed)
    x = load_input(tag).to(DEV)
    y1 = net(x)        # captures the graph
    y2 = net(x)        # replays it
    assert torch.equal(y1, y2)
    assert torch.equal(net._forward_tc(x), y1)
    net.load_state_dict(fill_state_dict(net.state_dict(), seed + 100))
    y3 = net(x)
    assert not torch.equal(y3, y1)
    assert torch.equal(y3, _build(kw, seed + 100)._forward_tc(x))


@pytest.mark.parametrize("tag,shape,msg", [("A", (1, 1, 16, 64, 48), "divisible by 4 x 32 x 32"),
                                           ("B", (1, 2, 48, 32, 18), "divisible by 16 x 16 x 4"),
                                           ("C", (1, 1, 32, 14, 32), "divisible by 8 x 4 x 8")])
def test_dynunet_aniso_rejects_shapes_not_divisible_per_axis(tag, shape, msg):
    kw, _, seed = ANISO_CASES[tag][:3]
    net = _build(kw, seed)
    n0 = L.launch_count()
    with pytest.raises(ValueError, match=msg):
        net(torch.zeros(shape, device=DEV, dtype=torch.float16))
    assert L.launch_count() == n0


@pytest.mark.parametrize("tag,vol", [("A", (1, 1, 24, 96, 80)), ("B", (1, 2, 64, 48, 24)), ("C", (1, 1, 48, 24, 40))])
def test_dynunet_aniso_sliding_window_vs_generic_fp32(tag, vol):
    kw, shape, seed = ANISO_CASES[tag][:3]
    net = _build(kw, seed)
    v = torch.randn(vol, generator=_gen(95)).half()
    roi = shape[2:]
    got = sliding_window_inference(v.to(DEV), roi, 3, net, 0.5, "gaussian")
    ref = sliding_window_inference(v.float().to(DEV), roi, 3, net, 0.5, "gaussian")
    assert got.shape == ref.shape
    gg, r = got.float().cpu().numpy(), ref.cpu().numpy()
    err = _rel(gg, r)
    assert err <= 3e-2, f"rel err {err}"
    agree = float((gg.argmax(1) == r.argmax(1)).mean())
    assert agree >= 0.98, agree
