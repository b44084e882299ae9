"""The fp16 tensor-core forward of DynUNet and the affine InstanceNorm of the NC8 kernels (b200_norm_act_affine_nc8,
b200_conv3x3x3_tc_affine, b200_head_conv_norm_affine_nc8), against torch and against fixtures of the real reference
(tests/golden/dynunet_tc.npz, configurations in dynunet_tc_cases.py)."""
import importlib.util
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from monai_b200 import _kernels as K
from monai_b200 import _lib as L
from monai_b200.inferers import sliding_window_inference
from monai_b200.networks.nets import DynUNet
from weights import fill_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
TC_KERNELS = {"gemm_tc", "conv3x3x3_tc", "conv3x3x3_tc_affine", "conv_cin1_tc", "conv_gather_tc", "norm_act_nc8", "norm_act_affine_nc8",
              "head_conv_norm_nc8", "head_conv_norm_affine_nc8"}


def _load(golden_dir, name):
    spec = importlib.util.spec_from_file_location("_" + name, os.path.join(golden_dir, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _cases(golden_dir):
    mod = _load(golden_dir, "dynunet_tc_cases")
    return mod.DYNUNET_TC_CASES, mod.make_input


def _input(golden_dir, tag, g=None):
    """The case's fp16 input regenerated from its seed, checked against the sample the fixture keeps of the reference's input."""
    cases, make_input = _cases(golden_dir)
    _, shape, _, xseed = cases[tag]
    g = g if g is not None else np.load(os.path.join(golden_dir, "dynunet_tc.npz"))
    x = make_input(shape, xseed)
    s = int(g[f"{tag}.x_stride"])
    assert np.array_equal(x.numpy()[..., ::s, ::s, ::s], g[f"{tag}.x_sub"]), "regenerated input differs from the reference's"
    return x.to(DEV)


def _build(kw, seed):
    net = DynUNet(**kw)
    net.load_state_dict(fill_state_dict(net.state_dict(), seed))
    return net.eval().to(DEV)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(1e-6, np.abs(b).max()))


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _affine_params(C, seed):
    """gamma with negative, zero and positive entries; beta of either sign."""
    g = torch.randn(C, generator=_gen(seed)) * 1.5
    g[::5] = 0.0
    return g.to(DEV), (torch.randn(C, generator=_gen(seed + 1)) * 0.5).to(DEV)


def _stats(t):
    """{sum, sumsq} per (n, c) of an fp32 [N, C, ...] tensor, as the kernels' statistics."""
    f = t.flatten(2).double()
    return torch.stack([f.sum(-1), (f * f).sum(-1)], -1).reshape(-1, 2).float().contiguous()


def _torch_norm(x, g, b, eps):
    return F.instance_norm(x, weight=g, bias=b, eps=eps)


# ---------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("act,slope", [(L.ACT_NONE, 0.0), (L.ACT_LEAKY, 0.01), (L.ACT_LEAKY, 0.3), (L.ACT_RELU, 0.0)])
@pytest.mark.parametrize("with_res", [False, True])
def test_norm_act_affine_nc8_vs_torch(act, slope, with_res):
    N, C, sp, eps = 2, 32, (6, 10, 12), 1e-4
    x = torch.randn(N, 48, *sp, generator=_gen(1)).half().to(DEV) * 3 + 1
    r = torch.randn(N, 40, *sp, generator=_gen(2)).half().to(DEV) * 2 - 0.5
    xs, rs = x[:, 8:8 + C].float(), r[:, 8:8 + C].float()   # non-zero channel offsets in x, res and the output
    g, b = _affine_params(C, 3)
    rg, rb = _affine_params(C, 5)
    xn, rn = K.pack_nc8(x), K.pack_nc8(r)
    out = K.NC8(N, 48, sp, DEV)
    out.buf.zero_()
    kw = dict(res=rn, res_coff=8, res_stats=_stats(rs), res_gamma=rg, res_beta=rb) if with_res else {}
    K.norm_act_nc8(xn, C, _stats(xs), x_coff=8, act=act, slope=slope, out=out, out_coff=16, eps=eps, gamma=g, beta=b, **kw)
    ref = _torch_norm(xs, g, b, eps)
    if with_res:
        ref = ref + _torch_norm(rs, rg, rb, eps)
    if act == L.ACT_LEAKY:
        ref = F.leaky_relu(ref, slope)
    elif act == L.ACT_RELU:
        ref = F.relu(ref)
    got = K.unpack_nc8(out, dtype=torch.float32)
    assert torch.count_nonzero(got[:, :16]) == 0 and torch.count_nonzero(got[:, 16 + C:]) == 0
    err = float((got[:, 16:16 + C] - ref).abs().max())
    assert err <= 2.0**-10 * float(ref.abs().max()) + 1e-3, err   # fp16 storage of the result


def test_norm_act_affine_symbol_with_null_params_matches_old_symbol():
    N, C, sp = 2, 24, (5, 6, 7)
    x = K.pack_nc8(torch.randn(N, C, *sp, generator=_gen(11)).half().to(DEV))
    r = K.pack_nc8(torch.randn(N, C, *sp, generator=_gen(12)).half().to(DEV))
    st, rst = _stats(K.unpack_nc8(x, dtype=torch.float32)), _stats(K.unpack_nc8(r, dtype=torch.float32))
    old = K.norm_act_nc8(x, C, st, res=r, res_stats=rst, act=L.ACT_LEAKY, slope=0.01)
    new = K.NC8(N, C, sp, DEV)
    K._call("norm_act_affine_nc8", L.ptr(x.buf), x.C, 0, N, C, x.S, L.ptr(st), 1e-5, L.ptr(r.buf), r.C, 0, L.ptr(rst), L.ACT_LEAKY, 0.01,
            L.ptr(new.buf), new.C, 0, None, None, None, None, L.stream_ptr(torch.device(DEV)))
    assert torch.equal(old.buf, new.buf)


@pytest.mark.parametrize("Cin,Cout,N,D", [(32, 32, 1, 16), (32, 64, 1, 6), (64, 128, 1, 3), (64, 320, 1, 2), (48, 32, 1, 1), (32, 64, 3, 24)])
def test_conv_tc_affine_norm_on_load_equals_unfused(Cin, Cout, N, D):
    """in_affine fused on the operand load == affine norm_act_nc8 followed by the plain launch, bit for bit.  D selects BD = 4
    (D % 4 == 0 or D >= 16), 2 and 1; Cout 320 runs on 80-wide N tiles; the batch-3 launch has more tiles than SMs, so the
    operand table is rebuilt when the batch item changes."""
    sp = (D, 40, 24)
    raw = K.pack_nc8((torch.randn(N, Cin, *sp, generator=_gen(D + Cout)) * 2 + 0.3).half().to(DEV))
    st = _stats(K.unpack_nc8(raw, dtype=torch.float32))
    g, b = _affine_params(Cin, Cout)
    w = K.conv3x3x3_tc_pack_weight((torch.randn(Cout, Cin, 3, 3, 3, generator=_gen(7)) / (27 * Cin) ** 0.5).to(DEV))
    eps, slope = 1e-4, 0.1
    fused, fst = K.conv3x3x3_tc(raw, w, Cin, Cout, want_stats=True, in_norm=(st, eps, L.ACT_LEAKY, slope), in_affine=(g, b))
    normed = K.norm_act_nc8(raw, Cin, st, act=L.ACT_LEAKY, slope=slope, eps=eps, gamma=g, beta=b)
    plain, pst = K.conv3x3x3_tc(normed, w, Cin, Cout, want_stats=True)
    assert torch.equal(fused.buf, plain.buf)
    assert torch.equal(fst, pst)
    again, _ = K.conv3x3x3_tc(raw, w, Cin, Cout, want_stats=True, in_norm=(st, eps, L.ACT_LEAKY, slope), in_affine=(g, b))
    assert torch.equal(again.buf, fused.buf)
    # and the normalised operand is the affine InstanceNorm of torch
    ref = F.leaky_relu(_torch_norm(K.unpack_nc8(raw, dtype=torch.float32), g, b, eps), slope)
    nerr = float((K.unpack_nc8(normed, dtype=torch.float32) - ref).abs().max())
    assert nerr <= 2.0**-10 * float(ref.abs().max()) + 1e-3, nerr


@pytest.mark.parametrize("Cout", [1, 3, 14])
def test_head_conv_norm_affine_vs_torch(Cout):
    N, C, sp, eps, slope = 2, 32, (8, 12, 10), 1e-5, 0.01
    x = torch.randn(N, C, *sp, generator=_gen(21)).half().to(DEV) * 2 + 0.5
    g, b = _affine_params(C, 22)
    wt = torch.randn(Cout, C, 1, 1, 1, generator=_gen(23)).to(DEV) / C**0.5
    bias = torch.randn(Cout, generator=_gen(24)).to(DEV)
    y = K.head_conv_norm_nc8(K.pack_nc8(x), _stats(x.float()), None, 0, None, slope, eps, wt, bias, out_dtype=torch.float32, gamma=g, beta=b)
    # float64 on the CPU: cuDNN convolutions may run in TF32, far coarser than the kernel's fp32 FMAs
    x64, g64, b64 = x.double().cpu(), g.double().cpu(), b.double().cpu()
    ref = F.conv3d(F.leaky_relu(_torch_norm(x64, g64, b64, eps), slope), wt.double().cpu(), bias.double().cpu())
    err = float((y.double().cpu() - ref).abs().max())
    assert err <= 1e-4 * float(ref.abs().max()) + 1e-4, err


# ---------------------------------------------------------------------------------------------------- network
@pytest.mark.parametrize("tag,half", [("A", False), ("A", True), ("B", False)])
def test_dynunet_tc_matches_reference_fixture(golden_dir, tag, half):
    kw, shape, seed, _ = _cases(golden_dir)[0][tag]
    g = np.load(os.path.join(golden_dir, "dynunet_tc.npz"))
    net = _build(kw, seed)
    if half:
        net = net.half()   # a checkpoint moved to fp16 as a whole takes the same path
    x = _input(golden_dir, tag, g)
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


def test_dynunet_dispatch_is_measured(golden_dir):
    kw, _, seed, _ = _cases(golden_dir)[0]["A"]
    net = _build(kw, seed)
    x = _input(golden_dir, "A")[:1]
    K.profile_start()
    net(x)
    fp16 = K.profile_stop()
    assert {"conv3x3x3_tc_affine", "conv3x3x3_tc", "conv_gather_tc", "gemm_tc", "head_conv_norm_affine_nc8"} <= set(fp16), sorted(fp16)
    assert "conv3d_direct" not in fp16, sorted(fp16)
    K.profile_start()
    y32 = net(x.float())
    fp32 = K.profile_stop()
    assert y32.dtype == torch.float32
    assert not (TC_KERNELS & set(fp32)), sorted(fp32)
    assert "conv3d_direct" in fp32


def _ineligible(golden_dir):
    """Case 1 of the generic fixture (anisotropic plan, filters of 8) and a BatchNorm variant of case A."""
    kw1, _, seed1 = _load(golden_dir, "dynunet_cases").DYNUNET_CASES[1]
    kwa, _, seeda, _ = _cases(golden_dir)[0]["A"]
    return [(kw1, seed1, (1, 2, 16, 32, 24)), (dict(kwa, norm_name="batch"), seeda, (1, 1, 32, 32, 32))]


@pytest.mark.parametrize("i", [0, 1])
def test_dynunet_ineligible_configs_take_the_generic_path(golden_dir, i):
    kw, seed, shape = _ineligible(golden_dir)[i]
    net = _build(kw, seed).half()
    assert not net._tc_ok
    x = torch.randn(shape, generator=_gen(50 + i)).half().to(DEV)
    K.profile_start()
    y = net(x)
    prof = K.profile_stop()
    assert not (TC_KERNELS & set(prof)) and "conv3d_direct" in prof, sorted(prof)
    assert torch.equal(y, net._forward_generic(x))


def test_dynunet_tc_deterministic_graphed_and_follows_new_weights(golden_dir):
    kw, _, seed, _ = _cases(golden_dir)[0]["B"]
    net = _build(kw, seed)
    x = _input(golden_dir, "B")
    y1 = net(x)        # captures the graph
    y2 = net(x)        # replays it
    assert torch.equal(y1, y2)
    assert torch.equal(net._forward_tc(x), y1)
    net.load_state_dict(fill_state_dict(net.state_dict(), seed + 100))
    y3 = net(x)
    assert not torch.equal(y3, y1)
    fresh = _build(kw, seed + 100)
    assert torch.equal(y3, fresh._forward_tc(x))


def test_dynunet_tc_rejects_bad_shapes(golden_dir):
    kw, _, seed, _ = _cases(golden_dir)[0]["A"]
    net = _build(kw, seed)
    with pytest.raises(ValueError, match="divisible by 32"):
        net(torch.zeros(1, 1, 64, 64, 48, device=DEV, dtype=torch.float16))
    with pytest.raises(ValueError, match="input"):
        net(torch.zeros(1, 2, 64, 64, 64, device=DEV, dtype=torch.float16))


def test_dynunet_tc_sliding_window_vs_generic_fp32(golden_dir):
    kw, _, seed, _ = _cases(golden_dir)[0]["A"]
    net = _build(kw, seed)
    vol = torch.randn(1, 1, 96, 80, 64, generator=_gen(95)).half()
    # 4 windows of 64^3 at overlap 0.5: one batch of 3 and a remainder batch of 1
    got = sliding_window_inference(vol.to(DEV), (64, 64, 64), 3, net, 0.5, "gaussian")
    ref = sliding_window_inference(vol.float().to(DEV), (64, 64, 64), 3, net, 0.5, "gaussian")
    assert got.shape == ref.shape
    g, r = got.float().cpu().numpy(), ref.cpu().numpy()
    err = _rel(g, r)
    assert err <= 3e-2, f"rel err {err}"
    agree = float((g.argmax(1) == r.argmax(1)).mean())
    assert agree >= 0.98, agree
