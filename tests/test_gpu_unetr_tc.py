"""The fp16 tensor-core forward of UNETR and its wgmma attention kernel (b200_mhsa_tc), against torch and against fixtures of the
real reference (tests/golden/unetr_tc.npz, configurations in unetr_tc_cases.py)."""
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

from monai_b200 import _kernels as K
from monai_b200.inferers import sliding_window_inference
from monai_b200.networks.nets import UNETR
from weights import fill_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
TC_KERNELS = {"gemm_tc", "mhsa_tc", "conv3x3x3_tc", "conv_cin1_tc", "conv_gather_tc", "window_attention_tc", "mlp_fused_tc"}


def _cases(golden_dir):
    spec = importlib.util.spec_from_file_location("_unetr_tc_cases", os.path.join(golden_dir, "unetr_tc_cases.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.UNETR_TC_CASES, mod.make_input


def _input(golden_dir, tag, g=None):
    """The case's fp16 input regenerated from its seed, checked against the sample the fixture keeps of the reference's input."""
    cases, make_input = _cases(golden_dir)
    _, shape, _, xseed = cases[tag]
    g = g if g is not None else np.load(os.path.join(golden_dir, "unetr_tc.npz"))
    x = make_input(shape, xseed)
    s = int(g[f"{tag}.x_stride"])
    assert np.array_equal(x.numpy()[..., ::s, ::s, ::s], g[f"{tag}.x_sub"]), "regenerated input differs from the reference's"
    return x.to(DEV)


def _build(kw, seed):
    net = UNETR(**kw)
    net.load_state_dict(fill_state_dict(net.state_dict(), seed))
    return net.eval().to(DEV)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(1e-6, np.abs(b).max()))


def _qkv(N, heads, S, dim, seed):
    """fp16 qkv [N, 3C, S] with q pre-scaled by dim^-0.5 * log2(e), as the host folds it into the projection."""
    g = torch.Generator().manual_seed(seed)
    C = heads * dim
    qkv = torch.randn((N, 3 * C, S), generator=g)
    qkv[:, :C] *= dim**-0.5 * K.LOG2E
    return qkv.half()


@pytest.mark.parametrize("N,heads,S", [(1, 12, 216), (3, 12, 144), (2, 6, 512), (1, 1, 27), (2, 12, 1000), (1, 2, 1)])
def test_mhsa_tc_vs_torch(N, heads, S):
    qkv = _qkv(N, heads, S, 64, 100 + S)
    C = heads * 64
    got = K.mhsa_tc(K.pack_nc8(qkv.reshape(N, 3 * C, S, 1, 1).to(DEV)), C, heads)
    y = K.unpack_nc8(got, dtype=torch.float32).reshape(N, C, S)
    # fp32 attention on the same fp16 values; scores are in log2 units: softmax_2(s) = softmax(s * ln 2)
    q, k, v = qkv.float().to(DEV).reshape(N, 3, heads, 64, S).unbind(1)
    att = torch.softmax(torch.einsum("nhdx,nhdy->nhxy", q, k) * math.log(2.0), dim=-1)
    ref = torch.einsum("nhxy,nhdy->nhdx", att, v).reshape(N, C, S)
    # P is rounded to fp16 (relative 2^-11 per weight, the row sum uses the same rounded values) and the output is stored in
    # fp16 (2^-11 of its magnitude): the error stays below 2^-10 of max|v| plus 2^-10 of max|out|
    tol = 2.0**-10 * float(v.abs().max()) + 2.0**-10 * float(ref.abs().max())
    err = float((y - ref).abs().max())
    assert err <= tol, (err, tol)
    again = K.mhsa_tc(K.pack_nc8(qkv.reshape(N, 3 * C, S, 1, 1).to(DEV)), C, heads)
    assert torch.equal(again.buf, got.buf)


def test_mhsa_tc_refuses_other_head_dims():
    qkv = _qkv(1, 4, 40, 32, 5)
    with pytest.raises(ValueError, match="head_dim must be 64"):
        K.mhsa_tc(K.pack_nc8(qkv.reshape(1, 3 * 128, 40, 1, 1).to(DEV)), 128, 4)


@pytest.mark.parametrize("tag", ["A", "B"])
def test_unetr_tc_matches_reference_fixture(golden_dir, tag):
    kw, shape, seed, _ = _cases(golden_dir)[0][tag]
    g = np.load(os.path.join(golden_dir, "unetr_tc.npz"))
    net = _build(kw, seed)
    if tag == "A":
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


def test_unetr_dispatch_is_measured(golden_dir):
    kw, _, seed, _ = _cases(golden_dir)[0]["A"]
    net = _build(kw, seed)
    x = _input(golden_dir, "A")[:1]
    K.profile_start()
    net(x)
    fp16 = K.profile_stop()
    assert {"mhsa_tc", "gemm_tc", "conv3x3x3_tc"} <= set(fp16), sorted(fp16)
    assert "conv3d_direct" not in fp16 and "mhsa_cf" not in fp16, sorted(fp16)
    K.profile_start()
    y32 = net(x.float())
    fp32 = K.profile_stop()
    assert y32.dtype == torch.float32
    assert not (TC_KERNELS & set(fp32)), sorted(fp32)
    assert "conv3d_direct" in fp32 and "mhsa_cf" in fp32


def test_unetr_tc_deterministic_graphed_and_follows_new_weights(golden_dir):
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


def test_unetr_tc_sliding_window_vs_generic_fp32(golden_dir):
    kw, _, seed, _ = _cases(golden_dir)[0]["A"]
    net = _build(kw, seed)
    vol = torch.randn(1, 1, 128, 112, 96, generator=torch.Generator().manual_seed(95)).half()
    # 4 windows of 96^3 at overlap 0.5: one batch of 3 and a remainder batch of 1
    got = sliding_window_inference(vol.to(DEV), (96, 96, 96), 3, net, 0.5, "gaussian")
    ref = sliding_window_inference(vol.float().to(DEV), (96, 96, 96), 3, net, 0.5, "gaussian")
    assert got.shape == ref.shape
    g, r = got.float().cpu().numpy(), ref.cpu().numpy()
    err = _rel(g, r)
    assert err <= 3e-2, f"rel err {err}"
    agree = float((g.argmax(1) == r.argmax(1)).mean())
    assert agree >= 0.98, agree
