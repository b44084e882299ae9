"""GPU parity of the SwinUNETR path (wgmma convs / GEMMs, window attention, LayerNorm / merging kernels) against the
reference fixtures (real MONAI outputs) and the torch-CPU oracle.  The network computes in fp16 with fp32
accumulation, the oracle in fp32: tolerances are stated relative to the output scale."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from monai_b200 import _kernels as K
from monai_b200 import _lib as L
from monai_b200.networks.nets import SwinUNETR
from monai_b200.networks.nets.swin_unetr import window_plan
from oracle import networks as onet
from weights import fill_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    return float(np.abs(a - b).max() / max(1e-6, np.abs(b).max()))


def _to_nc8(x):  # [N,C,*sp] float -> NC8
    return K.pack_nc8(x.to(DEV).half())


def test_gemm_tc_linear_bias_gelu_residual():
    g = torch.Generator().manual_seed(0)
    for (S, Kd, N) in [(300, 48, 144), (1000, 192, 48), (129, 768, 3072), (64, 3072, 768)]:
        x = torch.randn((2, Kd, 1, 1, S), generator=g).half()
        w = (torch.randn((N, Kd), generator=g) / Kd**0.5).half()
        b = torch.randn(N, generator=g)
        r = torch.randn((2, N, 1, 1, S), generator=g).half()
        ref = F.linear(x.float().reshape(2, Kd, S).transpose(1, 2), w.float(), b)  # [2,S,N]
        y, _ = K.gemm_tc(_to_nc8(x), K.gemm_tc_pack_weight(w.to(DEV)), Kd, N, bias=b.to(DEV))
        got = K.unpack_nc8(y, dtype=torch.float32).cpu().reshape(2, N, S).transpose(1, 2)
        assert _rel(got.numpy(), ref.numpy()) < 3e-3, (S, Kd, N)
        y, _ = K.gemm_tc(_to_nc8(x), K.gemm_tc_pack_weight(w.to(DEV)), Kd, N, bias=b.to(DEV), act=L.ACT_GELU, res=_to_nc8(r))
        got = K.unpack_nc8(y, dtype=torch.float32).cpu().reshape(2, N, S).transpose(1, 2)
        ref2 = F.gelu(ref) + r.float().reshape(2, N, S).transpose(1, 2)
        assert _rel(got.numpy(), ref2.numpy()) < 3e-3, (S, Kd, N)


def test_fused_mlp_matches_reference_math_and_the_unfused_kernels():
    """x + fc2(gelu(fc1(LN(x)))) -- monai/networks/nets/swin_unetr.py:675-698 with blocks/mlp.py:75-80 -- in one launch."""
    g = torch.Generator().manual_seed(3)
    C, Hd = 48, 192
    for (Nb, S) in [(1, 128), (2, 1000), (3, 128 * 151 + 77), (4, 110592)]:
        x = (torch.randn((Nb, C, 1, 1, S), generator=g) * 1.5 + 0.3).half()
        w1 = (torch.randn((Hd, C), generator=g) / C**0.5).half()
        w2 = (torch.randn((C, Hd), generator=g) / Hd**0.5).half()
        b1, b2 = torch.randn(Hd, generator=g) * 0.2, torch.randn(C, generator=g) * 0.2
        gam, bet = 1 + 0.2 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
        xd = _to_nc8(x)
        p1, p2 = K.gemm_tc_pack_weight(w1.to(DEV)), K.gemm_tc_pack_weight(w2.to(DEV))
        out = K.mlp_fused_tc(xd, p1, b1.to(DEV), p2, b2.to(DEV), Hd, gam.to(DEV), bet.to(DEV), 1e-5)
        got = K.unpack_nc8(out, dtype=torch.float32).reshape(Nb, C, S)
        # the unfused kernels (LayerNorm, two GEMMs): the fused path rounds the same intermediates to fp16
        y = K.layernorm_nc8(xd, gam.to(DEV), bet.to(DEV), 1e-5)
        h, _ = K.gemm_tc(y, p1, C, Hd, bias=b1.to(DEV), act=L.ACT_GELU)
        o2, _ = K.gemm_tc(h, p2, Hd, C, bias=b2.to(DEV), res=xd)
        unf = K.unpack_nc8(o2, dtype=torch.float32).reshape(Nb, C, S)
        d_unf = float((got - unf).abs().max())
        assert d_unf < 4e-3 * float(unf.abs().max()), (Nb, S, d_unf)
        if S <= 20000:
            xt = x.float().reshape(Nb, C, S).transpose(1, 2).to(DEV)
            ref = xt + F.linear(F.gelu(F.linear(F.layer_norm(xt, (C,), gam.to(DEV), bet.to(DEV), 1e-5), w1.float().to(DEV), b1.to(DEV))), w2.float().to(DEV), b2.to(DEV))
            r = _rel(got.transpose(1, 2).cpu().numpy(), ref.cpu().numpy())
            assert r < 3e-3, (Nb, S, r)
        # run to run bit-identical
        out2 = K.mlp_fused_tc(xd, p1, b1.to(DEV), p2, b2.to(DEV), Hd, gam.to(DEV), bet.to(DEV), 1e-5)
        assert torch.equal(out.buf, out2.buf)


def test_gemm_tc_conv_transpose_k2s2_and_1x1_stats():
    g = torch.Generator().manual_seed(1)
    x = torch.randn((2, 96, 3, 5, 6), generator=g).half()
    w = (torch.randn((96, 48, 2, 2, 2), generator=g) / 10).half()
    ref = F.conv_transpose3d(x.float(), w.float(), stride=2)
    wg = w.float().permute(2, 3, 4, 1, 0).reshape(8 * 48, 96).contiguous()
    cat = K.NC8(2, 96, (6, 10, 12), DEV)
    cat.buf.zero_()
    K.gemm_tc(_to_nc8(x), K.gemm_tc_pack_weight(wg.to(DEV)), 96, 8 * 48, out=cat, out_coff=48, mode=2)
    got = K.unpack_nc8(cat, 48, c_off=48, dtype=torch.float32).cpu()
    assert _rel(got.numpy(), ref.numpy()) < 3e-3
    assert float(cat.buf[:, :6].abs().max()) == 0.0
    w1 = (torch.randn((48, 96, 1, 1, 1), generator=g) / 10).half()
    ref1 = F.conv3d(x.float(), w1.float())
    y, st = K.gemm_tc(_to_nc8(x), K.gemm_tc_pack_weight(w1.reshape(48, 96).to(DEV)), 96, 48, want_stats=True)
    assert _rel(K.unpack_nc8(y, dtype=torch.float32).cpu().numpy(), ref1.numpy()) < 3e-3
    torch.testing.assert_close(st[:, 0].cpu(), ref1.sum(dim=(2, 3, 4)).reshape(-1), rtol=2e-2, atol=2e-2)


def test_layernorm_gather_and_patch_merging():
    g = torch.Generator().manual_seed(2)
    x = torch.randn((2, 48, 6, 9, 10), generator=g).half()
    gamma, beta = torch.rand(48, generator=g) + 0.5, torch.randn(48, generator=g)
    ref = F.layer_norm(x.float().permute(0, 2, 3, 4, 1), (48,), gamma, beta).permute(0, 4, 1, 2, 3)
    got = K.unpack_nc8(K.layernorm_nc8(_to_nc8(x), gamma.to(DEV), beta.to(DEV)), dtype=torch.float32).cpu()
    assert _rel(got.numpy(), ref.numpy()) < 2e-3
    # gather with the window plan (shifted, padded): compare against pad + roll + window_partition
    src, region, nW, n = window_plan((6, 9, 10), (7, 7, 7), (3, 3, 3))
    xw = K.layernorm_nc8(_to_nc8(x), gamma.to(DEV), beta.to(DEV), src=torch.from_numpy(src).to(DEV), out_sp=(1, nW, n))
    got = K.unpack_nc8(xw, dtype=torch.float32).cpu().reshape(2, 48, nW, n).permute(0, 2, 3, 1).reshape(-1, n, 48)
    t = ref.permute(0, 2, 3, 4, 1)
    t = F.pad(t, (0, 0, 0, 4, 0, 5, 0, 0))  # to (6->6 [window clamps to 6], 9->14, 10->14)
    ws, ss = (6, 7, 7), (0, 3, 3)
    t = torch.roll(t, shifts=(-ss[0], -ss[1], -ss[2]), dims=(1, 2, 3))
    want = onet._window_partition(t, ws)
    assert _rel(got.numpy(), want.numpy()) < 2e-3
    want_mask = onet._compute_mask([6, 14, 14], ws, ss)
    reg = torch.from_numpy(region)
    got_mask = torch.where(reg[:, None, :] != reg[:, :, None], -100.0, 0.0)
    torch.testing.assert_close(got_mask, want_mask.float(), rtol=0, atol=0)
    # patch merging (both slice orders), odd sizes padded
    sd = {"p.norm.weight": torch.rand(384, generator=g) + 0.5, "p.norm.bias": torch.randn(384, generator=g), "p.reduction.weight": torch.eye(96, 384)}
    for v2 in (False, True):
        m = K.patch_merge_ln_nc8(_to_nc8(x), sd["p.norm.weight"].to(DEV), sd["p.norm.bias"].to(DEV), v2=v2)
        got = K.unpack_nc8(m, dtype=torch.float32).cpu()
        xt = F.pad(x.float().permute(0, 2, 3, 4, 1), (0, 0, 0, 0, 0, 1, 0, 0))
        order = list(__import__("itertools").product(range(2), range(2), range(2))) if v2 else [(0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 1, 1)]
        cat = torch.cat([xt[:, i::2, j::2, k::2, :] for i, j, k in order], -1)
        want = F.layer_norm(cat, (384,), sd["p.norm.weight"], sd["p.norm.bias"]).permute(0, 4, 1, 2, 3)
        assert _rel(got.numpy(), want.numpy()) < 2e-3, v2


@pytest.mark.parametrize("ws,n,nW,heads", [((7, 7, 7), 343, 5, 3), ((7, 7, 7), 216, 3, 6), ((7, 7, 7), 8, 4, 24)])
def test_window_attention_matches_reference_math(ws, n, nW, heads):
    from monai_b200.networks.nets.swin_unetr import WindowAttention

    g = torch.Generator().manual_seed(3)
    C, B = heads * 16, 2
    mod = WindowAttention(C, heads, ws, qkv_bias=True)
    table = torch.randn(mod.relative_position_bias_table.shape, generator=g)
    qkv = torch.randn((B, nW, n, 3 * C), generator=g).half()
    # reference bias gather: table[relative_position_index[:n, :n]] (swin_unetr.py:514-518)
    bias = table[mod.relative_position_index[:n, :n].reshape(-1)].reshape(n, n, heads).permute(2, 0, 1)
    region = torch.randint(0, 3, (nW, n), generator=g, dtype=torch.int32)
    q, k, v = qkv.float().reshape(B, nW, n, 3, heads, 16).permute(3, 0, 1, 4, 2, 5)
    attn = (q * 0.25) @ k.transpose(-2, -1) + bias[None, None]
    mask = torch.where(region[:, None, :] != region[:, :, None], -100.0, 0.0)  # [nW, i, j]
    for reg, a in ((region, attn + mask[None, :, None]), (None, attn)):
        ref = (a.softmax(-1) @ v).permute(0, 1, 3, 2, 4).reshape(B, nW, n, C)
        x = K.pack_nc8(qkv.permute(0, 3, 1, 2).reshape(B, 3 * C, 1, nW, n).contiguous().to(DEV))
        out = K.window_attention_nc8(x, C, heads, nW, n, 0.25, table.to(DEV), ws, None if reg is None else reg.to(DEV))
        got = K.unpack_nc8(out, dtype=torch.float32).cpu().reshape(B, C, nW, n).permute(0, 2, 3, 1)
        assert _rel(got.numpy(), ref.numpy()) < 4e-3, (n, reg is None)


@pytest.mark.parametrize("ws,n,nW,heads", [((7, 7, 7), 343, 5, 3), ((7, 7, 7), 216, 3, 6), ((7, 7, 7), 8, 4, 24), ((7, 7, 7), 196, 9, 12)])
def test_window_attention_tcgen05_matches_reference_math(ws, n, nW, heads):
    """b200_window_attention_tc: bias + shift mask added by the tensor core, online softmax in registers, P V on wgmma."""
    from monai_b200.networks.nets.swin_unetr import WindowAttention

    g = torch.Generator().manual_seed(5)
    C, B = heads * 16, 3
    mod = WindowAttention(C, heads, ws, qkv_bias=True)
    table = torch.randn(mod.relative_position_bias_table.shape, generator=g)
    qkv = torch.randn((B, nW, n, 3 * C), generator=g).half()
    bias = table[mod.relative_position_index[:n, :n].reshape(-1)].reshape(n, n, heads).permute(2, 0, 1)
    # at most 8 distinct mask patterns (as the shift mask has): windows draw their region row from 3 prototypes
    protos = torch.randint(0, 3, (3, n), generator=g, dtype=torch.int32)
    region = protos[torch.arange(nW) % 3]
    q, k, v = qkv.float().reshape(B, nW, n, 3, heads, 16).permute(3, 0, 1, 4, 2, 5)
    attn = (q * 0.25) @ k.transpose(-2, -1) + bias[None, None]
    mask = torch.where(region[:, None, :] != region[:, :, None], -100.0, 0.0)
    # the kernel works in log2 units: q rows pre-scaled by scale * log2(e) (done in the qkv projection in the network)
    qs = qkv.clone().float()
    qs[..., :C] *= 0.25 * K.LOG2E
    x = K.pack_nc8(qs.half().permute(0, 3, 1, 2).reshape(B, 3 * C, 1, nW, n).contiguous().to(DEV))
    for reg, a in ((region, attn + mask[None, :, None]), (None, attn)):
        ref = (a.softmax(-1) @ v).permute(0, 1, 3, 2, 4).reshape(B, nW, n, C)
        sched, reps, ntypes = K.window_attention_tc_plan(None if reg is None else reg.numpy(), nW, n)
        assert ntypes <= 8
        pb = K.window_attention_tc_pack_bias(table.to(DEV), heads, n, ws, None if reps is None else torch.from_numpy(reps).to(DEV), ntypes)
        out = K.window_attention_tc(x, C, heads, nW, n, pb, torch.from_numpy(sched).to(DEV), ntypes)
        torch.cuda.synchronize()
        got = K.unpack_nc8(out, dtype=torch.float32).cpu().reshape(B, C, nW, n).permute(0, 2, 3, 1)
        err = _rel(got.numpy(), ref.numpy())
        assert err < 4e-3, (n, reg is None, err)


def _conv_cin1_cuda_core(x, weight, bias, k, stride, pad, want_stats=False):
    """b200_conv_cin1_nc8 called directly: the CUDA-core stem on shapes that K.conv_cin1_nc8 sends to the wgmma stem."""
    N, _, D, H, W = x.shape
    Cout = weight.shape[0]
    out = K.NC8(N, Cout, tuple((s + 2 * pad - k) // stride + 1 for s in (D, H, W)), x.device)
    stats = ws = None
    if want_stats:
        stats = torch.empty((N * Cout, 2), device=x.device, dtype=torch.float32)
        ws = K._ws(L.load().b200_conv_cin1_nc8_workspace_bytes(N, D, H, W, Cout, k, stride, pad), x.device)
    w32, b32 = weight.float().contiguous(), None if bias is None else bias.float().contiguous()
    K._call("conv_cin1_nc8", L.ptr(x), L.dt(x), N, D, H, W, L.ptr(w32), L.ptr(b32), Cout, k, stride, pad, L.ptr(out.buf), out.C, 0,
            L.ptr(stats), L.ptr(ws), L.stream_ptr(x.device))
    return out, stats


def test_instance_norm_statistics_are_deterministic():
    """The epilogue statistics never go through floating-point atomics: two runs give the same bits, and the values agree
    with a float64 reference (conv3x3x3_tc, gemm_tc with a 1x1x1 conv, the single-channel stems)."""
    g = torch.Generator().manual_seed(6)
    x = torch.randn((3, 32, 10, 20, 24), generator=g).half()
    w = (torch.randn((48, 32, 3, 3, 3), generator=g) / 30).half()
    xn, wp = _to_nc8(x), K.conv3x3x3_tc_pack_weight(w.float().to(DEV))
    runs = [K.conv3x3x3_tc(xn, wp, 32, 48, want_stats=True) for _ in range(3)]
    torch.cuda.synchronize()
    ref = F.conv3d(x.double(), w.double(), padding=1)
    for y, st in runs[1:]:
        assert torch.equal(st, runs[0][1]) and torch.equal(y.buf, runs[0][0].buf)
    st = runs[0][1].cpu().double().reshape(3, 48, 2)
    torch.testing.assert_close(st[..., 0], ref.sum(dim=(2, 3, 4)), rtol=2e-3, atol=5e-2)
    torch.testing.assert_close(st[..., 1], (ref * ref).sum(dim=(2, 3, 4)), rtol=2e-3, atol=5e-2)
    w1 = (torch.randn((48, 32, 1, 1, 1), generator=g) / 6).half()
    wl = K.gemm_tc_pack_weight(w1.reshape(48, 32).to(DEV))
    r1 = [K.gemm_tc(xn, wl, 32, 48, want_stats=True)[1] for _ in range(3)]
    assert torch.equal(r1[0], r1[1]) and torch.equal(r1[0], r1[2])
    ref1 = F.conv3d(x.double(), w1.double())
    torch.testing.assert_close(r1[0].cpu().double().reshape(3, 48, 2)[..., 1], (ref1 * ref1).sum(dim=(2, 3, 4)), rtol=2e-3, atol=5e-2)
    u = torch.randn((3, 1, 12, 20, 24), generator=g).half().to(DEV)
    wc = torch.randn((48, 1, 3, 3, 3), generator=g).to(DEV) / 5
    for stem in (K.conv_cin1_nc8, _conv_cin1_cuda_core):
        rs = [stem(u, wc, None, 3, 1, 1, want_stats=True)[1] for _ in range(3)]
        assert torch.equal(rs[0], rs[1]) and torch.equal(rs[0], rs[2])
        refc = F.conv3d(u.double().cpu(), wc.double().cpu(), padding=1)
        torch.testing.assert_close(rs[0].cpu().double().reshape(3, 48, 2)[..., 1], (refc * refc).sum(dim=(2, 3, 4)), rtol=3e-3, atol=5e-2)


@pytest.mark.parametrize("force_cuda_core", [False, True])
def test_cin1_stem_and_head(force_cuda_core):
    g = torch.Generator().manual_seed(4)
    x = torch.randn((2, 1, 8, 10, 12), generator=g)
    stem = _conv_cin1_cuda_core if force_cuda_core else K.conv_cin1_nc8   # False: wgmma stems for (3,1,1) and (2,2,0)
    for k, s, p in [(3, 1, 1), (2, 2, 0), (1, 1, 0)]:
        w, b = torch.randn((48, 1, k, k, k), generator=g) / k**1.5, torch.randn(48, generator=g)
        ref = F.conv3d(x, w, b, stride=s, padding=p)
        for xin in (x, x.half()):
            y, st = stem(xin.to(DEV), w.to(DEV), b.to(DEV), k, s, p, want_stats=True)
            assert _rel(K.unpack_nc8(y, dtype=torch.float32).cpu().numpy(), ref.numpy()) < 3e-3, (k, s, p, xin.dtype)
            torch.testing.assert_close(st[:, 0].cpu(), ref.sum(dim=(2, 3, 4)).reshape(-1), rtol=2e-3, atol=3e-2)
    # a volume that needs several tiles per axis and a partial last tile on every axis
    xb = torch.randn((2, 1, 21, 37, 19), generator=g).half()
    wb = torch.randn((32, 1, 3, 3, 3), generator=g) / 5
    refb = F.conv3d(xb.float(), wb, padding=1)
    yb, _ = stem(xb.to(DEV), wb.to(DEV), None, 3, 1, 1)
    assert _rel(K.unpack_nc8(yb, dtype=torch.float32).cpu().numpy(), refb.numpy()) < 3e-3
    h = torch.randn((2, 48, 4, 5, 6), generator=g).half()
    w, b = torch.randn((2, 48, 1, 1, 1), generator=g) / 7, torch.randn(2, generator=g)
    ref = F.conv3d(h.float(), w, b)
    got = K.head_conv_nc8(_to_nc8(h), w.to(DEV), b.to(DEV), out_dtype=torch.float32)
    assert _rel(got.cpu().numpy(), ref.numpy()) < 1e-3


def test_fused_residual_tail_kernels():
    """head_conv_norm_nc8 (norm2 + residual + lrelu + 1x1x1 head in one pass) and norm_act_cin1res_nc8 (the one-channel
    residual branch evaluated analytically) against the unfused formulation in torch fp32."""
    g = torch.Generator().manual_seed(11)
    N, C, sp = 2, 48, (6, 10, 12)
    y2 = (torch.randn((N, C, *sp), generator=g) * 1.7 + 0.3).half()
    y3 = (torch.randn((N, C, *sp), generator=g) * 0.6 - 0.2).half()
    w = torch.randn((2, C, 1, 1, 1), generator=g) / C**0.5
    b = torch.randn(2, generator=g)
    y2n, y3n = _to_nc8(y2), _to_nc8(y3)
    st2, st3 = K.instnorm_stats(y2.to(DEV)), K.instnorm_stats(y3.to(DEV))
    t = F.leaky_relu(F.instance_norm(y2.float()) + F.instance_norm(y3.float()), 0.01)
    ref = F.conv3d(t, w, b)
    got = K.head_conv_norm_nc8(y2n, st2, y3n, 0, st3, 0.01, 1e-5, w.to(DEV), b.to(DEV), out_dtype=torch.float32)
    assert _rel(got.cpu().numpy(), ref.numpy()) < 3e-3
    # identity residual (no conv3 branch): res added as is
    ref_id = F.conv3d(F.leaky_relu(F.instance_norm(y2.float()) + y3.float(), 0.01), w, b)
    got_id = K.head_conv_norm_nc8(y2n, st2, y3n, 0, None, 0.01, 1e-5, w.to(DEV), b.to(DEV), out_dtype=torch.float16)
    assert _rel(got_id.float().cpu().numpy(), ref_id.numpy()) < 5e-3
    # one-channel residual branch: instnorm(conv1x1x1(u)) == alpha_c * u + beta_c
    u = (torch.randn((N, 1, *sp), generator=g) * 2.0 + 0.5).half()
    w3 = torch.randn((C, 1, 1, 1, 1), generator=g)
    ref_c = F.leaky_relu(F.instance_norm(y2.float()) + F.instance_norm(F.conv3d(u.float(), w3)), 0.01)
    got_c = K.norm_act_cin1res_nc8(y2n, C, st2, u.to(DEV), K.instnorm_stats(u.to(DEV)), w3.to(DEV), act=L.ACT_LEAKY, slope=0.01)
    assert _rel(K.unpack_nc8(got_c).float().cpu().numpy(), ref_c.numpy()) < 3e-3


def test_head_at_48_channels_and_14_classes():
    """head_conv_norm_nc8 at C = 48: 14 classes, several batch items, a ragged last block, fp16 and fp32 logits -- against
    torch fp32 (dynunet_block.py:104-111 + 247-267)."""
    g = torch.Generator().manual_seed(5)
    N, C, sp, CO = 3, 48, (9, 20, 23), 14
    y2 = (torch.randn((N, C, *sp), generator=g) * 1.3 + 0.2).half()
    y3 = (torch.randn((N, C, *sp), generator=g) * 0.8 - 0.1).half()
    w = torch.randn((CO, C, 1, 1, 1), generator=g) / C**0.5
    b = torch.randn(CO, generator=g)
    y2n, y3n = _to_nc8(y2), _to_nc8(y3)
    st2, st3 = K.instnorm_stats(y2.to(DEV)), K.instnorm_stats(y3.to(DEV))
    ref = F.conv3d(F.leaky_relu(F.instance_norm(y2.float()) + F.instance_norm(y3.float()), 0.01), w, b)
    for dt in (torch.float32, torch.float16):
        got = K.head_conv_norm_nc8(y2n, st2, y3n, 0, st3, 0.01, 1e-5, w.to(DEV), b.to(DEV), out_dtype=dt)
        assert got.dtype == dt and tuple(got.shape) == tuple(ref.shape)
        r = _rel(got.float().cpu().numpy(), ref.numpy())
        assert r < 3e-3, (dt, r)
    again = K.head_conv_norm_nc8(y2n, st2, y3n, 0, st3, 0.01, 1e-5, w.to(DEV), b.to(DEV), out_dtype=torch.float16)
    assert torch.equal(again, got)


def _build():
    with contextlib.redirect_stdout(io.StringIO()):
        net = SwinUNETR(in_channels=1, out_channels=2, feature_size=48)
    net.load_state_dict(fill_state_dict(net.state_dict(), 4))
    return net.eval().to(DEV)


@pytest.mark.parametrize("tag", ["64", "96x64x64"])
def test_swin_unetr_matches_reference_fixture(golden_dir, tag):
    g = np.load(os.path.join(golden_dir, f"swin_unetr_fs48_{tag}.npz"))
    net = _build()
    x = torch.from_numpy(g["x"]).to(DEV)  # fp16 input
    y = net(x).float().cpu().numpy()
    assert y.shape[2:] == g["x"].shape[2:]
    err = _rel(y[..., ::4, ::4, ::4], g["y_sub"])
    assert err < 3e-2, f"rel err {err}"  # fp16 activations through ~40 layers vs the fp32 reference
    assert abs(float(y.mean()) - float(g["y_mean"])) < 2e-2 * float(g["y_absmean"])
    agree = (y[..., ::4, ::4, ::4].argmax(1) == g["y_sub"].argmax(1)).mean()
    assert agree > 0.98, agree


def test_swin_unetr_batch_and_fp32_input_vs_oracle():
    net = _build()
    x = torch.randn(2, 1, 64, 64, 64, generator=torch.Generator().manual_seed(8))
    sd = {k: (v.float() if v.is_floating_point() else v).cpu() for k, v in net.state_dict().items()}
    with torch.no_grad():
        ref = onet.swin_unetr_forward(sd, x).numpy()
    y = net(x.to(DEV))  # fp32 in -> fp32 logits (internals fp16)
    assert y.dtype == torch.float32
    assert _rel(y.cpu().numpy(), ref) < 3e-2
    with pytest.raises(ValueError, match="must be divisible by 2\\*\\*5"):
        net(torch.zeros(1, 1, 48, 64, 64, device=DEV))
