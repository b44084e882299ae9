"""GPU parity of the wgmma implicit-GEMM 3x3x3 convolution against a torch fp32 reference of the same op.

Inputs and weights are rounded to fp16 first (the kernel's storage type), so the only differences left are the
fp32 accumulation order and the final fp16 rounding of the output: tolerance 2e-3 relative to the output scale.
"""
import pytest
import torch
import torch.nn.functional as F

from monai_b200 import _kernels as K

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _run(N, Cin, Cout, sp, bias, seed=0, in_pad=0, out_pad=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((N, Cin, *sp), generator=g).half()
    w = (torch.randn((Cout, Cin, 3, 3, 3), generator=g) / (27 * Cin) ** 0.5).half()
    b = torch.randn(Cout, generator=g) if bias else None
    ref = F.conv3d(x.float(), w.float(), b, padding=1)
    # optionally embed the input / output in wider concat buffers (channel offsets)
    xin = K.NC8(N, Cin + in_pad, sp, DEV)
    xin.buf.fill_(float("nan")) if in_pad else None
    K.pack_nc8(x.to(DEV), xin, c_off=in_pad)
    out = K.NC8(N, Cout + out_pad, sp, DEV)
    out.buf.zero_()
    pw = K.conv3x3x3_tc_pack_weight(w.float().to(DEV))
    y, stats = K.conv3x3x3_tc(xin, pw, Cin, Cout, in_coff=in_pad, bias=None if b is None else b.to(DEV), out=out, out_coff=out_pad, want_stats=True)
    torch.cuda.synchronize()
    got = K.unpack_nc8(y, Cout, c_off=out_pad, dtype=torch.float32).cpu()
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    assert err <= 2e-3 * scale + 1e-3, f"max err {err} (scale {scale}) for N={N} Cin={Cin} Cout={Cout} sp={sp}"
    S = sp[0] * sp[1] * sp[2]
    torch.testing.assert_close(stats[:, 0].cpu() / S, ref.mean(dim=(2, 3, 4)).reshape(-1), rtol=1e-2, atol=2e-3 * scale)
    torch.testing.assert_close(stats[:, 1].cpu() / S, (ref * ref).mean(dim=(2, 3, 4)).reshape(-1), rtol=1e-2, atol=1e-3 * scale * scale)
    if out_pad:
        assert float(out.buf[:, : out_pad // 8].abs().max()) == 0.0  # neighbouring channels untouched


@pytest.mark.parametrize(
    "N,Cin,Cout,sp",
    [
        (1, 16, 16, (4, 16, 8)),      # exactly one CTA tile, one K slice
        (1, 16, 16, (5, 19, 11)),     # ragged edges in all three axes
        (2, 48, 48, (8, 32, 16)),     # SwinUNETR encoder shapes (NT=48)
        (1, 96, 48, (12, 24, 24)),    # decoder1.conv1 shape class
        (1, 32, 128, (6, 12, 12)),    # NT=128
        (1, 64, 192, (3, 6, 6)),      # Cout tiled 2 x 96, tiny volume
        (1, 384, 32, (2, 3, 3)),      # deep K loop on a volume smaller than one tile
    ],
)
def test_conv3x3x3_tc(N, Cin, Cout, sp):
    _run(N, Cin, Cout, sp, bias=False)


def test_conv3x3x3_tc_bias_and_channel_slices():
    _run(2, 32, 48, (7, 20, 13), bias=True, seed=3, in_pad=16, out_pad=8)


def test_conv3x3x3_tc_full_window_shape():
    _run(1, 48, 48, (96, 96, 96), bias=False, seed=5)


@pytest.mark.parametrize(
    "N,Cin,Cout,sp",
    [
        (1, 16, 16, (5, 19, 11)),     # ragged edges: the zero padding must stay zero AFTER the normalisation
        (2, 48, 48, (8, 32, 16)),     # UnetResBlock conv2 of SwinUNETR (BD = 4)
        (3, 48, 48, (6, 12, 12)),     # BD = 2 path, batch > 1 (per-item statistics)
        (1, 192, 96, (3, 6, 6)),      # many K slices on a tiny volume (BD = 1)
    ],
)
def test_conv3x3x3_tc_instance_norm_on_the_operand_load(N, Cin, Cout, sp):
    """conv2(lrelu(norm1(y1))) of UnetResBlock (monai/networks/blocks/dynunet_block.py:97-103) with the normalisation applied to
    the staged halo tile: bit-identical to running norm_act_nc8 first (same expression, same fp16 rounding of the operand)."""
    from monai_b200 import _lib as L

    g = torch.Generator().manual_seed(11)
    x = (torch.randn((N, Cin, *sp), generator=g) * torch.rand((1, Cin, 1, 1, 1), generator=g) * 3 + torch.randn((1, Cin, 1, 1, 1), generator=g)).half()
    w = (torch.randn((Cout, Cin, 3, 3, 3), generator=g) / (27 * Cin) ** 0.5).half()
    pw = K.conv3x3x3_tc_pack_weight(w.float().to(DEV))
    xr = K.pack_nc8(x.to(DEV))
    S = sp[0] * sp[1] * sp[2]
    xf = x.float()
    st = torch.stack([xf.sum(dim=(2, 3, 4)), (xf * xf).sum(dim=(2, 3, 4))], dim=-1).reshape(N * Cin, 2).contiguous().to(DEV)
    fused, fst = K.conv3x3x3_tc(xr, pw, Cin, Cout, want_stats=True, in_norm=(st, 1e-5, L.ACT_LEAKY, 0.01))
    xn = K.norm_act_nc8(xr, Cin, st, act=L.ACT_LEAKY, slope=0.01)
    plain, pst = K.conv3x3x3_tc(xn, pw, Cin, Cout, want_stats=True)
    assert torch.equal(fused.buf, plain.buf)
    assert torch.equal(fst, pst)
    # and against torch: instance_norm + leaky_relu + conv3d in fp32 on the fp16-rounded normalised operand
    ref = F.conv3d(K.unpack_nc8(xn, dtype=torch.float32).cpu(), w.float(), None, padding=1)
    got = K.unpack_nc8(fused, dtype=torch.float32).cpu()
    assert (got - ref).abs().max().item() <= 2e-3 * ref.abs().max().item() + 1e-3
    nrm = F.leaky_relu(F.instance_norm(xf, eps=1e-5), 0.01)
    assert (K.unpack_nc8(xn, dtype=torch.float32).cpu() - nrm).abs().max().item() < 2e-2
    assert not (S == 0)


@pytest.mark.parametrize(
    "N,Cin,Cout,sp",
    [
        (2, 96, 48, (8, 32, 16)),     # decoder1 / decoder2 of SwinUNETR: single accumulator set (BD = 4, 2 x 192 columns)
        (1, 32, 16, (5, 19, 11)),     # ragged edges, two accumulator sets
        (3, 48, 96, (6, 12, 12)),     # BD = 2, wider N, batch > 1
        (1, 192, 128, (3, 6, 6)),     # many K slices, BD = 1
    ],
)
def test_conv3x3x3_tc_with_the_folded_residual_convolution(N, Cin, Cout, sp):
    """UnetResBlock.conv1 and .conv3 (1x1x1, same input; monai/networks/blocks/dynunet_block.py:75-87, 104-108) from ONE launch: the
    3x3x3 output is bit-identical to the plain launch (its statistics to fp32 round-off), the 1x1x1 output matches gemm_tc and torch."""
    g = torch.Generator().manual_seed(21)
    x = torch.randn((N, Cin, *sp), generator=g).half()
    w = (torch.randn((Cout, Cin, 3, 3, 3), generator=g) / (27 * Cin) ** 0.5).half()
    w3 = (torch.randn((Cout, Cin), generator=g) / Cin**0.5).half()
    pw = K.conv3x3x3_tc_pack_weight(w.float().to(DEV))
    pw3 = K.gemm_tc_pack_weight(w3.float().to(DEV))
    xr = K.pack_nc8(x.to(DEV))
    y, st, y3, st3 = K.conv3x3x3_tc(xr, pw, Cin, Cout, want_stats=True, res_w=pw3)
    y_plain, st_plain = K.conv3x3x3_tc(xr, pw, Cin, Cout, want_stats=True)
    assert torch.equal(y.buf, y_plain.buf)
    # same fp32 values, but two epilogue groups split the planes: the partial sums associate differently (fp64 finish)
    torch.testing.assert_close(st, st_plain, rtol=2e-6, atol=1e-6 * float(st_plain.abs().max()))
    g3, gst3 = K.gemm_tc(xr, pw3, Cin, Cout, want_stats=True)
    a, b = K.unpack_nc8(y3, dtype=torch.float32), K.unpack_nc8(g3, dtype=torch.float32)
    assert float((a - b).abs().max()) <= 2e-3 * float(b.abs().max())
    torch.testing.assert_close(st3, gst3, rtol=2e-3, atol=2e-3 * float(gst3.abs().max()))
    ref3 = F.conv3d(x.float(), w3.float().reshape(Cout, Cin, 1, 1, 1))
    assert float((a.cpu() - ref3).abs().max()) <= 2e-3 * float(ref3.abs().max()) + 1e-3
    # deterministic
    y_b, st_b, y3_b, st3_b = K.conv3x3x3_tc(xr, pw, Cin, Cout, want_stats=True, res_w=pw3)
    assert torch.equal(y3.buf, y3_b.buf) and torch.equal(st3, st3_b)
