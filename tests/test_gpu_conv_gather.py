"""GPU parity of the general wgmma convolution (cp.async im2col producer): stride-1/2 Conv3d and ConvTranspose3d
vs torch fp32 references on fp16-rounded operands (tolerance 2e-3 of the output scale, fp32 accumulation)."""
import pytest
import torch
import torch.nn.functional as F

from monai_b200 import _kernels as K

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _check(got, ref, what):
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    assert err <= 2e-3 * scale + 1e-3, f"{what}: max err {err} (scale {scale})"


@pytest.mark.parametrize(
    "N,Cin,Cout,k,s,p,sp",
    [(2, 16, 32, 3, 2, 1, (12, 10, 14)), (1, 32, 64, 3, 2, 1, (24, 24, 24)), (1, 128, 256, 3, 1, 1, (6, 6, 6)), (2, 16, 16, 3, 1, 1, (5, 9, 7)),
     (1, 64, 128, 3, 2, 1, (12, 12, 12)), (1, 48, 48, 1, 1, 0, (7, 8, 9))],
)
def test_conv_forward(N, Cin, Cout, k, s, p, sp):
    g = torch.Generator().manual_seed(0)
    x = torch.randn((N, Cin, *sp), generator=g).half()
    w = (torch.randn((Cout, Cin, k, k, k), generator=g) / (k**3 * Cin) ** 0.5).half()
    b = torch.randn(Cout, generator=g)
    ref = F.conv3d(x.float(), w.float(), b, stride=s, padding=p)
    pw = K.conv_gather_tc_pack_weight(w.float().to(DEV), k, s, p, False)
    y, st = K.conv_gather_tc(K.pack_nc8(x.to(DEV)), pw, Cin, Cout, k, s, p, bias=b.to(DEV), want_stats=True)
    _check(K.unpack_nc8(y, dtype=torch.float32).cpu(), ref, "forward")
    S = ref[0, 0].numel()
    torch.testing.assert_close(st[:, 0].cpu() / S, ref.mean(dim=(2, 3, 4)).reshape(-1), rtol=1e-2, atol=3e-3 * ref.abs().max().item())


@pytest.mark.parametrize("N,Cin,Cout,sp", [(2, 32, 16, (6, 5, 7)), (1, 384, 64, (6, 6, 6)), (1, 64, 16, (12, 12, 12))])
def test_conv_transposed_k3_s2(N, Cin, Cout, sp):
    g = torch.Generator().manual_seed(1)
    x = torch.randn((N, Cin, *sp), generator=g).half()
    w = (torch.randn((Cin, Cout, 3, 3, 3), generator=g) / (27 * Cin / 8) ** 0.5).half()
    b = torch.randn(Cout, generator=g)
    ref = F.conv_transpose3d(x.float(), w.float(), b, stride=2, padding=1, output_padding=1)
    pw = K.conv_gather_tc_pack_weight(w.float().to(DEV), 3, 2, 1, True)
    # write into a channel slice of a wider concat buffer
    cat = K.NC8(N, Cout + 16, tuple(2 * s for s in sp), DEV)
    cat.buf.zero_()
    y, st = K.conv_gather_tc(K.pack_nc8(x.to(DEV)), pw, Cin, Cout, 3, 2, 1, transposed=True, output_padding=1, bias=b.to(DEV), out=cat, out_coff=16, want_stats=True)
    _check(K.unpack_nc8(cat, Cout, c_off=16, dtype=torch.float32).cpu(), ref, "transposed")
    assert float(cat.buf[:, :2].abs().max()) == 0.0
    S = ref[0, 0].numel()
    torch.testing.assert_close(st[:, 1].cpu() / S, (ref * ref).mean(dim=(2, 3, 4)).reshape(-1), rtol=2e-2, atol=3e-3 * ref.abs().max().item() ** 2)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_transposed_head_to_ncdhw(dtype):
    """the UNet top layer: ConvTranspose3d(32 -> 2, k3, s2) written as NCDHW logits"""
    g = torch.Generator().manual_seed(2)
    x = torch.randn((2, 32, 8, 9, 10), generator=g).half()
    w = (torch.randn((32, 2, 3, 3, 3), generator=g) / 10).half()
    b = torch.randn(2, generator=g)
    ref = F.conv_transpose3d(x.float(), w.float(), b, stride=2, padding=1, output_padding=1)
    pw = K.conv_gather_tc_pack_weight(w.float().to(DEV), 3, 2, 1, True)
    y, _ = K.conv_gather_tc(K.pack_nc8(x.to(DEV)), pw, 32, 2, 3, 2, 1, transposed=True, output_padding=1, bias=b.to(DEV), ncdhw_dtype=dtype)
    assert y.shape == ref.shape and y.dtype == dtype
    _check(y.float().cpu(), ref, "head")


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_thin_head_cuda_core_kernel(dtype):
    g = torch.Generator().manual_seed(4)
    x = torch.randn((2, 32, 6, 7, 9), generator=g).half()
    w = (torch.randn((32, 2, 3, 3, 3), generator=g) / 10).half()
    b = torch.randn(2, generator=g)
    ref = F.conv_transpose3d(x.float(), w.float(), b, stride=2, padding=1, output_padding=1)
    y = K.convt3s2_head_nc8(K.pack_nc8(x.to(DEV)), 32, w.float().to(DEV), b.to(DEV), out_dtype=dtype)
    assert y.shape == ref.shape and y.dtype == dtype
    _check(y.float().cpu(), ref, "thin head")
