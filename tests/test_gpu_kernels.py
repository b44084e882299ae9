"""GPU parity of the individual CUDA kernels (through the C ABI) against plain torch fp32 references."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from monai_b200 import _kernels as K
from monai_b200 import _lib as L

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize(
    "cin,cout,k,s,p,sp",
    [(1, 16, 3, 2, 1, (18, 17, 20)), (16, 32, 3, 2, 1, (12, 12, 12)), (5, 7, 3, 1, 1, (6, 9, 11)), (8, 4, 1, 1, 0, (5, 5, 5)),
     (3, 2, (3, 1, 2), (2, 1, 1), (1, 0, 0), (9, 8, 7)), (32, 16, 2, 2, 0, (8, 8, 8))],
)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_conv3d_direct(cin, cout, k, s, p, sp, dtype):
    g = torch.Generator().manual_seed(0)
    x = torch.randn((2, cin, *sp), generator=g)
    w = torch.randn((cout, cin, *([k] * 3 if isinstance(k, int) else k)), generator=g) * 0.2
    b = torch.randn(cout, generator=g)
    xd = x.to(DEV, dtype)
    ref = F.conv3d(xd.float().cpu(), w, b, stride=s, padding=p)
    got = K.conv3d_direct(xd, w.to(DEV), b.to(DEV), stride=s, padding=p)
    assert got.dtype == dtype
    tol = 1e-4 if dtype == torch.float32 else 2e-2
    torch.testing.assert_close(got.float().cpu(), ref, rtol=tol, atol=tol)


@pytest.mark.parametrize("cin,cout,k,s,p,op,sp", [(6, 4, 3, 2, 1, 1, (5, 6, 7)), (32, 2, 3, 2, 1, 1, (8, 8, 8)), (8, 8, 2, 2, 0, 0, (4, 5, 6)), (4, 3, 3, 1, 1, 0, (5, 5, 5))])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_conv_transpose3d_direct(cin, cout, k, s, p, op, sp, dtype):
    g = torch.Generator().manual_seed(1)
    x = torch.randn((2, cin, *sp), generator=g)
    w = torch.randn((cin, cout, k, k, k), generator=g) * 0.2
    b = torch.randn(cout, generator=g)
    xd = x.to(DEV, dtype)
    ref = F.conv_transpose3d(xd.float().cpu(), w, b, stride=s, padding=p, output_padding=op)
    got = K.conv3d_direct(xd, w.to(DEV), b.to(DEV), stride=s, padding=p, transposed=True, output_padding=op)
    tol = 1e-4 if dtype == torch.float32 else 2e-2
    torch.testing.assert_close(got.float().cpu(), ref, rtol=tol, atol=tol)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_instance_norm_prelu_and_residual(dtype):
    g = torch.Generator().manual_seed(2)
    x = (torch.randn((3, 5, 7, 9, 11), generator=g) * 2 + 0.5).to(DEV, dtype)
    r = torch.randn((3, 5, 7, 9, 11), generator=g).to(DEV, dtype)
    gamma, beta = torch.rand(5, generator=g).to(DEV) + 0.5, torch.randn(5, generator=g).to(DEV)
    slope = torch.tensor([0.2], device=DEV)
    stats = K.instnorm_stats(x)
    xf = x.float()
    torch.testing.assert_close(stats[:, 0].cpu(), xf.sum(dim=(2, 3, 4)).reshape(-1).cpu(), rtol=1e-4, atol=1e-2)
    got = K.norm_act(x, stats, 1e-5, gamma, beta, None, None, L.ACT_PRELU, 0.0, slope)
    ref = F.prelu(F.instance_norm(xf, weight=gamma, bias=beta, eps=1e-5), slope)
    tol = 1e-4 if dtype == torch.float32 else 1e-2
    torch.testing.assert_close(got.float(), ref, rtol=tol, atol=tol)
    # UnetResBlock tail: lrelu(norm(x) + norm(res))
    got = K.norm_act(x, stats, 1e-5, None, None, r, K.instnorm_stats(r), L.ACT_LEAKY, 0.01)
    ref = F.leaky_relu(F.instance_norm(xf, eps=1e-5) + F.instance_norm(r.float(), eps=1e-5), 0.01)
    torch.testing.assert_close(got.float(), ref, rtol=tol, atol=tol)
    got = K.norm_act(x, act=L.ACT_GELU)
    torch.testing.assert_close(got.float(), F.gelu(xf), rtol=tol, atol=tol)


def test_maxpool_and_cat():
    x = torch.randn((2, 3, 8, 6, 10), device=DEV)
    torch.testing.assert_close(K.maxpool3d_2(x), F.max_pool3d(x, 2), rtol=0, atol=0)
    y = torch.randn((2, 5, 8, 6, 10), device=DEV)
    torch.testing.assert_close(K.cat_channels([x, y]), torch.cat([x, y], 1), rtol=0, atol=0)
    small = torch.randn((1, 2, 3, 4, 5), device=DEV)
    dst = torch.zeros((1, 4, 4, 5, 6), device=DEV)
    K.copy_channels(small, dst, 1)
    ref = F.pad(small, (0, 1, 0, 1, 0, 1), mode="replicate")
    torch.testing.assert_close(dst[:, 1:3], ref, rtol=0, atol=0)


def _grid_sample_ref(src, mat, out_shape, mode, pad, align):
    """reference semantics via F.grid_sample on an explicitly normalised grid (fp64)."""
    Do, Ho, Wo = out_shape
    idx = torch.stack(torch.meshgrid(torch.arange(Do), torch.arange(Ho), torch.arange(Wo), indexing="ij"), -1).double()
    m = torch.tensor(mat, dtype=torch.float64).reshape(3, 4)
    coords = idx @ m[:, :3].T + m[:, 3]  # (d, h, w) source voxel coordinates
    size = torch.tensor(src.shape[1:], dtype=torch.float64)
    if align:
        norm = coords / (size - 1) * 2 - 1
    else:
        norm = (coords * 2 + 1) / size - 1
    grid = norm.flip(-1)[None]  # xyz order
    return F.grid_sample(src[None].double(), grid, mode=mode, padding_mode=pad, align_corners=align)[0].float()


@pytest.mark.parametrize("interp,mode", [(L.INTERP_LINEAR, "bilinear"), (L.INTERP_NEAREST, "nearest")])
@pytest.mark.parametrize("pad,pname", [(L.PAD_ZEROS, "zeros"), (L.PAD_BORDER, "border"), (L.PAD_REFLECTION, "reflection")])
@pytest.mark.parametrize("align", [False, True])
def test_resample_affine_matches_grid_sample(interp, mode, pad, pname, align):
    g = torch.Generator().manual_seed(3)
    src = torch.randn((2, 9, 11, 13), generator=g)
    mat = [0.9137, 0.1021, -0.0533, -1.3177, -0.1219, 1.0931, 0.0713, 0.8049, 0.0307, -0.0911, 0.8467, 2.1043]
    out_shape = (12, 10, 15)
    ref = _grid_sample_ref(src, mat, out_shape, mode, pname, align)
    got = K.resample_affine(src.to(DEV), out_shape, mat, interp, pad, align)
    if interp == L.INTERP_NEAREST:
        frac = (got.cpu() != ref).float().mean().item()
        assert frac < 0.01, frac  # rounding ties may differ at fp64 round-off
    else:
        torch.testing.assert_close(got.cpu(), ref, rtol=1e-4, atol=1e-4)


def test_separable_filter_matches_conv3d():
    g = torch.Generator().manual_seed(4)
    x = torch.randn((2, 10, 12, 14), generator=g)
    taps = [torch.rand(5, generator=g), torch.rand(3, generator=g), torch.rand(7, generator=g)]
    ref = x[None]
    for d, t in enumerate(taps):
        shape = [1, 1, 1, 1, 1]
        shape[d + 2] = -1
        k = t.reshape(shape).repeat(2, 1, 1, 1, 1)
        padv = [0, 0, 0]
        padv[d] = (t.numel() - 1) // 2
        ref = F.conv3d(ref, k, padding=padv, groups=2)
    got = K.separable_filter3d(x.to(DEV), [t.to(DEV) for t in taps])
    torch.testing.assert_close(got.cpu(), ref[0], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("n,sp", [(9, (20, 37, 48)), (9, (5, 3, 8)), (5, (33, 17, 64)), (3, (16, 16, 16)), (1, (4, 4, 4))])
def test_separable_filter_sliding_window_path(n, sp):
    """Equal odd tap counts <= 9, fp32 and W % 4 == 0 take the register sliding-window kernels (runs of 16 along D / H,
    ragged run tails, volumes shorter than the filter radius): compare with conv3d AND bit-compare with the generic path
    (same data embedded in a volume whose W is not a multiple of 4 cannot share a launch, so the generic path is forced
    through fp16->fp32 dispatch rules instead: different tap counts per axis)."""
    g = torch.Generator().manual_seed(n + sp[0])
    x = torch.randn((2, *sp), generator=g)
    taps = [torch.rand(n, generator=g) for _ in range(3)]
    ref = x[None]
    for d, t in enumerate(taps):
        shape = [1, 1, 1, 1, 1]
        shape[d + 2] = -1
        padv = [0, 0, 0]
        padv[d] = (n - 1) // 2
        ref = F.conv3d(ref, t.reshape(shape).repeat(2, 1, 1, 1, 1), padding=padv, groups=2)
    got = K.separable_filter3d(x.to(DEV), [t.to(DEV) for t in taps])
    torch.testing.assert_close(got.cpu(), ref[0], rtol=1e-5, atol=1e-5)
    if n >= 3:
        # generic kernels: pad the last axis' taps with two zeros on each side (n + 4 taps, unequal counts -> generic path);
        # zero taps add exact zeros, so the two paths must agree bit for bit
        wide = torch.cat([torch.zeros(2), taps[2], torch.zeros(2)])
        gen = K.separable_filter3d(x.to(DEV), [taps[0].to(DEV), taps[1].to(DEV), wide.to(DEV)])
        torch.testing.assert_close(got, gen, rtol=0, atol=0)


def test_nc8_roundtrip():
    x = torch.randn((2, 24, 5, 6, 7), device=DEV).half()
    p = K.pack_nc8(x)
    assert p.buf.shape == (2, 3, 5, 6, 7, 8)
    torch.testing.assert_close(p.buf, x.reshape(2, 3, 8, 5, 6, 7).permute(0, 1, 3, 4, 5, 2).contiguous(), rtol=0, atol=0)
    torch.testing.assert_close(K.unpack_nc8(p), x, rtol=0, atol=0)


def test_errors_surface_as_python_exceptions():
    with pytest.raises(ValueError, match="multiples of 16"):
        K.conv3x3x3_tc_pack_weight(torch.zeros(8, 8, 3, 3, 3, device=DEV))
    with pytest.raises(TypeError):
        K.instnorm_stats(torch.zeros(1, 1, 4, 4, 4, device=DEV, dtype=torch.float64))
