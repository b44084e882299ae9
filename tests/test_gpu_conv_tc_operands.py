"""The 3x3x3 tensor-core convolution at every N tile width (16-128) and depth block (BD = 1, 2, 4), plain, with the input
normalisation on the operand load (NORM) and with the folded 1x1x1 residual convolution (RES), at small ragged shapes.

Inputs and weights are rounded to fp16 first, so the torch fp32 reference differs only by accumulation order and the final fp16
rounding (tolerance 2e-3 of the output scale, as in test_gpu_conv_tc.py).  NORM must give the same bits as norm_act_nc8 followed
by the plain launch, and every variant the same bits run to run.
"""
import pytest
import torch
import torch.nn.functional as F

from monai_b200 import _kernels as K
from monai_b200 import _lib as L

pytestmark = pytest.mark.gpu
DEV = "cuda"

# depth -> BD chosen by the dispatcher (dispatch_bd in csrc/conv_tc.cu): 4 when 4 * NT (twice that with RES) fits 256
# accumulator columns, else 2; depth 1 always runs BD = 1
DEPTHS = [1, 3, 4]
WIDTHS = [16, 32, 48, 64, 80, 96, 112, 128]


def _inputs(N, Cin, Cout, sp, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn((N, Cin, *sp), generator=g) * torch.rand((1, Cin, 1, 1, 1), generator=g) * 3 + torch.randn((1, Cin, 1, 1, 1), generator=g)).half()
    w = (torch.randn((Cout, Cin, 3, 3, 3), generator=g) / (27 * Cin) ** 0.5).half()
    return x, w


def _close(got: torch.Tensor, ref: torch.Tensor):
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    assert err <= 2e-3 * scale + 1e-3, f"max err {err} (scale {scale})"


@pytest.mark.parametrize("D", DEPTHS)
@pytest.mark.parametrize("Cout", WIDTHS)
def test_plain(Cout, D):
    x, w = _inputs(2, 32, Cout, (D, 19, 11), seed=Cout + D)
    xr, pw = K.pack_nc8(x.to(DEV)), K.conv3x3x3_tc_pack_weight(w.float().to(DEV))
    y, st = K.conv3x3x3_tc(xr, pw, 32, Cout, want_stats=True)
    y_b, st_b = K.conv3x3x3_tc(xr, pw, 32, Cout, want_stats=True)
    assert torch.equal(y.buf, y_b.buf) and torch.equal(st, st_b)
    _close(K.unpack_nc8(y, dtype=torch.float32).cpu(), F.conv3d(x.float(), w.float(), None, padding=1))


@pytest.mark.parametrize("D", DEPTHS)
@pytest.mark.parametrize("Cout", WIDTHS)
def test_norm_on_the_operand_load(Cout, D):
    N, Cin = 2, 32
    x, w = _inputs(N, Cin, Cout, (D, 19, 11), seed=100 + Cout + D)
    xr, pw = K.pack_nc8(x.to(DEV)), K.conv3x3x3_tc_pack_weight(w.float().to(DEV))
    xf = x.float()
    st = torch.stack([xf.sum(dim=(2, 3, 4)), (xf * xf).sum(dim=(2, 3, 4))], dim=-1).reshape(N * Cin, 2).contiguous().to(DEV)
    fused, fst = K.conv3x3x3_tc(xr, pw, Cin, Cout, want_stats=True, in_norm=(st, 1e-5, L.ACT_LEAKY, 0.01))
    fused_b, fst_b = K.conv3x3x3_tc(xr, pw, Cin, Cout, want_stats=True, in_norm=(st, 1e-5, L.ACT_LEAKY, 0.01))
    assert torch.equal(fused.buf, fused_b.buf) and torch.equal(fst, fst_b)
    xn = K.norm_act_nc8(xr, Cin, st, act=L.ACT_LEAKY, slope=0.01)
    plain, pst = K.conv3x3x3_tc(xn, pw, Cin, Cout, want_stats=True)
    assert torch.equal(fused.buf, plain.buf) and torch.equal(fst, pst)
    _close(K.unpack_nc8(fused, dtype=torch.float32).cpu(), F.conv3d(K.unpack_nc8(xn, dtype=torch.float32).cpu(), w.float(), None, padding=1))


@pytest.mark.parametrize("D", DEPTHS)
@pytest.mark.parametrize("Cout", WIDTHS)
def test_folded_residual(Cout, D):
    N, Cin = 2, 32
    x, w = _inputs(N, Cin, Cout, (D, 19, 11), seed=200 + Cout + D)
    w3 = (torch.randn((Cout, Cin), generator=torch.Generator().manual_seed(Cout)) / Cin**0.5).half()
    xr, pw = K.pack_nc8(x.to(DEV)), K.conv3x3x3_tc_pack_weight(w.float().to(DEV))
    pw3 = K.gemm_tc_pack_weight(w3.float().to(DEV))
    y, st, y3, st3 = K.conv3x3x3_tc(xr, pw, Cin, Cout, want_stats=True, res_w=pw3)
    y_b, st_b, y3_b, st3_b = K.conv3x3x3_tc(xr, pw, Cin, Cout, want_stats=True, res_w=pw3)
    assert torch.equal(y.buf, y_b.buf) and torch.equal(y3.buf, y3_b.buf) and torch.equal(st, st_b) and torch.equal(st3, st3_b)
    _close(K.unpack_nc8(y, dtype=torch.float32).cpu(), F.conv3d(x.float(), w.float(), None, padding=1))
    _close(K.unpack_nc8(y3, dtype=torch.float32).cpu(), F.conv3d(x.float(), w3.float().reshape(Cout, Cin, 1, 1, 1)))


def test_norm_table_follows_the_batch_item():
    """More tiles than SMs, so a CTA walks tiles of several batch items and the per-item scale / shift table is rebuilt."""
    N, Cin, Cout, sp = 3, 48, 48, (16, 48, 32)
    x, w = _inputs(N, Cin, Cout, sp, seed=7)
    xr, pw = K.pack_nc8(x.to(DEV)), K.conv3x3x3_tc_pack_weight(w.float().to(DEV))
    xf = x.float()
    st = torch.stack([xf.sum(dim=(2, 3, 4)), (xf * xf).sum(dim=(2, 3, 4))], dim=-1).reshape(N * Cin, 2).contiguous().to(DEV)
    fused, fst = K.conv3x3x3_tc(xr, pw, Cin, Cout, want_stats=True, in_norm=(st, 1e-5, L.ACT_LEAKY, 0.01))
    xn = K.norm_act_nc8(xr, Cin, st, act=L.ACT_LEAKY, slope=0.01)
    plain, pst = K.conv3x3x3_tc(xn, pw, Cin, Cout, want_stats=True)
    assert torch.equal(fused.buf, plain.buf) and torch.equal(fst, pst)
