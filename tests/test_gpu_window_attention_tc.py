"""b200_window_attention_tc (csrc/attn_tc.cu) across its schedule: every padded-key template, row tiles whose last warps
or whole warpgroups hold only padding rows, 1-8 shift-mask types, batch > 1, 3 / 6 / 12 / 24 heads and launches with more tiles than SMs
(grouped tile order, bias reloads).  Checked against the fp32 torch formula, against the mma.sync kernel
(b200_window_attention_nc8) and for bit-identical reruns."""
import pytest
import torch

from monai_b200 import _kernels as K
from monai_b200.networks.nets.swin_unetr import WindowAttention

pytestmark = pytest.mark.gpu
DEV = "cuda"
SCALE = 0.25   # head_dim 16 ** -0.5


def _rel(a, b):
    return float((a - b).abs().max() / max(1e-6, float(b.abs().max())))


def _case(ws, n, nW, heads, B, ntypes, seed):
    """(kernel output, fp32 reference, window_attention_nc8 output, rerun), all [B, nW, n, C] float32 on the device."""
    g = torch.Generator().manual_seed(seed)
    C = heads * 16
    mod = WindowAttention(C, heads, ws, qkv_bias=True)
    table = torch.randn(mod.relative_position_bias_table.shape, generator=g)
    qkv = torch.randn((B, nW, n, 3 * C), generator=g).half()
    region = None
    if ntypes > 1:
        protos = torch.randint(0, 4, (ntypes, n), generator=g, dtype=torch.int32)
        region = protos[torch.arange(nW) % ntypes]
    sched, reps, nt = K.window_attention_tc_plan(None if region is None else region.numpy(), nW, n)
    assert nt == ntypes

    # fp32 reference on the device: softmax(q k^T * scale + bias [+ mask]) v
    bias = table[mod.relative_position_index[:n, :n].reshape(-1)].reshape(n, n, heads).permute(2, 0, 1).to(DEV)
    q, k, v = qkv.to(DEV).float().reshape(B, nW, n, 3, heads, 16).permute(3, 0, 1, 4, 2, 5)
    a = (q * SCALE) @ k.transpose(-2, -1) + bias[None, None]
    if region is not None:
        r = region.to(DEV)
        a = a + torch.where(r[:, None, :] != r[:, :, None], -100.0, 0.0)[None, :, None]
    ref = (a.softmax(-1) @ v).permute(0, 1, 3, 2, 4).reshape(B, nW, n, C)
    del a

    def unpack(out):
        return K.unpack_nc8(out, dtype=torch.float32).reshape(B, C, nW, n).permute(0, 2, 3, 1)

    qs = qkv.clone().float()
    qs[..., :C] *= SCALE * K.LOG2E   # the kernel works in log2 units (the network folds this into the qkv projection)
    x = K.pack_nc8(qs.half().permute(0, 3, 1, 2).reshape(B, 3 * C, 1, nW, n).contiguous().to(DEV))
    pb = K.window_attention_tc_pack_bias(table.to(DEV), heads, n, ws, None if reps is None else torch.from_numpy(reps).to(DEV), ntypes)
    sd = torch.from_numpy(sched).to(DEV)
    got = unpack(K.window_attention_tc(x, C, heads, nW, n, pb, sd, ntypes))
    again = unpack(K.window_attention_tc(x, C, heads, nW, n, pb, sd, ntypes))
    x8 = K.pack_nc8(qkv.permute(0, 3, 1, 2).reshape(B, 3 * C, 1, nW, n).contiguous().to(DEV))
    nc8 = unpack(K.window_attention_nc8(x8, C, heads, nW, n, SCALE, table.to(DEV), ws, None if region is None else region.to(DEV)))
    torch.cuda.synchronize()
    return got, ref, nc8, again


# one case per padded-key template (n_pad = 32 .. 352); with 192-row tiles, 343 and 129 have warps whose rows are all padding,
# and 8, 96 and 216 have whole warpgroups of padding rows
@pytest.mark.parametrize("ws,n,nW,heads,B,ntypes", [
    ((7, 7, 7), 8, 6, 24, 2, 1),
    ((7, 7, 7), 33, 5, 12, 2, 2),
    ((7, 7, 7), 96, 4, 6, 3, 3),
    ((7, 7, 7), 128, 4, 3, 2, 4),
    ((7, 7, 7), 129, 5, 6, 2, 5),
    ((7, 7, 7), 196, 6, 12, 1, 6),
    ((6, 6, 6), 216, 7, 24, 2, 7),
    ((7, 7, 7), 256, 8, 3, 2, 8),
    ((7, 7, 7), 300, 3, 6, 2, 1),
    ((7, 7, 7), 320, 3, 3, 2, 2),
    ((7, 7, 7), 343, 9, 3, 2, 4),
    ((8, 8, 8), 352, 3, 6, 2, 1),
])
def test_window_attention_tc_shapes(ws, n, nW, heads, B, ntypes):
    got, ref, nc8, again = _case(ws, n, nW, heads, B, ntypes, seed=n)
    assert torch.isfinite(got).all()
    assert _rel(got, ref) < 4e-3
    assert _rel(got, nc8) < 4e-3
    assert torch.equal(got, again)


# more tiles than SMs: 61 windows x 2 items x 3 heads x 3 row tiles, 8 mask types with window counts that leave partial
# schedule groups, so each CTA walks several groups and reloads the bias image
@pytest.mark.parametrize("n,ntypes", [(343, 8), (343, 1), (129, 3)])
def test_window_attention_tc_many_tiles(n, ntypes):
    got, ref, nc8, again = _case((7, 7, 7), n, 61, 3, 2, ntypes, seed=7 + ntypes)
    assert _rel(got, ref) < 4e-3
    assert _rel(got, nc8) < 4e-3
    assert torch.equal(got, again)
