"""Unit sweep of the tensor-core kernels other than the 3x3x3 convolution -- gemm_tc, conv_gather_tc and conv_cin1_tc -- at
every compiled N tile width, in every form, against float64 references of the same operation.

Operands are rounded to fp16 first (the kernels' storage type), the bias stays fp32, and every output element is held to a
bound derived from the arithmetic instead of a fraction of the tensor's maximum:

    |y - r| <= 2^-11 |r| + C_ACC 2^-24 A + 2^-24

r is the float64 result and A the same operation on |x| and |w| plus |b| (plus |res|), which bounds every partial sum the
fp32 accumulator holds.  2^-11 |r| is the final fp16 rounding (dropped for fp32 NCDHW outputs), 2^-24 the fp16 subnormal
spacing.  The {sum, sumsq} statistics of each (n, c) are held to the per-element bound (without the fp16 term) summed over
that (n, c); every case with statistics runs twice and must give the same bits.

Every output is a channel slice in the middle of a wider NC8 buffer (or a whole NCDHW tensor), and that buffer is a view
into a larger allocation filled with a sentinel: afterwards every element outside the slice still holds the sentinel's bits.
Input slices have NaN in the neighbouring channels and around their buffer, so a read outside the slice shows up as NaN.

The persistent loops are run in three regimes (total tiles <= SMs; tiles per statistics group < grid < total tiles; tiles
per group > grid, where CTAs cross group boundaries mid-walk), read against the device's SM count.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from monai_b200 import _kernels as K
from monai_b200 import _lib as L

DEV = "cuda"

# C_ACC: no case below runs more than MAX_K16_STEPS = 64 wgmma K16 steps into one accumulator (asserted per case).  A step
# adds 16 exact fp16 products to the fp32 accumulator and loses at most 2 fp32 ulps of a partial sum bounded by A (operand
# alignment and rounding: 2 * 2^-23 A = 4 * 2^-24 A), and the epilogue rounds at most four more values bounded by A (bias,
# GELU, residual, and the fp32 running statistics sums, which add at most 16 partial sums in sequence here): (64 + 4) * 4 =
# 272.  GELU is 1.13-Lipschitz and its polynomial erf (gelu.cuh) is off by at most 6e-6 |x| < 101 * 2^-24 A:
# 1.13 * 272 + 101 = 409.  512 leaves room for the accumulation order inside wgmma, which is not documented.
C_ACC = 512
MAX_K16_STEPS = 64
WIDTHS = (128, 96, 64, 48, 32, 16)            # compiled N tiles of gemm_tc and conv_gather_tc
_BITS = {torch.float16: torch.int16, torch.float32: torch.int32}
SENTINEL = {torch.float16: 0x7E5A, torch.float32: 0x7FC05A5A}   # NaN payloads that no kernel writes
NAN = {torch.float16: 0x7E00, torch.float32: 0x7FC00000}
WORST: dict[str, float] = {}                  # largest err / bound seen per kernel (printed at the end of the module)


# ---------------------------------------------------------------------------------------------- tiling, restated from csrc
def gemm_tc_nt(N):
    """gemm_tc.cu:31 gemm_tc_nt: width of the packed weight tiles P, the widest multiple of 16 up to 256 dividing N."""
    return next((nt for nt in range(256, 15, -16) if N % nt == 0), 16)


def gemm_tile_n(P):
    """gemm_tc.cu:38 gemm_tile_n: the kernel's N tile, the widest compiled width dividing P."""
    return next((nt for nt in WIDTHS if P % nt == 0), 16)


def cg_nt(cout_pad):
    """conv_gather_tc.cu:304 cg_nt: the widest compiled width dividing the padded Cout."""
    return next((nt for nt in WIDTHS if cout_pad % nt == 0), 16)


def cin1_tile(Cout):
    """conv_cin1_tc.cu:223 dispatch_cin1_tc: (NT, BD) per Cout; any other Cout is unsupported."""
    return {16: (16, 4), 32: (32, 4), 48: (48, 4), 64: (64, 4), 96: (96, 2), 128: (128, 2)}[Cout]


def _cdiv(a, b):
    return -(-a // b)


def regime(tiles_per_group, total_tiles, sms):
    """Persistent regime: i = one tile per CTA at most; ii = tiles per group < grid < total tiles; iii = tiles per group > grid
    (stats.cuh: R = min(tiles_per_group, grid) CTAs share a group, and a CTA's walk crosses from one group into the next)."""
    grid = min(total_tiles, sms)
    if total_tiles <= sms:
        return "i"
    if tiles_per_group < grid:
        return "ii"
    return "iii" if tiles_per_group > grid else "tiles per group == grid"


def gemm_tiles(Nb, S, N):
    """(tiles per (batch item, N tile) group, total tiles, N tiles) of gemm_tc (gemm_tc.cu:363)."""
    nt = gemm_tile_n(gemm_tc_nt(N))
    return _cdiv(S, 128), _cdiv(S, 128) * Nb * (N // nt), N // nt


def cg_out_sp(sp, form):
    k, s, p, t, op = form
    return tuple((i - 1) * s - 2 * p + k + op for i in sp) if t else tuple((i + 2 * p - k) // s + 1 for i in sp)


def cg_tiles(form, N, Cout, osp):
    """(tiles per group, total tiles) of conv_gather_tc (conv_gather_tc.cu:389): transposed convs run s^3 parity classes of
    ceil(out / s) coarse voxels each."""
    k, s, p, t, op = form
    coarse = math.prod(_cdiv(o, s) for o in osp) if t else math.prod(osp)
    tpg = (s**3 if t else 1) * _cdiv(coarse, 128)
    pad = _cdiv(Cout, 16) * 16
    return tpg, tpg * N * (pad // cg_nt(pad))


def cg_k16_steps(form, Cin):
    """wgmma K16 steps of the longest parity class: Cin / 16 per live tap."""
    k, s, p, t, op = form
    return Cin // 16 * (_cdiv(k, s) ** 3 if t else k**3)


def cin1_tiles(N, Cout, osp):
    """(tiles per group, total tiles) of conv_cin1_tc: 16 x 8 patches of BD planes (conv_epi.cuh:29)."""
    bd = cin1_tile(Cout)[1]
    tpg = _cdiv(osp[2], 8) * _cdiv(osp[1], 16) * _cdiv(osp[0], bd)
    return tpg, tpg * N


# ---------------------------------------------------------------------------------------------- case tables
# conv_gather_tc forms: (k, stride, pad, transposed, output_padding)
T321_OP1, T321_OP0 = (3, 2, 1, True, 1), (3, 2, 1, True, 0)
T220, T311, T120 = (2, 2, 0, True, 0), (3, 1, 1, True, 0), (1, 2, 0, True, 1)
CG_FORMS = [(3, 2, 1, False, 0), (1, 2, 0, False, 0), (2, 2, 0, False, 0), (3, 1, 1, False, 0), (1, 1, 0, False, 0),
            T321_OP0, T321_OP1, T220, T311, T120, (1, 2, 0, True, 0)]
# (form, N, Cin, Cout, input spatial, in_coff, out_coff, regime); T120 is ConvTranspose3d(k1, s2): no tap reaches the odd
# outputs, which are the bias alone
CG_CASES = [
    ((3, 2, 1, False, 0), 2, 16, 8, (7, 9, 11), 8, 8, "i"),
    ((3, 2, 1, False, 0), 2, 32, 320, (6, 5, 8), 0, 16, "i"),
    ((1, 2, 0, False, 0), 2, 32, 24, (5, 7, 9), 16, 8, "i"),
    ((1, 2, 0, False, 0), 2, 48, 256, (8, 6, 10), 8, 8, "i"),
    ((2, 2, 0, False, 0), 2, 16, 48, (5, 8, 9), 8, 24, "i"),
    ((2, 2, 0, False, 0), 3, 64, 96, (4, 6, 2), 0, 8, "i"),
    ((3, 1, 1, False, 0), 2, 16, 40, (1, 7, 9), 8, 8, "i"),
    ((3, 1, 1, False, 0), 2, 32, 16, (3, 5, 4), 24, 8, "i"),
    ((1, 1, 0, False, 0), 2, 64, 192, (3, 5, 7), 8, 8, "i"),
    ((1, 1, 0, False, 0), 2, 16, 128, (1, 1, 9), 0, 8, "i"),
    (T321_OP1, 2, 64, 64, (3, 4, 5), 8, 8, "i"),
    (T321_OP0, 2, 32, 32, (3, 4, 5), 0, 16, "i"),
    (T321_OP0, 2, 16, 8, (1, 2, 3), 8, 8, "i"),
    (T220, 2, 32, 24, (3, 2, 5), 8, 8, "i"),
    (T220, 2, 16, 256, (2, 3, 1), 0, 8, "i"),
    (T311, 2, 16, 40, (3, 4, 6), 16, 8, "i"),
    (T120, 2, 16, 16, (3, 4, 5), 8, 8, "i"),
    ((1, 2, 0, True, 0), 2, 32, 48, (2, 3, 4), 0, 8, "i"),
    (T120, 20, 16, 16, (3, 4, 5), 8, 8, "ii"),     # CTAs run a live class, then an empty one: stale accumulators would show
    ((1, 2, 0, False, 0), 2, 16, 192, (32, 32, 40), 8, 8, "ii"),
    (T321_OP1, 3, 16, 16, (8, 8, 34), 8, 8, "iii"),
]
# NCDHW outputs (the segmentation heads), each in fp16 and fp32: (form, N, Cin, Cout, input spatial, in_coff)
CG_HEADS = [(T321_OP1, 2, 16, 1, (3, 4, 5), 8), ((3, 1, 1, False, 0), 2, 16, 3, (4, 5, 6), 0), (T321_OP1, 2, 32, 14, (3, 4, 5), 8),
            (T321_OP1, 2, 16, 105, (2, 3, 4), 16)]
# gemm_tc mode 0: (Nb, S, K, N, bias, gelu, residual, stats, in_coff, out_coff, res_coff, regime)
GEMM_CASES = [
    (2, 1, 16, 16, True, False, False, True, 8, 8, 0, "i"),
    (2, 127, 48, 32, True, True, False, False, 0, 8, 0, "i"),
    (2, 128, 64, 48, False, False, True, True, 8, 16, 8, "i"),
    (2, 129, 80, 64, True, True, True, True, 16, 8, 8, "i"),
    (2, 300, 768, 96, True, False, False, True, 8, 8, 0, "i"),
    (2, 1000, 64, 128, False, True, False, False, 0, 8, 0, "i"),
    (2, 129, 48, 144, True, False, False, True, 8, 8, 0, "i"),
    (2, 200, 80, 160, False, False, True, True, 8, 16, 8, "i"),
    (2, 127, 16, 176, True, True, False, False, 8, 8, 0, "i"),
    (2, 257, 768, 256, True, False, True, False, 8, 8, 16, "i"),
    (2, 130, 64, 320, True, False, False, True, 0, 8, 0, "i"),
    (2, 129, 48, 384, True, True, False, True, 8, 8, 0, "i"),
    (2, 128 * 40, 64, 192, True, False, False, True, 8, 8, 0, "ii"),
    (3, 20000, 64, 48, True, False, True, True, 8, 8, 8, "iii"),
]
# gemm_tc mode 1 (row map): (Nb, S, S_out, mapped rows, K, N, gelu, regime); always bias, residual and statistics
GEMM_MAP_CASES = [(2, 300, 256, 200, 64, 96, False, "i"), (3, 343, 300, 250, 48, 48, True, "i")]
# gemm_tc mode 2 (ConvTranspose k2 s2): (Nb, (D, H, W), K, Cout, gelu, in_coff, out_coff, regime); N = 8 Cout
GEMM_UP_CASES = [(2, (3, 5, 7), 48, 48, True, 8, 8, "i"), (2, (1, 3, 5), 32, 16, False, 0, 16, "i"), (2, (3, 3, 5), 64, 24, True, 8, 8, "i")]
# conv_cin1_tc: every Cout x form x input dtype at odd sizes, plus the persistent regimes
CIN1_COUTS = [16, 32, 48, 64, 96, 128]
CIN1_FORMS = [(3, 1, 1), (2, 2, 0)]
CIN1_SP = {(3, 1, 1): (5, 9, 11), (2, 2, 0): (7, 9, 11)}
CIN1_REGIMES = [(2, 48, (20, 64, 32), "ii"), (3, 32, (24, 64, 48), "iii")]   # (N, Cout, input spatial, regime), (3, 1, 1)


# ---------------------------------------------------------------------------------------------- helpers
@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for k in sorted(WORST):
        print(f"\n[tc sweep] {k}: largest err / bound {WORST[k]:.3g}")


class Guarded:
    """`shape` elements of `dtype` inside a larger allocation filled with `bits`: 384 bytes before, 640 bytes after, so the view
    keeps the 128-byte alignment the bulk copies need."""

    def __init__(self, shape, dtype, bits):
        per = 128 // torch.empty((), dtype=dtype).element_size()
        self.shape, self.dtype, self.bits = tuple(shape), dtype, bits
        self.lead, self.n = 3 * per, math.prod(shape)
        self.alloc = torch.empty(self.lead + self.n + 5 * per, dtype=dtype, device=DEV)
        self.alloc.view(_BITS[dtype]).fill_(bits)
        self.view = self.alloc[self.lead: self.lead + self.n].view(self.shape)
        assert self.view.data_ptr() % 128 == 0

    def bits_tensor(self):
        return self.alloc.view(_BITS[self.dtype])

    def assert_untouched_outside(self, region, what):
        keep = torch.ones(self.alloc.numel(), dtype=torch.bool, device=DEV)
        keep[self.lead: self.lead + self.n].view(self.shape)[region] = False
        bad = (self.bits_tensor() != self.bits) & keep
        assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements outside the output were written"


def nc8_input(x, coff, extra=8):
    """x [N, C, *sp] fp16 (CPU) at channel coff of a guarded NC8 buffer with `extra` channels after it, NaN everywhere else."""
    N, C = x.shape[:2]
    sp = tuple(x.shape[2:])
    g = Guarded((N, (coff + C + extra) // 8, *sp, 8), torch.float16, NAN[torch.float16])
    g.view[:, coff // 8: (coff + C) // 8] = x.reshape(N, C // 8, 8, *sp).permute(0, 1, 3, 4, 5, 2).to(DEV)
    return g, K.NC8(N, coff + C + extra, sp, DEV, buf=g.view)


def nc8_output(N, C, coff, sp, extra=8):
    """guarded NC8 destination of coff + C + extra channels, sentinel everywhere"""
    g = Guarded((N, (coff + C + extra) // 8, *sp, 8), torch.float16, SENTINEL[torch.float16])
    return g, K.NC8(N, coff + C + extra, sp, DEV, buf=g.view)


def from_nc8(view, coff, C):
    """channels [coff, coff + C) of an NC8 view [N, ctot/8, D, H, W, 8] -> [N, C, D, H, W]"""
    v = view[:, coff // 8: (coff + C) // 8]
    return v.permute(0, 1, 5, 2, 3, 4).reshape(v.shape[0], C, *v.shape[2:5])


def check(kernel, what, got, r, A, fp16_out=True):
    got = got.to(r.device).double()
    assert bool(torch.isfinite(got).all()), f"{what}: {int((~torch.isfinite(got)).sum())} non-finite outputs"
    bound = C_ACC * 2.0**-24 * A + 2.0**-24
    if fp16_out:
        bound = bound + 2.0**-11 * r.abs()
    ratio = (got - r).abs() / bound
    worst = float(ratio.max())
    WORST[kernel] = max(WORST.get(kernel, 0.0), worst)
    at = tuple(int(i) for i in np.unravel_index(int(ratio.argmax()), tuple(ratio.shape)))
    assert worst <= 1.0, f"{what}: error {worst:.3g} x the bound at {at}: got {float(got[at])}, want {float(r[at])}"


def check_stats(kernel, what, st, r, A):
    """st [N*C, 2] {sum, sumsq}; r, A [N, C, M]: float64 values of the M elements the statistics of (n, c) cover"""
    e = C_ACC * 2.0**-24 * A + 2.0**-24
    s = st.to(r.device).double().reshape(r.shape[0], r.shape[1], 2)
    want_s, want_q = r.sum(-1), (r * r).sum(-1)
    tol_s = e.sum(-1) + 2.0**-24 * want_s.abs()                     # + the float32 rounding of the stored sum
    tol_q = (e * (2 * r.abs() + e)).sum(-1) + 2.0**-24 * want_q      # |f^2 - r^2| <= e (2 |r| + e)
    worst = max(float(((s[..., 0] - want_s).abs() / tol_s).max()), float(((s[..., 1] - want_q).abs() / tol_q).max()))
    WORST[kernel + " statistics"] = max(WORST.get(kernel + " statistics", 0.0), worst)
    assert worst <= 1.0, f"{what}: statistics error {worst:.3g} x the bound"


def assert_regime(name, tpg, total):
    sms = torch.cuda.get_device_properties(torch.device(DEV)).multi_processor_count
    got = regime(tpg, total, sms)
    assert got == name, f"a case for persistent regime {name} lands in {got} on {sms} SMs ({tpg} tiles per group, {total} tiles)"


def twice(launch):
    """launch() -> (Guarded output, stats), run twice: the first run and a check that the second gave the same bits (called
    after the value checks, so that a wrong value is reported as one)"""
    (g1, s1), (g2, s2) = launch(), launch()
    torch.cuda.synchronize()

    def same_bits():
        assert torch.equal(g1.bits_tensor(), g2.bits_tensor()), "outputs differ run to run"
        if s1 is not None:
            assert torch.equal(s1.view(torch.int32), s2.view(torch.int32)), "statistics differ run to run"

    return g1, s1, same_bits


# ---------------------------------------------------------------------------------------------- conv_gather_tc
def _conv_gather(form, N, Cin, Cout, sp, in_coff, out_coff, reg, ncdhw=None, seed=0):
    k, s, p, t, op = form
    assert cg_k16_steps(form, Cin) <= MAX_K16_STEPS
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((N, Cin, *sp), generator=g).half()
    w = (torch.randn((Cin, Cout, k, k, k) if t else (Cout, Cin, k, k, k), generator=g) / (Cin * k**3) ** 0.5).half()
    b = torch.randn(Cout, generator=g)
    osp = cg_out_sp(sp, form)
    assert_regime(reg, *cg_tiles(form, N, Cout, osp))

    def conv(a, ww, bb):
        if t:
            return F.conv_transpose3d(a, ww, bb, stride=s, padding=p, output_padding=op)
        return F.conv3d(a, ww, bb, stride=s, padding=p)

    r = conv(x.double(), w.double(), b.double())
    A = conv(x.double().abs(), w.double().abs(), b.double().abs())
    assert tuple(r.shape[2:]) == osp
    _, xin = nc8_input(x, in_coff)
    pw = K.conv_gather_tc_pack_weight(w.float().to(DEV), k, s, p, t)
    bd = b.to(DEV)

    def launch():
        if ncdhw is None:
            go, out = nc8_output(N, Cout, out_coff, osp)
        else:
            go = Guarded((N, Cout, *osp), ncdhw, SENTINEL[ncdhw])
            out = go.view
        _, st = K.conv_gather_tc(xin, pw, Cin, Cout, k, s, p, transposed=t, output_padding=op, in_coff=in_coff, bias=bd, out=out,
                                 out_coff=out_coff, ncdhw_dtype=ncdhw, want_stats=True)
        return go, st

    go, st, same_bits = twice(launch)
    what = f"conv_gather_tc {form} N={N} Cin={Cin} Cout={Cout} sp={sp}"
    if ncdhw is None:
        go.assert_untouched_outside((slice(None), slice(out_coff // 8, (out_coff + Cout) // 8)), what)
        got = from_nc8(go.view, out_coff, Cout)
    else:
        go.assert_untouched_outside((slice(None),), what)
        got = go.view
    check("conv_gather_tc", what, got.cpu(), r, A, fp16_out=ncdhw != torch.float32)
    check_stats("conv_gather_tc", what, st.cpu(), r.reshape(N, Cout, -1), A.reshape(N, Cout, -1))
    same_bits()


def _cg_id(c):
    return f"{'T' if c[0][3] else ''}k{c[0][0]}s{c[0][1]}p{c[0][2]}{'op' + str(c[0][4]) if c[0][3] else ''}-N{c[1]}-Cin{c[2]}-Cout{c[3]}-{'x'.join(map(str, c[4]))}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", CG_CASES, ids=_cg_id)
def test_conv_gather_tc(case):
    _conv_gather(*case, seed=len(CG_CASES) + case[3])


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32], ids=["f16", "f32"])
@pytest.mark.parametrize("case", CG_HEADS, ids=lambda c: f"Cout{c[3]}")
def test_conv_gather_tc_ncdhw(case, dtype):
    _conv_gather(*case, 0, "i", ncdhw=dtype, seed=case[3])


# ---------------------------------------------------------------------------------------------- gemm_tc
def _gemm_rows(Nb, S, Kd, N, bias, gelu, res, stats, in_coff, out_coff, res_coff, reg, S_out=None, mapped=0, seed=0):
    """mode 0 (S_out None) or mode 1: rows scattered through a row map with -1 entries into S_out < S destination rows"""
    mode = 0 if S_out is None else 1
    So = S if mode == 0 else S_out
    assert Kd // 16 <= MAX_K16_STEPS
    if stats:
        assert_regime(reg, *gemm_tiles(Nb, S, N)[:2])
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((Nb, Kd, 1, 1, S), generator=g).half()
    w = (torch.randn((N, Kd), generator=g) / Kd**0.5).half()
    b = torch.randn(N, generator=g) if bias else None
    rs = torch.randn((Nb, N, 1, 1, So), generator=g).half() if res else None
    rmap = None
    if mode == 1:
        src, dst = torch.randperm(S, generator=g)[:mapped], torch.randperm(So, generator=g)[:mapped]
        rmap = torch.full((S,), -1, dtype=torch.int32)
        rmap[src] = dst.int()
        src = src.sort().values
        dst = rmap[src].long()
    else:
        src = dst = torch.arange(S)
    # float64 reference: on the GPU for the large GEMMs
    rd = DEV if Nb * S * N * Kd > 2**26 else "cpu"
    x64, w64 = x.double().reshape(Nb, Kd, S).to(rd), w.double().to(rd)
    r = torch.einsum("nks,ok->nos", x64, w64)
    A = torch.einsum("nks,ok->nos", x64.abs(), w64.abs())
    if bias:
        r, A = r + b.double().to(rd)[None, :, None], A + b.double().abs().to(rd)[None, :, None]
    if gelu:
        r = F.gelu(r)
    r, A = r[:, :, src.to(rd)], A[:, :, src.to(rd)]
    if res:
        rr = rs.double().reshape(Nb, N, So).to(rd)[:, :, dst.to(rd)]
        r, A = r + rr, A + rr.abs()
    _, xin = nc8_input(x, in_coff)
    rin = nc8_input(rs, res_coff)[1] if res else None
    pw = K.gemm_tc_pack_weight(w.float().to(DEV))
    bd, md = (None if b is None else b.to(DEV)), (None if rmap is None else rmap.to(DEV))

    def launch():
        go, out = nc8_output(Nb, N, out_coff, (1, 1, So))
        _, st = K.gemm_tc(xin, pw, Kd, N, bias=bd, in_coff=in_coff, out=out, out_coff=out_coff, res=rin, res_coff=res_coff, row_map=md,
                          mode=mode, act=L.ACT_GELU if gelu else L.ACT_NONE, want_stats=stats)
        return go, st

    go, st, same_bits = twice(launch)
    what = f"gemm_tc mode {mode} Nb={Nb} S={S} K={Kd} N={N}"
    go.assert_untouched_outside((slice(None), slice(out_coff // 8, (out_coff + N) // 8), slice(None), slice(None), dst.to(DEV)), what)
    got = from_nc8(go.view, out_coff, N).reshape(Nb, N, So)[:, :, dst.to(DEV)]
    check("gemm_tc", what, got, r, A)
    if stats:
        check_stats("gemm_tc", what, st, r, A)
    same_bits()


def _gemm_id(c):
    flags = "".join(f for f, on in zip(("b", "g", "r", "s"), c[4:8]) if on)
    return f"Nb{c[0]}-S{c[1]}-K{c[2]}-N{c[3]}-{flags}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", GEMM_CASES, ids=_gemm_id)
def test_gemm_tc(case):
    _gemm_rows(*case, seed=case[3] + case[2])


@pytest.mark.gpu
@pytest.mark.parametrize("case", GEMM_MAP_CASES, ids=lambda c: f"S{c[1]}-Sout{c[2]}-N{c[5]}")
def test_gemm_tc_row_map(case):
    """Swin's window-reverse projection: rows scattered to a destination through an index table; unmapped destination rows
    stay untouched, the residual is read at the destination row and the statistics cover the mapped rows only"""
    Nb, S, So, mapped, Kd, N, gelu, reg = case
    _gemm_rows(Nb, S, Kd, N, True, gelu, True, True, 8, 8, 8, reg, S_out=So, mapped=mapped, seed=S)


@pytest.mark.gpu
@pytest.mark.parametrize("case", GEMM_UP_CASES, ids=lambda c: f"{'x'.join(map(str, c[1]))}-K{c[2]}-Cout{c[3]}")
def test_gemm_tc_upsample_scatter(case):
    """ConvTranspose3d(k2, s2) as one GEMM with columns [tap][cout] scattered into a concat slice of the 2x volume; the
    statistics are per GEMM column"""
    Nb, sp, Kd, Cout, gelu, in_coff, out_coff, reg = case
    N, S = 8 * Cout, math.prod(sp)
    assert Kd // 16 <= MAX_K16_STEPS
    assert_regime(reg, *gemm_tiles(Nb, S, N)[:2])
    g = torch.Generator().manual_seed(Cout)
    x = torch.randn((Nb, Kd, *sp), generator=g).half()
    wt = (torch.randn((Kd, Cout, 2, 2, 2), generator=g) / Kd**0.5).half()
    b = torch.randn(Cout, generator=g)
    wg = wt.double().permute(2, 3, 4, 1, 0).reshape(N, Kd)          # GEMM column = tap * Cout + cout
    act = F.gelu if gelu else (lambda v: v)
    r = act(F.conv_transpose3d(x.double(), wt.double(), b.double(), stride=2))
    A = F.conv_transpose3d(x.double().abs(), wt.double().abs(), b.double().abs(), stride=2)
    xs = x.double().reshape(Nb, Kd, S)
    rg = act(torch.einsum("nks,ok->nos", xs, wg) + b.double().repeat(8)[None, :, None])
    ag = torch.einsum("nks,ok->nos", xs.abs(), wg.abs()) + b.double().abs().repeat(8)[None, :, None]
    _, xin = nc8_input(x, in_coff)
    pw = K.gemm_tc_pack_weight(wg.float().to(DEV))
    osp = tuple(2 * v for v in sp)

    def launch():
        go, out = nc8_output(Nb, Cout, out_coff, osp)
        _, st = K.gemm_tc(xin, pw, Kd, N, bias=b.to(DEV), in_coff=in_coff, out=out, out_coff=out_coff, mode=2,
                          act=L.ACT_GELU if gelu else L.ACT_NONE, want_stats=True)
        return go, st

    go, st, same_bits = twice(launch)
    what = f"gemm_tc mode 2 sp={sp} K={Kd} Cout={Cout}"
    go.assert_untouched_outside((slice(None), slice(out_coff // 8, (out_coff + Cout) // 8)), what)
    check("gemm_tc", what, from_nc8(go.view, out_coff, Cout).cpu(), r, A)
    check_stats("gemm_tc", what, st.cpu(), rg, ag)
    same_bits()


# ---------------------------------------------------------------------------------------------- conv_cin1_tc
def _cin1_launch(name, x, w, b, form, out_coff, want_stats=True):
    """b200_conv_cin1_tc (wgmma) or b200_conv_cin1_nc8 (CUDA cores) called directly, into a guarded channel slice"""
    k, s, p = form
    N, _, D, H, W = x.shape
    Cout = w.shape[0]
    osp = tuple((v + 2 * p - k) // s + 1 for v in (D, H, W))
    go, out = nc8_output(N, Cout, out_coff, osp)
    st = torch.empty((N * Cout, 2), device=DEV, dtype=torch.float32)
    ws = K._ws(getattr(L.load(), f"b200_{name}_workspace_bytes")(N, D, H, W, Cout, k, s, p), DEV)
    K._call(name, L.ptr(x), L.dt(x), N, D, H, W, L.ptr(w), L.ptr(b), Cout, k, s, p, L.ptr(out.buf), out.C, out_coff, L.ptr(st), L.ptr(ws),
            L.stream_ptr(torch.device(DEV)))
    return go, st


def _cin1(N, Cout, form, dtype, sp, out_coff, reg, seed):
    k, s, p = form
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((N, 1, *sp), generator=g).half()               # fp16 values, given to the kernels in `dtype`
    w = (torch.randn((Cout, 1, k, k, k), generator=g) / k**1.5).half().float()
    b = torch.randn(Cout, generator=g)
    r = F.conv3d(x.double(), w.double(), b.double(), stride=s, padding=p)
    A = F.conv3d(x.double().abs(), w.double().abs(), b.double().abs(), stride=s, padding=p)
    osp = tuple(r.shape[2:])
    assert_regime(reg, *cin1_tiles(N, Cout, osp))
    xd, wd, bd = x.to(dtype).to(DEV), w.to(DEV), b.to(DEV)
    for name in ("conv_cin1_tc", "conv_cin1_nc8"):
        go, st, same_bits = twice(lambda: _cin1_launch(name, xd, wd, bd, form, out_coff))
        what = f"{name} {form} {dtype} N={N} Cout={Cout} sp={sp}"
        go.assert_untouched_outside((slice(None), slice(out_coff // 8, (out_coff + Cout) // 8)), what)
        check(name, what, from_nc8(go.view, out_coff, Cout).cpu(), r, A)
        check_stats(name, what, st.cpu(), r.reshape(N, Cout, -1), A.reshape(N, Cout, -1))
        same_bits()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32], ids=["f16", "f32"])
@pytest.mark.parametrize("form", CIN1_FORMS, ids=lambda f: "k%ds%dp%d" % f)
@pytest.mark.parametrize("Cout", CIN1_COUTS)
def test_conv_cin1_tc(Cout, form, dtype):
    """every instantiation of the single-channel stem, with a bias, into a channel slice, at odd sizes; the CUDA-core stem on
    the same inputs"""
    _cin1(2, Cout, form, dtype, CIN1_SP[form], 8 if Cout % 16 else 16, "i", seed=Cout)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CIN1_REGIMES, ids=lambda c: f"regime-{c[3]}")
def test_conv_cin1_tc_persistent(case):
    N, Cout, sp, reg = case
    _cin1(N, Cout, (3, 1, 1), torch.float16, sp, 8, reg, seed=N)


# ---------------------------------------------------------------------------------------------- coverage (no GPU)
def test_case_tables_reach_every_instantiation():
    """The tables above reach every compiled N tile, every mode and form, both tile orders of gemm_tc (gemm_tc.cu:81 gemm_tile:
    N tile fastest without statistics, row tile fastest with them) and every persistent regime with statistics."""
    # gemm_tc
    rows = [(c[0], c[1], c[2], c[3], c[7], c[11]) for c in GEMM_CASES]
    rows += [(c[0], c[1], c[4], c[5], True, c[7]) for c in GEMM_MAP_CASES]
    rows += [(c[0], math.prod(c[1]), c[2], 8 * c[3], True, c[7]) for c in GEMM_UP_CASES]
    assert {gemm_tile_n(gemm_tc_nt(r[3])) for r in rows} == set(WIDTHS)
    assert any(gemm_tc_nt(r[3]) != gemm_tile_n(gemm_tc_nt(r[3])) for r in rows if r[4])        # P != NT, with statistics
    assert {r[3] for r in rows} >= {16, 32, 48, 64, 96, 128, 144, 160, 176, 192, 256, 320, 384}
    assert {r[2] for r in rows} >= {16, 48, 64, 80, 768}
    assert {r[1] for r in rows} >= {1, 127, 128, 129} and max(r[1] for r in rows) > 128 * 132
    assert any(r[4] and gemm_tiles(r[0], r[1], r[3])[2] > 1 for r in rows)                    # row-tile-fastest order
    assert any(not r[4] and gemm_tiles(r[0], r[1], r[3])[2] > 1 for r in rows)                # N-tile-fastest order
    assert {r[5] for r in rows if r[4]} == {"i", "ii", "iii"}
    assert all(r[0] >= 3 for r in rows if r[5] == "iii")
    assert GEMM_MAP_CASES and GEMM_UP_CASES
    assert all(c[2] < c[1] and c[3] < c[2] for c in GEMM_MAP_CASES)                            # -1 entries, unreached rows
    assert any(c[5] for c in GEMM_CASES) and any(c[6] for c in GEMM_CASES) and any(c[4] and c[5] and c[6] for c in GEMM_CASES)
    assert any(c[4] for c in GEMM_UP_CASES) and any(v % 2 for c in GEMM_UP_CASES for v in c[1])
    # conv_gather_tc
    allcg = CG_CASES + [(c[0], c[1], c[2], c[3], c[4], c[5], 0, "i") for c in CG_HEADS]
    pads = [_cdiv(c[3], 16) * 16 for c in allcg]
    assert {cg_nt(p) for p in pads} == set(WIDTHS)
    assert {c[3] for c in CG_CASES} >= {8, 16, 24, 32, 40, 48, 64, 96, 128, 192, 256, 320}
    assert any(c[3] % 16 for c in CG_CASES)                                                    # a zero-padded N tile
    assert {c[0] for c in CG_CASES} == set(CG_FORMS)
    assert any(f[3] and f[0] < f[1] for f in CG_FORMS)                                         # parity classes without taps
    assert {c[3] for c in CG_HEADS} == {1, 3, 14, 105}
    assert any(c[5] for c in CG_CASES) and any(c[5] for c in CG_HEADS)                         # input channel slices
    assert any(1 in c[4] for c in CG_CASES) and any(1 in cg_out_sp(c[4], c[0]) for c in CG_CASES)            # size-1 axes
    assert all(any(v % 2 for v in c[4] + cg_out_sp(c[4], c[0])) for c in CG_CASES if c[7] == "i")            # odd axes
    assert {c[7] for c in CG_CASES} == {"i", "ii", "iii"}
    assert all(c[1] >= 3 for c in CG_CASES if c[7] == "iii")
    assert all(cg_k16_steps(c[0], c[2]) <= MAX_K16_STEPS for c in allcg)
    # conv_cin1_tc: all 6 Cout x 2 forms x 2 input dtypes (test_conv_cin1_tc's parameters), both depth blocks
    assert sorted(CIN1_COUTS) == sorted([16, 32, 48, 64, 96, 128]) and sorted(CIN1_FORMS) == [(2, 2, 0), (3, 1, 1)]
    assert {cin1_tile(c)[1] for c in CIN1_COUTS} == {2, 4}
    assert all(any(v % 2 for v in CIN1_SP[f]) for f in CIN1_FORMS)
    assert {c[3] for c in CIN1_REGIMES} == {"ii", "iii"} and all(c[0] >= 3 for c in CIN1_REGIMES if c[3] == "iii")
