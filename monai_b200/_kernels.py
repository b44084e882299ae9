"""Tensor-level wrappers around the C ABI (include/monai_b200.h).

PyTorch only supplies device memory and the current stream here; every computation below is a hand-written
sm_90a kernel reached through ctypes.  All functions require CUDA tensors.
"""
from __future__ import annotations

import ctypes as C
import weakref
from typing import Sequence

import torch

from . import _lib as L


class _Prof:
    on = False
    events: list = []


def profile_start() -> None:
    """Record a CUDA-event pair around every C-ABI launch until profile_stop() (used by bench.py for the roofline)."""
    _Prof.on, _Prof.events = True, []


def profile_stop(by_shape: bool = False) -> dict:
    """Totals per entry point; with `by_shape` launches are further split by their (flops, bytes) signature."""
    torch.cuda.synchronize()
    _Prof.on = False
    out: dict = {}
    for name, e0, e1, flops, nbytes in _Prof.events:
        if by_shape:
            name = f"{name} [{flops / 1e9:.2f} GF, {nbytes / 1e6:.1f} MB]"
        d = out.setdefault(name, {"ms": 0.0, "n": 0, "flops": 0.0, "bytes": 0.0})
        d["ms"] += e0.elapsed_time(e1)
        d["n"] += 1
        d["flops"] += flops
        d["bytes"] += nbytes
    _Prof.events = []
    return out


def _call(name: str, *args, flops: float = 0.0, nbytes: float = 0.0) -> None:
    """Launch one C-ABI entry point (b200_<name>) and raise on a non-zero status.  The launch runs with the device of the
    stream handle among `args` current (see _lib.stream_ptr), so tensors on a non-current GPU work."""
    fn = getattr(L.load(), "b200_" + name)
    dev = L.take_stream_device()   # the device whose stream handle is among `args`
    if dev is not None and dev.index is not None and dev.index != torch.cuda.current_device():
        with torch.cuda.device(dev):   # kernels, tensor maps and events belong to the tensors' device, not to the current one
            return _call_on(fn, name, args, flops, nbytes)
    return _call_on(fn, name, args, flops, nbytes)


def _call_on(fn, name, args, flops, nbytes) -> None:
    if _Prof.on:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = fn(*args)
        e1.record()
        _Prof.events.append((name, e0, e1, flops, nbytes))
    else:
        rc = fn(*args)
    L.check(rc, name)


_F32_CACHE: dict = {}


def _f32c(t: torch.Tensor | None) -> torch.Tensor | None:
    """float32 contiguous view of a (parameter) tensor, cached so fp16 models do not re-convert their weights on every
    forward.  An entry is tied to the IDENTITY of its source tensor (weak reference + version counter): when a model is
    freed and another one lands on the same addresses, the stale entry is neither hit (the weak reference is dead or
    points elsewhere) nor kept (its finaliser evicts it)."""
    if t is None:
        return None
    src = t
    t = t.detach()
    if t.dtype == torch.float32 and t.is_contiguous():
        return t
    key = (id(src), tuple(t.shape), t.dtype, t.device)
    hit = _F32_CACHE.get(key)
    if hit is not None and hit[0]() is src and hit[1] == src._version and hit[2] == src.data_ptr():
        return hit[3]
    val = t.to(torch.float32).contiguous()
    try:
        ref = weakref.ref(src, lambda _r, k=key: _F32_CACHE.pop(k, None))
    except TypeError:   # pragma: no cover - objects without weak references are not cached
        return val
    _F32_CACHE[key] = (ref, src._version, src.data_ptr(), val)
    return val


def _ws(nbytes: int, device) -> torch.Tensor | None:
    """Scratch for the deterministic statistics of the tensor-core epilogues (include/monai_b200.h): a fresh allocation per
    call, so CUDA-graph capture keeps it alive inside the graph's pool."""
    if nbytes < 0:
        raise ValueError("monai_b200: workspace query failed for this shape")
    return torch.empty(max(int(nbytes), 16), device=device, dtype=torch.uint8)


def _nb(*tensors) -> float:
    return float(sum(t.numel() * t.element_size() for t in tensors if t is not None))


def _t3(v) -> tuple[int, int, int]:
    if isinstance(v, int):
        return (v, v, v)
    v = tuple(int(i) for i in v)
    if len(v) != 3:
        raise ValueError(f"expected 3 values, got {v}")
    return v  # type: ignore[return-value]


# ------------------------------------------------------------------------------------------- convolution (direct)
def conv_out_shape(in_sp, k, s, p, transposed=False, output_padding=(0, 0, 0)):
    if transposed:
        return tuple((i - 1) * st - 2 * pd + kk + op for i, kk, st, pd, op in zip(in_sp, k, s, p, output_padding))
    return tuple((i + 2 * pd - kk) // st + 1 for i, kk, st, pd in zip(in_sp, k, s, p))


def conv3d_direct(
    x: torch.Tensor,
    weight: torch.Tensor,
    bias: torch.Tensor | None = None,
    stride=1,
    padding=0,
    transposed: bool = False,
    output_padding=0,
    out: torch.Tensor | None = None,
    out_dtype: torch.dtype | None = None,
) -> torch.Tensor:
    """Conv3d / ConvTranspose3d (groups=1, dilation=1) with fp32 accumulation.  x: [N,Cin,D,H,W] contiguous per sample
    (a channel slice of a larger buffer is allowed); `out` may be a channel slice of a concat buffer."""
    L.require_cuda(x, weight)
    lib = L.load()
    s, p, op = _t3(stride), _t3(padding), _t3(output_padding)
    N, Cin, Di, Hi, Wi = x.shape
    k = tuple(weight.shape[2:])
    Cout = weight.shape[1] if transposed else weight.shape[0]
    wc = weight.shape[0] if transposed else weight.shape[1]
    if wc != Cin:
        raise ValueError(f"weight expects {wc} input channels, input has {Cin}")
    Do, Ho, Wo = conv_out_shape((Di, Hi, Wi), k, s, p, transposed, op)
    if out is None:
        out = torch.empty((N, Cout, Do, Ho, Wo), device=x.device, dtype=out_dtype or x.dtype)
    if tuple(out.shape) != (N, Cout, Do, Ho, Wo):
        raise ValueError(f"out has shape {tuple(out.shape)}, expected {(N, Cout, Do, Ho, Wo)}")
    for t, nm in ((x, "x"), (out, "out")):
        if not t[0].is_contiguous():
            raise ValueError(f"{nm} must be contiguous within each sample")
    w32 = _f32c(weight)
    b32 = _f32c(bias)
    d = L.ConvDesc(
        N, Cin, Cout, Di, Hi, Wi, Do, Ho, Wo, k[0], k[1], k[2], s[0], s[1], s[2], p[0], p[1], p[2], int(transposed),
        L.dt(x), L.dt(out), x.stride(0) if N > 1 else Cin * Di * Hi * Wi, out.stride(0) if N > 1 else Cout * Do * Ho * Wo,
    )
    taps = k[0] * k[1] * k[2]
    macs = float(N) * (Di * Hi * Wi if transposed else Do * Ho * Wo) * Cin * Cout * taps
    _call("conv3d_direct", C.byref(d), L.ptr(x), L.ptr(w32), L.ptr(b32), L.ptr(out), L.stream_ptr(x.device),
          flops=2.0 * macs, nbytes=_nb(x, out, w32))
    return out


# ---------------------------------------------------------------------------------------------- norm / activation
def instnorm_stats(x: torch.Tensor) -> torch.Tensor:
    """Per-(n,c) {sum, sumsq} of x[N,C,*spatial] -> float32 [N*C, 2]."""
    L.require_cuda(x)
    N, Cc = x.shape[:2]
    S = x[0, 0].numel()
    stats = torch.empty((N * Cc, 2), device=x.device, dtype=torch.float32)
    nws = L.load().b200_instnorm_stats_workspace_bytes(N, Cc, S)
    ws = _ws(nws, x.device) if nws > 0 else None
    _call("instnorm_stats", L.ptr(x), L.dt(x), N, Cc, S, x.stride(0) if N > 1 else Cc * S, L.ptr(stats), L.ptr(ws), L.stream_ptr(x.device), nbytes=_nb(x))
    return stats


def norm_act(
    x: torch.Tensor,
    stats: torch.Tensor | None = None,
    eps: float = 1e-5,
    gamma: torch.Tensor | None = None,
    beta: torch.Tensor | None = None,
    res: torch.Tensor | None = None,
    res_stats: torch.Tensor | None = None,
    act: int = L.ACT_NONE,
    slope: float = 0.0,
    slope_t: torch.Tensor | None = None,
    out: torch.Tensor | None = None,
) -> torch.Tensor:
    L.require_cuda(x)
    N, Cc = x.shape[:2]
    S = x[0, 0].numel()
    if out is None:
        out = torch.empty_like(x)
    g, b, sl = _f32c(gamma), _f32c(beta), _f32c(slope_t)
    _call("norm_act", L.ptr(x), L.dt(x), N, Cc, S, x.stride(0) if N > 1 else Cc * S, L.ptr(stats), eps, L.ptr(g), L.ptr(b), L.ptr(res),
            (res.stride(0) if N > 1 else Cc * S) if res is not None else 0, L.ptr(res_stats), act, float(slope), L.ptr(sl),
            0 if sl is None else sl.numel(), L.ptr(out), out.stride(0) if N > 1 else Cc * S, L.stream_ptr(x.device))
    return out


def layernorm_cf(x: torch.Tensor, gamma: torch.Tensor | None, beta: torch.Tensor | None, eps: float = 1e-5) -> torch.Tensor:
    """nn.LayerNorm over the channel axis of channels-first tokens x[N, C, S]."""
    L.require_cuda(x)
    x = x.contiguous()
    N, Cc, S = x.shape
    out = torch.empty_like(x)
    _call("layernorm_cf", L.ptr(x), L.dt(x), N, Cc, S, L.ptr(_f32c(gamma)), L.ptr(_f32c(beta)), float(eps), L.ptr(out), L.stream_ptr(x.device), nbytes=_nb(x, out))
    return out


def patchify(x: torch.Tensor, patch: Sequence[int]) -> torch.Tensor:
    """x [N, C, D, H, W] -> [N, C*pd*ph*pw, n_patches]: non-overlapping patches flattened into the channel axis."""
    L.require_cuda(x)
    x = x.contiguous()
    N, Cc, D, H, W = x.shape
    pd, ph, pw = (int(v) for v in patch)
    out = torch.empty((N, Cc * pd * ph * pw, (D // pd) * (H // ph) * (W // pw)), device=x.device, dtype=x.dtype)
    _call("patchify", L.ptr(x), L.dt(x), N, Cc, D, H, W, pd, ph, pw, L.ptr(out), L.stream_ptr(x.device), nbytes=_nb(x, out))
    return out


def mhsa_cf(qkv: torch.Tensor, heads: int, dim_head: int, scale: float, win: int = 0, bias: torch.Tensor | None = None,
            region: torch.Tensor | None = None) -> torch.Tensor:
    """softmax(q k^T * scale [+ bias] [+ shift mask]) v per head; qkv [N, 3*heads*dim_head, S] with channels (q|k|v, head, dim) ->
    [N, heads*dim_head, S].  win > 0: S holds windows of `win` tokens, bias float32 [heads, win, win], region int32 [S // win, win]."""
    L.require_cuda(qkv)
    qkv = qkv.contiguous()
    N, C3, S = qkv.shape
    if C3 != 3 * heads * dim_head:
        raise ValueError(f"mhsa_cf: {C3} channels for {heads} heads of {dim_head}")
    if bias is not None and (bias.dtype != torch.float32 or tuple(bias.shape) != (heads, win, win) or not bias.is_contiguous()):
        raise ValueError("mhsa_cf: bias must be a contiguous float32 [heads, win, win] tensor")
    if region is not None and (region.dtype != torch.int32 or region.numel() != S or not region.is_contiguous()):
        raise ValueError("mhsa_cf: region must be a contiguous int32 tensor with one label per token")
    out = torch.empty((N, heads * dim_head, S), device=qkv.device, dtype=qkv.dtype)
    keys = win if win > 0 else S
    _call("mhsa_cf", L.ptr(qkv), L.dt(qkv), N, heads, dim_head, S, float(scale), int(win), L.ptr(bias), L.ptr(region), L.ptr(out), L.stream_ptr(qkv.device),
          flops=4.0 * N * heads * S * keys * dim_head, nbytes=_nb(qkv, out))
    return out


def gather_cf(x: torch.Tensor, src: torch.Tensor, s_out: int | None = None) -> torch.Tensor:
    """y[n, c, r] = x[n, c, src[r]] (zeros where src[r] < 0) on channels-first tokens x[N, C, S]; src int32 on the device."""
    L.require_cuda(x, src)
    x = x.contiguous()
    N, Cc, S = x.shape
    s_out = int(src.numel()) if s_out is None else int(s_out)
    out = torch.empty((N, Cc, s_out), device=x.device, dtype=x.dtype)
    _call("gather_cf", L.ptr(x), L.dt(x), N, Cc, S, L.ptr(src), s_out, L.ptr(out), L.stream_ptr(x.device), nbytes=_nb(x, out))
    return out


def maxpool3d_2(x: torch.Tensor) -> torch.Tensor:
    L.require_cuda(x)
    N, Cc, D, H, W = x.shape
    x = x.contiguous()
    y = torch.empty((N, Cc, D // 2, H // 2, W // 2), device=x.device, dtype=x.dtype)
    _call("maxpool3d_2", L.ptr(x), L.dt(x), N * Cc, D, H, W, L.ptr(y), L.stream_ptr(x.device))
    return y


def copy_channels(x: torch.Tensor, dst: torch.Tensor, c_off: int) -> None:
    """dst[:, c_off:c_off+C] = replicate_pad(x) (dst spatial >= x spatial, padding on the high side only)."""
    L.require_cuda(x, dst)
    x = x.contiguous()
    N, Cc, Di, Hi, Wi = x.shape
    _, Ct, Do, Ho, Wo = dst.shape
    if not dst.is_contiguous():
        raise ValueError("dst must be contiguous")
    _call("copy_channels", L.ptr(x), L.dt(x), N, Cc, Di, Hi, Wi, L.ptr(dst), Ct, c_off, Do, Ho, Wo, L.stream_ptr(x.device))


# ------------------------------------------------------------------------------------------------ sliding window
def sw_gather(vol: torch.Tensor, win_tab: torch.Tensor, roi: Sequence[int], out_dtype: torch.dtype | None = None, w_align: int = 1) -> torch.Tensor:
    """vol [B,C,D,H,W] -> [n_win,C,*roi]; win_tab int32 device [n_win,4] = (batch, d0, h0, w0); `w_align` = a common divisor of every
    w0 (the caller knows the starts on the host), which lets the copy use 16-byte vectors."""
    L.require_cuda(vol, win_tab)
    vol = vol.contiguous()
    B, Cc, D, H, W = vol.shape
    n = win_tab.shape[0]
    out = torch.empty((n, Cc, *roi), device=vol.device, dtype=out_dtype or vol.dtype)
    _call("sw_gather", L.ptr(vol), L.dt(vol), L.ptr(out), L.dt(out), L.ptr(win_tab), n, Cc, D, H, W, roi[0], roi[1], roi[2], int(w_align),
          L.stream_ptr(vol.device), nbytes=2.0 * _nb(out))
    return out


def sw_blend(
    mode: int,
    preds: torch.Tensor | None,
    win_begin: int,
    win_end: int,
    vol_shape: Sequence[int],
    roi: Sequence[int],
    starts: Sequence[torch.Tensor],
    g: Sequence[torch.Tensor] | None,
    clamp_min: float,
    wmap: torch.Tensor | None,
    out: torch.Tensor,
    acc: torch.Tensor | None = None,
    box: Sequence[int] = (0, 0, 0, 0),
    slot_map: torch.Tensor | None = None,
    n_slots: int = 0,
    resample: "tuple | None" = None,
) -> None:
    """`resample` = (mat12, (oD, oH, oW), interp, pad) selects the fused blend + affine resample (see include/monai_b200.h)."""
    d = L.BlendDesc()
    B, Cc, D, H, W = vol_shape
    if preds is not None:
        L.require_cuda(preds)
        d.preds, d.pred_dtype = L.ptr(preds), L.dt(preds)
        st = preds.stride()
        for i in range(5):
            d.pred_stride[i] = st[i]
    d.win_begin, d.win_end = win_begin, win_end
    d.B, d.C, d.D, d.H, d.W = B, Cc, D, H, W
    d.rd, d.rh, d.rw = roi
    d.starts_d, d.nd = L.ptr(starts[0]), starts[0].numel()
    d.starts_h, d.nh = L.ptr(starts[1]), starts[1].numel()
    d.starts_w, d.nw = L.ptr(starts[2]), starts[2].numel()
    if g is not None:
        d.gd, d.gh, d.gw = L.ptr(g[0]), L.ptr(g[1]), L.ptr(g[2])
    d.clamp_min = clamp_min
    d.wmap = L.ptr(wmap)
    d.out, d.out_dtype = L.ptr(out), L.dt(out)
    d.acc = L.ptr(acc)
    for i in range(4):
        d.box[i] = box[i]
    d.starts_w_align = int(getattr(starts[2], "_align", 1))
    d.max_cover = int(getattr(starts[2], "_max_cover", 0))
    d.slot_map, d.n_slots = L.ptr(slot_map), int(n_slots)
    keep = None
    if resample is not None:
        mat, oshape, interp, pad = resample
        keep = (C.c_double * 12)(*[float(v) for v in mat])
        d.resample = C.cast(keep, C.POINTER(C.c_double))
        d.out_D, d.out_H, d.out_W = (int(v) for v in oshape)
        d.resample_interp, d.resample_pad = int(interp), int(pad)
    nb = _nb(preds) + (_nb(out) if mode == 0 else 0.0) + (2.0 * _nb(out) if mode == 1 else 0.0) + (_nb(out, acc) if mode == 2 else 0.0)
    _call("sw_blend", C.byref(d), mode, L.stream_ptr(out.device), nbytes=nb)


# ---------------------------------------------------------------------------------------------------- transforms
def resample_affine(
    src: torch.Tensor, out_shape: Sequence[int], mat: "Sequence[float]", interp: int, pad: int, align_corners: bool,
    out_dtype: torch.dtype = torch.float32,
) -> torch.Tensor:
    """src [C,D,H,W]; mat = 12 doubles (3x4 row-major) mapping output voxel index -> source voxel index."""
    L.require_cuda(src)
    src = src.contiguous()
    Cc, Di, Hi, Wi = src.shape
    dst = torch.empty((Cc, *out_shape), device=src.device, dtype=out_dtype)
    m = (C.c_double * 12)(*[float(v) for v in mat])
    _call("resample_affine", L.ptr(src), L.dt(src), Cc, Di, Hi, Wi, L.ptr(dst), L.dt(dst), out_shape[0], out_shape[1], out_shape[2], m, interp, pad, int(bool(align_corners)), L.stream_ptr(src.device),
          nbytes=_nb(src, dst))
    return dst


BOUNDS = {"replicate": 0, "nearest": 0, "border": 0, "dct1": 1, "mirror": 1, "dct2": 2, "reflect": 2, "dst1": 3, "antimirror": 3,
          "dst2": 4, "antireflect": 4, "dft": 5, "wrap": 5, "zero": 7, "zeros": 7}
ORDERS = {"nearest": 0, "linear": 1, "quadratic": 2, "cubic": 3, "fourth": 4, "fifth": 5, "sixth": 6, "seventh": 7}


def grid_pull(src: torch.Tensor, grid: torch.Tensor, bound: Sequence[int], order: Sequence[int], extrapolate: bool = True,
              channel_last: bool = True, scale: Sequence[float] | None = None, shift: Sequence[float] | None = None,
              half_even: bool = False, out_dtype: torch.dtype | None = None) -> torch.Tensor:
    """src [B,C,X,Y,Z]; grid [B,Xo,Yo,Zo,3] (channel_last) or [>=3,Xo,Yo,Zo] shared by the batch (channel first), float32 /
    float64, voxel coordinates after the per-axis `scale` / `shift`.  See b200_grid_pull."""
    L.require_cuda(src, grid)
    src = src.contiguous()
    grid = grid.contiguous()
    if grid.dtype not in (torch.float32, torch.float64):
        grid = grid.float()
    Bn, Cc, X, Y, Z = src.shape
    if channel_last:
        _, Xo, Yo, Zo, ncomp = grid.shape
        if ncomp != 3 or grid.shape[0] != Bn:
            raise ValueError(f"grid must be [B, Xo, Yo, Zo, 3] with B = {Bn}, got {tuple(grid.shape)}")
        sb, sc, sv = Xo * Yo * Zo * 3, 1, 3
    else:
        ncomp, Xo, Yo, Zo = grid.shape
        if ncomp < 3:
            raise ValueError(f"channel-first grid needs at least 3 coordinate rows, got {tuple(grid.shape)}")
        sb, sc, sv = 0, Xo * Yo * Zo, 1
    out = torch.empty((Bn, Cc, Xo, Yo, Zo), device=src.device, dtype=out_dtype or (src.dtype if src.dtype in (torch.float16, torch.float32) else torch.float32))
    dbl3 = C.c_double * 3
    int3 = C.c_int * 3
    sc3 = dbl3(*[float(v) for v in scale]) if scale is not None else None
    sh3 = dbl3(*[float(v) for v in shift]) if shift is not None else None
    _call("grid_pull", L.ptr(src), L.dt(src), Bn, Cc, X, Y, Z, L.ptr(grid), 2 if grid.dtype == torch.float64 else 0, sb, sc, sv, Xo, Yo, Zo,
          sc3, sh3, int3(*[int(b) for b in bound]), int3(*[int(o) for o in order]), int(bool(extrapolate)), int(bool(half_even)),
          L.ptr(out), L.dt(out), L.stream_ptr(src.device), nbytes=_nb(src, out) + 3.0 * Xo * Yo * Zo * grid.element_size() * (Bn if channel_last else 1))
    return out


def grid_push(inp: torch.Tensor | None, grid: torch.Tensor, shape: Sequence[int], bound: Sequence[int], order: Sequence[int],
              extrapolate: bool = True) -> torch.Tensor:
    """The adjoint of grid_pull: inp [B,C,Xi,Yi,Zi] (None = grid_count, the splat of ones) is scattered to out [B,C,*shape] (float32)
    at the voxel coordinates grid [B,Xi,Yi,Zi,3].  See b200_grid_push."""
    L.require_cuda(grid) if inp is None else L.require_cuda(inp, grid)
    grid = grid.contiguous()
    if grid.dtype not in (torch.float32, torch.float64):
        grid = grid.float()
    Bn, Xi, Yi, Zi, ncomp = grid.shape
    if ncomp != 3:
        raise ValueError(f"grid must be [B, Xi, Yi, Zi, 3], got {tuple(grid.shape)}")
    Cc = 1
    if inp is not None:
        inp = inp.contiguous()
        if inp.dtype not in (torch.float16, torch.float32):
            inp = inp.float()
        if inp.shape[0] != Bn or tuple(inp.shape[2:]) != (Xi, Yi, Zi):
            raise ValueError(f"input {tuple(inp.shape)} does not match the grid {tuple(grid.shape)}")
        Cc = inp.shape[1]
    X, Y, Z = (int(v) for v in shape)
    out = torch.empty((Bn, Cc, X, Y, Z), device=grid.device, dtype=torch.float32)
    int3 = C.c_int * 3
    _call("grid_push", L.ptr(inp) if inp is not None else None, L.dt(inp) if inp is not None else 0, Bn, Cc, Xi, Yi, Zi, L.ptr(grid),
          2 if grid.dtype == torch.float64 else 0, Xi * Yi * Zi * 3, 1, 3, X, Y, Z, None, None, int3(*[int(b) for b in bound]),
          int3(*[int(o) for o in order]), int(bool(extrapolate)), L.ptr(out), L.stream_ptr(grid.device),
          nbytes=_nb(out) + (_nb(inp) if inp is not None else 0) + float(grid.numel() * grid.element_size()))
    return out


def grid_grad(src: torch.Tensor, grid: torch.Tensor, bound: Sequence[int], order: Sequence[int], extrapolate: bool = True) -> torch.Tensor:
    """src [B,C,X,Y,Z]; grid [B,Xo,Yo,Zo,3] voxel coordinates -> spatial gradients [B,C,Xo,Yo,Zo,3].  See b200_grid_grad."""
    L.require_cuda(src, grid)
    src = src.contiguous()
    if src.dtype not in (torch.float16, torch.float32):
        src = src.float()
    grid = grid.contiguous()
    if grid.dtype not in (torch.float32, torch.float64):
        grid = grid.float()
    Bn, Cc, X, Y, Z = src.shape
    _, Xo, Yo, Zo, ncomp = grid.shape
    if ncomp != 3 or grid.shape[0] != Bn:
        raise ValueError(f"grid must be [B, Xo, Yo, Zo, 3] with B = {Bn}, got {tuple(grid.shape)}")
    out = torch.empty((Bn, Cc, Xo, Yo, Zo, 3), device=src.device, dtype=src.dtype)
    int3 = C.c_int * 3
    _call("grid_grad", L.ptr(src), L.dt(src), Bn, Cc, X, Y, Z, L.ptr(grid), 2 if grid.dtype == torch.float64 else 0, Xo * Yo * Zo * 3, 1, 3,
          Xo, Yo, Zo, None, None, int3(*[int(b) for b in bound]), int3(*[int(o) for o in order]), int(bool(extrapolate)), L.ptr(out), L.dt(out),
          L.stream_ptr(src.device), nbytes=_nb(src, out) + float(grid.numel() * grid.element_size()))
    return out


def separable_filter3d(src: torch.Tensor, taps: Sequence[torch.Tensor]) -> torch.Tensor:
    """src [C,D,H,W]; taps = three float32 device vectors of odd length; zero padding."""
    L.require_cuda(src)
    src = src.contiguous()
    Cc, D, H, W = src.shape
    dst = torch.empty_like(src)
    tmp = torch.empty((2, Cc, D, H, W), device=src.device, dtype=torch.float32)
    t = [x.detach().to(device=src.device, dtype=torch.float32).contiguous() for x in taps]
    _call("separable_filter3d", L.ptr(src), L.dt(src), Cc, D, H, W, L.ptr(t[0]), t[0].numel(), L.ptr(t[1]), t[1].numel(), L.ptr(t[2]), t[2].numel(), L.ptr(tmp), L.ptr(dst), L.stream_ptr(src.device),
          nbytes=_nb(src, dst) + 4.0 * src.numel() * 4)   # three passes: read + write each, two of them through the fp32 scratch
    return dst


def patch_accumulate(patch: torch.Tensor, values: torch.Tensor, counts: torch.Tensor, location: Sequence[int]) -> None:
    """values[:, :, loc : loc + patch_size] += patch, counts[...] += 1 (1-3 spatial dims, lifted to 3)."""
    L.require_cuda(patch)
    patch = patch.contiguous()
    nd = patch.dim() - 2
    if nd < 1 or nd > 3 or values.dim() != patch.dim() or counts.shape != values.shape or tuple(values.shape[:2]) != tuple(patch.shape[:2]):
        raise ValueError(f"patch {tuple(patch.shape)} / merged {tuple(values.shape)} shapes are incompatible")
    if values.dtype != torch.float32 or not values.is_contiguous() or not counts.is_contiguous() or counts.dtype not in (torch.uint8, torch.int32):
        raise ValueError("AvgMerger buffers must be contiguous float32 values and uint8 / int32 counts")
    ps = (1,) * (3 - nd) + tuple(patch.shape[2:])
    ms = (1,) * (3 - nd) + tuple(values.shape[2:])
    loc = (0,) * (3 - nd) + tuple(int(v) for v in location)
    _call("patch_accumulate", L.ptr(patch), L.dt(patch), patch.shape[0] * patch.shape[1], *ps, L.ptr(values), L.ptr(counts), counts.element_size(), *ms, *loc,
          L.stream_ptr(patch.device), nbytes=_nb(patch) + 2.0 * patch.numel() * (4 + counts.element_size()))


def add_f32(dst: torch.Tensor, src: torch.Tensor) -> None:
    """dst += src for contiguous float32 CUDA tensors of equal size."""
    if dst.dtype != torch.float32 or src.dtype != torch.float32 or not dst.is_contiguous() or not src.is_contiguous() or dst.numel() != src.numel():
        raise ValueError("add_f32 needs two contiguous float32 tensors of equal size")
    _call("add_f32", L.ptr(dst), L.ptr(src), dst.numel(), L.stream_ptr(dst.device), nbytes=3.0 * dst.numel() * 4)


def patch_finalize(values: torch.Tensor, counts: torch.Tensor) -> None:
    _call("patch_finalize", L.ptr(values), L.ptr(counts), counts.element_size(), values.numel(), L.stream_ptr(values.device), nbytes=_nb(values, counts) + _nb(values))


POST_SOFTMAX, POST_SIGMOID, POST_ARGMAX, POST_THRESHOLD, POST_ROUND, POST_ONEHOT = range(6)


def channel_post(x: torch.Tensor, op: int, param: float = 0.0, onehot: int = 0, out_dtype: torch.dtype | None = None) -> torch.Tensor:
    """Channel-first post-processing x[C, *spatial] -> y (see b200_channel_post): softmax / sigmoid / argmax / threshold / round / one-hot."""
    L.require_cuda(x)
    x = x.contiguous()
    Cc = x.shape[0]
    S = x[0].numel()
    Co = (onehot if onehot > 0 else 1) if op in (POST_ARGMAX, POST_ONEHOT) else Cc
    y = torch.empty((Co, *x.shape[1:]), device=x.device, dtype=out_dtype or x.dtype)
    _call("channel_post", L.ptr(x), L.dt(x), Cc, S, op, float(param), int(onehot), L.ptr(y), L.dt(y), L.stream_ptr(x.device), nbytes=_nb(x, y))
    return y


# ---------------------------------------------------------------------------------------------- tensor-core path
class NC8:
    """fp16 activation buffer in the channel-blocked layout [N][C/8][D][H][W][8] used by the tensor-core kernels."""

    __slots__ = ("buf", "N", "C", "sp")

    def __init__(self, N: int, C_: int, sp: Sequence[int], device, buf: torch.Tensor | None = None):
        if C_ % 8:
            raise ValueError("NC8 needs a channel count divisible by 8")
        self.N, self.C, self.sp = N, C_, tuple(int(s) for s in sp)
        self.buf = buf if buf is not None else torch.empty((N, C_ // 8, *self.sp, 8), device=device, dtype=torch.float16)

    @property
    def S(self) -> int:
        return self.sp[0] * self.sp[1] * self.sp[2]


def pack_nc8(x: torch.Tensor, dst: NC8 | None = None, c_off: int = 0) -> NC8:
    L.require_cuda(x)
    x = x.contiguous()
    N, Cc = x.shape[:2]
    if dst is None:
        dst = NC8(N, Cc, x.shape[2:], x.device)
    _call("pack_nc8", L.ptr(x), L.dt(x), N, Cc, dst.S, L.ptr(dst.buf), dst.C, c_off, L.stream_ptr(x.device))
    return dst


def unpack_nc8(src: NC8, C_: int | None = None, c_off: int = 0, dtype: torch.dtype = torch.float16) -> torch.Tensor:
    C_ = C_ or src.C
    y = torch.empty((src.N, C_, *src.sp), device=src.buf.device, dtype=dtype)
    _call("unpack_nc8", L.ptr(src.buf), src.C, c_off, src.N, C_, src.S, L.ptr(y), L.dt(y), L.stream_ptr(y.device))
    return y


def conv3x3x3_tc_pack_weight(weight: torch.Tensor) -> torch.Tensor:
    L.require_cuda(weight)
    Cout, Cin = weight.shape[:2]
    nbytes = L.load().b200_conv3x3x3_tc_weight_bytes(Cin, Cout)
    if nbytes < 0:
        raise ValueError(f"conv3x3x3_tc needs Cin, Cout multiples of 16, got {Cin}, {Cout}")
    w32 = weight.detach().float().contiguous()
    packed = torch.empty(nbytes // 2, device=weight.device, dtype=torch.float16)
    _call("conv3x3x3_tc_pack_weight", L.ptr(w32), Cin, Cout, L.ptr(packed), L.stream_ptr(weight.device))
    return packed


def conv3x3x3_tc(
    x: NC8, packed_w: torch.Tensor, Cin: int, Cout: int, in_coff: int = 0, bias: torch.Tensor | None = None,
    out: NC8 | None = None, out_coff: int = 0, want_stats: bool = False,
    in_norm: tuple[torch.Tensor, float, int, float] | None = None, res_w: torch.Tensor | None = None,
    in_affine: tuple[torch.Tensor | None, torch.Tensor | None] | None = None,
):
    """3x3x3 / stride 1 / pad 1 convolution.  `in_norm` = (stats, eps, act, slope): x is the RAW output of the previous
    convolution and InstanceNorm + activation are applied on the operand load (no norm_act pass in between).
    `in_affine` = (gamma, beta) of that InstanceNorm (affine=True; either may be None); it needs `in_norm`.
    `res_w` = gemm_tc_pack_weight image of a 1x1x1 convolution [Cout, Cin] of the SAME input: it is computed by the same launch
    and the call returns (out, stats, res_out, res_stats) instead of (out, stats)."""
    if out is None:
        out = NC8(x.N, Cout, x.sp, x.buf.device)
    dev = x.buf.device
    stats = torch.empty((x.N * Cout, 2), device=dev, dtype=torch.float32) if want_stats else None
    b32 = _f32c(bias)
    d = L.ConvTcDesc(x.N, Cin, Cout, x.sp[0], x.sp[1], x.sp[2], x.C, in_coff, out.C, out_coff, None, 0.0, 0, 0.0, None, None, 0, 0, None)
    res_out = res_stats = None
    if res_w is not None:
        if in_norm is not None or Cout > 128:
            raise ValueError("conv3x3x3_tc: the folded 1x1x1 convolution needs Cout <= 128 and no in_norm")
        res_out = NC8(x.N, Cout, x.sp, dev)
        res_stats = torch.empty((x.N * Cout, 2), device=dev, dtype=torch.float32) if want_stats else None
        d.res_w, d.res_y, d.res_ctot, d.res_coff, d.res_stats = L.ptr(res_w), L.ptr(res_out.buf), res_out.C, 0, L.ptr(res_stats)
    if in_norm is not None:
        st, eps, act, slope = in_norm
        if st.dtype != torch.float32 or st.numel() != x.N * Cin * 2 or not st.is_contiguous() or st.device != dev:
            raise ValueError("conv3x3x3_tc: in_norm statistics must be a contiguous float32 [N*Cin, 2] tensor on the input's device")
        d.in_stats, d.in_eps, d.in_act, d.in_slope = L.ptr(st), float(eps), int(act), float(slope)
    ws = _ws(L.load().b200_conv3x3x3_tc_workspace_bytes(C.byref(d)), dev) if want_stats else None
    if in_affine is not None and any(t is not None for t in in_affine):
        if in_norm is None:
            raise ValueError("conv3x3x3_tc: in_affine needs in_norm")
        name, extra = "conv3x3x3_tc_affine", (L.ptr(_f32c(in_affine[0])), L.ptr(_f32c(in_affine[1])))
    else:
        name, extra = "conv3x3x3_tc", ()
    _call(name, C.byref(d), *extra, L.ptr(x.buf), L.ptr(packed_w), L.ptr(b32), L.ptr(out.buf), L.ptr(stats), L.ptr(ws), L.stream_ptr(dev),
          flops=2.0 * x.N * x.S * Cin * Cout * (28 if res_w is not None else 27),
          nbytes=float(x.N * x.S * (Cin + Cout * (2 if res_w is not None else 1)) * 2) + _nb(packed_w))
    if res_w is not None:
        return out, stats, res_out, res_stats
    return out, stats


def norm_act_cin1res_nc8(x: NC8, C_: int, stats: torch.Tensor, raw: torch.Tensor, raw_stats: torch.Tensor, raw_weight: torch.Tensor,
                         act: int = L.ACT_NONE, slope: float = 0.0, out: NC8 | None = None, out_coff: int = 0, eps: float = 1e-5) -> NC8:
    """act(instnorm(x) + instnorm(conv1x1x1(raw))) for a ONE-channel `raw` [N,1,*sp] fp16: the residual branch is an affine
    function of raw per channel, so neither the 1x1x1 convolution nor its output exist (see the header)."""
    if raw.dtype != torch.float16 or raw.shape[1] != 1:
        raise ValueError("norm_act_cin1res_nc8 expects a contiguous fp16 [N,1,D,H,W] input")
    raw = raw.contiguous()
    if out is None:
        out = NC8(x.N, C_, x.sp, x.buf.device)
    w32 = _f32c(raw_weight.reshape(-1))
    _call("norm_act_cin1res_nc8", L.ptr(x.buf), x.C, 0, x.N, C_, x.S, L.ptr(stats), eps, L.ptr(raw), L.ptr(raw_stats), L.ptr(w32), act,
          float(slope), L.ptr(out.buf), out.C, out_coff, L.stream_ptr(x.buf.device), nbytes=float(x.N * x.S * C_ * 4))
    return out


def norm_act_nc8(
    x: NC8, C_: int, stats: torch.Tensor | None, x_coff: int = 0, res: NC8 | None = None, res_coff: int = 0,
    res_stats: torch.Tensor | None = None, act: int = L.ACT_NONE, slope: float = 0.0, out: NC8 | None = None,
    out_coff: int = 0, eps: float = 1e-5, gamma: torch.Tensor | None = None, beta: torch.Tensor | None = None,
    res_gamma: torch.Tensor | None = None, res_beta: torch.Tensor | None = None,
) -> NC8:
    """y = act(instnorm(x) [+ instnorm?(res)]) on NC8 channel slices; gamma / beta (res_gamma / res_beta) are the affine
    parameters of x's (res's) InstanceNorm."""
    if out is None:
        out = NC8(x.N, C_, x.sp, x.buf.device)
    affine = (gamma, beta, res_gamma, res_beta)
    name, extra = "norm_act_nc8", ()
    if any(t is not None for t in affine):
        name, extra = "norm_act_affine_nc8", tuple(L.ptr(_f32c(t)) for t in affine)
    _call(name, L.ptr(x.buf), x.C, x_coff, x.N, C_, x.S, L.ptr(stats), eps, L.ptr(res.buf) if res is not None else None,
          res.C if res is not None else 0, res_coff, L.ptr(res_stats), act, float(slope), L.ptr(out.buf), out.C, out_coff, *extra,
          L.stream_ptr(x.buf.device))
    return out


def cat_channels(tensors: Sequence[torch.Tensor]) -> torch.Tensor:
    """torch.cat(tensors, dim=1) for [N,C_i,*spatial] tensors of one dtype, done by the channel-copy kernel."""
    t0 = tensors[0]
    N, sp = t0.shape[0], tuple(t0.shape[2:])
    lift = 3 - len(sp)
    sp3 = (1,) * lift + sp
    ctot = sum(int(t.shape[1]) for t in tensors)
    out = torch.empty((N, ctot, *sp3), device=t0.device, dtype=t0.dtype)
    off = 0
    for t in tensors:
        if tuple(t.shape[2:]) != sp or t.dtype != t0.dtype:
            raise ValueError("cat_channels needs equal spatial shapes and dtypes")
        copy_channels(t.reshape(N, t.shape[1], *sp3), out, off)
        off += int(t.shape[1])
    return out.reshape(N, ctot, *sp)


def gemm_tc_pack_weight(w2d: torch.Tensor) -> torch.Tensor:
    """Pack W[N,K] (any float dtype, device) into the wgmma B-operand image used by gemm_tc."""
    L.require_cuda(w2d)
    w32 = w2d.detach().float().contiguous()
    N, Kd = w32.shape
    nbytes = L.load().b200_gemm_tc_weight_bytes(N, Kd)
    if nbytes < 0:
        raise ValueError(f"gemm_tc needs N and K multiples of 16, got {N}, {Kd}")
    packed = torch.empty(nbytes // 2, device=w32.device, dtype=torch.float16)
    _call("gemm_tc_pack_weight", L.ptr(w32), N, Kd, Kd, 1, L.ptr(packed), L.stream_ptr(w32.device))
    return packed


def gemm_tc(
    x: NC8, packed_w: torch.Tensor, Kd: int, N: int, bias: torch.Tensor | None = None, in_coff: int = 0,
    out: NC8 | None = None, out_coff: int = 0, res: NC8 | None = None, res_coff: int = 0, row_map: torch.Tensor | None = None,
    out_sp: Sequence[int] | None = None, mode: int = 0, act: int = L.ACT_NONE, want_stats: bool = False,
) -> tuple[NC8, torch.Tensor | None]:
    """y = [res +] act(x W^T + b).  mode 0: rows map to rows; mode 1: rows scattered through row_map into a
    destination with spatial shape out_sp; mode 2: ConvTranspose k2 s2 (N = 8*Cout, destination 2x upsampled)."""
    cout = N // 8 if mode == 2 else N
    if out is None:
        sp = tuple(out_sp) if out_sp is not None else (tuple(2 * s for s in x.sp) if mode == 2 else x.sp)
        out = NC8(x.N, cout, sp, x.buf.device)
    dev = x.buf.device
    stats = torch.empty((x.N * N, 2), device=dev, dtype=torch.float32) if want_stats else None
    b32 = _f32c(bias)
    d = L.GemmTcDesc(
        x.N, x.S, Kd, N, x.C, in_coff, out.C, out_coff, res.C if res is not None else 0, res_coff, out.S, mode, act,
        x.sp[0], x.sp[1], x.sp[2],
    )
    ws = _ws(L.load().b200_gemm_tc_workspace_bytes(C.byref(d)), dev) if want_stats else None
    _call("gemm_tc", C.byref(d), L.ptr(x.buf), L.ptr(packed_w), L.ptr(b32), L.ptr(res.buf) if res is not None else None,
          L.ptr(row_map), L.ptr(out.buf), L.ptr(stats), L.ptr(ws), L.stream_ptr(dev),
          flops=2.0 * x.N * x.S * Kd * N, nbytes=float(x.N * x.S * (Kd + N) * 2) + _nb(packed_w))
    return out, stats


def mlp_fused_supported(C_: int, hidden: int) -> bool:
    return C_ == 48 and hidden == 192


def mlp_fused_tc(x: NC8, packed_w1: torch.Tensor, b1: torch.Tensor, packed_w2: torch.Tensor, b2: torch.Tensor, hidden: int,
                 gamma: torch.Tensor | None, beta: torch.Tensor | None, eps: float = 1e-5) -> NC8:
    """x + fc2(gelu(fc1(LayerNorm(x)))) in one launch (hidden activations never reach HBM)."""
    out = NC8(x.N, x.C, x.sp, x.buf.device)
    _call("mlp_fused_tc", L.ptr(x.buf), x.C, x.N, x.S, x.C, hidden, L.ptr(packed_w1), L.ptr(_f32c(b1)), L.ptr(packed_w2), L.ptr(_f32c(b2)),
          L.ptr(_f32c(gamma)), L.ptr(_f32c(beta)), float(eps), L.ptr(out.buf), out.C, L.stream_ptr(x.buf.device),
          flops=4.0 * x.N * x.S * x.C * hidden, nbytes=float(x.N * x.S * x.C * 2 * 3))
    return out


def layernorm_nc8(x: NC8, gamma: torch.Tensor | None, beta: torch.Tensor | None, eps: float = 1e-5, src: torch.Tensor | None = None,
                  out_sp: Sequence[int] | None = None, out: NC8 | None = None) -> NC8:
    """LayerNorm over channels; with `src` (int32 [S_out]) the output rows are gathered (−1 = zero row)."""
    if out is None:
        out = NC8(x.N, x.C, tuple(out_sp) if out_sp is not None else x.sp, x.buf.device)
    g, b = _f32c(gamma), _f32c(beta)
    _call("layernorm_nc8", L.ptr(x.buf), x.N, x.C, x.S, L.ptr(src), out.S, L.ptr(g), L.ptr(b), float(eps), L.ptr(out.buf), L.stream_ptr(x.buf.device),
          nbytes=float(x.N * x.C * (x.S + out.S) * 2))
    return out


def patch_merge_ln_nc8(x: NC8, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5, v2: bool = False) -> NC8:
    sp2 = tuple((s + 1) // 2 for s in x.sp)
    out = NC8(x.N, 8 * x.C, sp2, x.buf.device)
    g, b = _f32c(gamma), _f32c(beta)
    _call("patch_merge_ln_nc8", L.ptr(x.buf), x.N, x.C, x.sp[0], x.sp[1], x.sp[2], L.ptr(g), L.ptr(b), float(eps), int(v2), L.ptr(out.buf), L.stream_ptr(x.buf.device))
    return out


def window_attention_nc8(qkv: NC8, Cc: int, heads: int, nW: int, n: int, scale: float, table: torch.Tensor, window: Sequence[int],
                         region: torch.Tensor | None) -> NC8:
    """table: relative_position_bias_table [(2w0-1)(2w1-1)(2w2-1), heads] of the module window `window`."""
    out = NC8(qkv.N, Cc, qkv.sp, qkv.buf.device)
    tab = _f32c(table)
    _call("window_attention_nc8", L.ptr(qkv.buf), qkv.N, Cc, heads, nW, n, float(scale), L.ptr(tab), int(window[0]), int(window[1]), int(window[2]),
          L.ptr(region), L.ptr(out.buf), L.stream_ptr(qkv.buf.device), flops=4.0 * qkv.N * nW * heads * n * n * 16,
          nbytes=float(qkv.N * 4 * Cc * nW * n * 2))
    return out


def window_attention_tc_plan(region, nW: int, n: int):
    """Host-side schedule of b200_window_attention_tc: windows grouped by shift-mask pattern.

    region: int array [nW, n] of compute_mask labels (or None without a shift).  Returns (sched int32 numpy [16 + nW] =
    count[8] | start[8] | window ids grouped by type, region_types int32 numpy [ntypes, n] or None, ntypes); ntypes > 8
    means "not representable" (the caller keeps the mma.sync kernel)."""
    import numpy as np

    if region is None:
        types = np.zeros(nW, dtype=np.int64)
        reps = None
        ntypes = 1
    else:
        region = np.asarray(region).reshape(nW, n)
        canon = np.empty_like(region)
        for w in range(nW):   # relabel by first appearance: equal masks <=> equal canonical rows
            _, first, inv = np.unique(region[w], return_index=True, return_inverse=True)
            order = np.argsort(np.argsort(first))
            canon[w] = order[inv]
        uniq, types = np.unique(canon, axis=0, return_inverse=True)
        types = types.reshape(-1)
        ntypes = int(uniq.shape[0])
        reps = uniq.astype(np.int32)
    sched = np.zeros(16 + nW, dtype=np.int32)
    if ntypes <= 8:
        pos = 0
        for t in range(ntypes):
            ids = np.nonzero(types == t)[0]
            sched[t], sched[8 + t] = len(ids), pos
            sched[16 + pos: 16 + pos + len(ids)] = ids
            pos += len(ids)
    return sched, reps, ntypes


def window_attention_tc_pack_bias(table: torch.Tensor, heads: int, n: int, window: Sequence[int], region_types: torch.Tensor | None, ntypes: int) -> torch.Tensor:
    """fp16 images of log2(e) * (relative-position bias + shift mask) per (mask type, head, 192-row tile), in the order of
    the kernel's score accumulators."""
    tab = _f32c(table)
    nbytes = L.load().b200_window_attention_tc_bias_bytes(heads, n, ntypes)
    if nbytes < 0:
        raise ValueError(f"window_attention_tc: unsupported shape (n={n}, mask types={ntypes})")
    packed = torch.empty(nbytes // 2, device=tab.device, dtype=torch.float16)
    _call("window_attention_tc_pack_bias", L.ptr(tab), heads, n, int(window[0]), int(window[1]), int(window[2]), L.ptr(region_types), ntypes,
          L.ptr(packed), L.stream_ptr(tab.device))
    return packed


def window_attention_tc(qkv: NC8, Cc: int, heads: int, nW: int, n: int, packed_bias: torch.Tensor, sched: torch.Tensor, ntypes: int) -> NC8:
    """Window attention on wgmma (b200_window_attention_tc); q must be pre-scaled by scale * log2(e)."""
    out = NC8(qkv.N, Cc, qkv.sp, qkv.buf.device)
    n_pad = (n + 31) // 32 * 32
    _call("window_attention_tc", L.ptr(qkv.buf), qkv.N, Cc, heads, nW, n, L.ptr(packed_bias), L.ptr(sched), ntypes, L.ptr(out.buf),
          L.stream_ptr(qkv.buf.device), flops=4.0 * qkv.N * nW * heads * n * n * 16, nbytes=float(qkv.N * 4 * Cc * nW * n * 2))
    return out


def mhsa_tc(qkv: NC8, C_: int, heads: int) -> NC8:
    """Global multi-head attention on wgmma (b200_mhsa_tc), head_dim 64: qkv NC8 [N][3C/8][S][8] with channels (q|k|v, head,
    dim) -> NC8 [N][C/8][S][8].  q must be pre-scaled by dim_head^-0.5 * log2(e)."""
    if qkv.C != 3 * C_:
        raise ValueError(f"mhsa_tc: qkv has {qkv.C} channels, expected 3 * {C_}")
    out = NC8(qkv.N, C_, qkv.sp, qkv.buf.device)
    S = qkv.S
    try:
        _call("mhsa_tc", L.ptr(qkv.buf), qkv.N, C_, heads, S, L.ptr(out.buf), L.stream_ptr(qkv.buf.device),
              flops=4.0 * qkv.N * heads * S * S * 64, nbytes=float(qkv.N * 4 * C_ * S * 2))
    except RuntimeError as e:
        if C_ != 64 * heads:   # B200_ERR_UNSUPPORTED: the kernel has no other head dimension, a bad argument of this call
            raise ValueError(str(e)) from None
        raise
    return out


LOG2E = 1.4426950408889634


def conv_cin1_nc8(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor | None, k: int, stride: int, pad: int,
                  out: NC8 | None = None, out_coff: int = 0, want_stats: bool = False) -> tuple[NC8, torch.Tensor | None]:
    """x [N,1,D,H,W] (f16/f32) -> NC8 with Cout channels."""
    L.require_cuda(x)
    x = x.contiguous()
    N, _, D, H, W = x.shape
    Cout = weight.shape[0]
    sp = tuple((s + 2 * pad - k) // stride + 1 for s in (D, H, W))
    if out is None:
        out = NC8(N, Cout, sp, x.device)
    w32 = _f32c(weight)
    b32 = _f32c(bias)
    stats = torch.empty((N * Cout, 2), device=x.device, dtype=torch.float32) if want_stats else None
    # tensor-core stem for the shapes it covers (the 3x3x3 stem and the patch embedding); CUDA-core kernel otherwise
    tc = (k, stride, pad) in ((3, 1, 1), (2, 2, 0)) and Cout in (16, 32, 48, 64, 96, 128)
    name = "conv_cin1_tc" if tc else "conv_cin1_nc8"
    ws = None
    if want_stats:
        ws = _ws(getattr(L.load(), f"b200_{name}_workspace_bytes")(N, D, H, W, Cout, k, stride, pad), x.device)
    _call(name, L.ptr(x), L.dt(x), N, D, H, W, L.ptr(w32), L.ptr(b32), Cout, k, stride, pad, L.ptr(out.buf), out.C, out_coff, L.ptr(stats), L.ptr(ws),
          L.stream_ptr(x.device), flops=2.0 * N * sp[0] * sp[1] * sp[2] * Cout * k**3, nbytes=_nb(x) + float(N * sp[0] * sp[1] * sp[2] * Cout * 2))
    return out, stats


def head_conv_nc8(x: NC8, weight: torch.Tensor, bias: torch.Tensor | None, out_dtype: torch.dtype = torch.float16) -> torch.Tensor:
    Cout = weight.shape[0]
    w32 = _f32c(weight)
    b32 = _f32c(bias)
    y = torch.empty((x.N, Cout, *x.sp), device=x.buf.device, dtype=out_dtype)
    _call("head_conv_nc8", L.ptr(x.buf), x.N, x.C, x.S, L.ptr(w32), L.ptr(b32), Cout, L.ptr(y), L.dt(y), L.stream_ptr(x.buf.device))
    return y


def head_conv_norm_nc8(x: NC8, stats: torch.Tensor, res: NC8 | None, res_coff: int, res_stats: torch.Tensor | None, slope: float, eps: float,
                       weight: torch.Tensor, bias: torch.Tensor | None, out_dtype: torch.dtype = torch.float16,
                       gamma: torch.Tensor | None = None, beta: torch.Tensor | None = None) -> torch.Tensor:
    """logits = W * lrelu(instnorm(x) + instnorm?(res)) + b: the last block's tail fused into the 1x1x1 head; gamma / beta are
    the affine parameters of x's InstanceNorm."""
    Cout = weight.shape[0]
    w32 = _f32c(weight)
    b32 = _f32c(bias)
    y = torch.empty((x.N, Cout, *x.sp), device=x.buf.device, dtype=out_dtype)
    name, extra = "head_conv_norm_nc8", ()
    if gamma is not None or beta is not None:
        name, extra = "head_conv_norm_affine_nc8", (L.ptr(_f32c(gamma)), L.ptr(_f32c(beta)))
    _call(name, L.ptr(x.buf), x.N, x.C, x.S, L.ptr(stats), float(eps), L.ptr(res.buf) if res is not None else None,
          res.C if res is not None else 0, res_coff, L.ptr(res_stats), float(slope), L.ptr(w32), L.ptr(b32), Cout, L.ptr(y), L.dt(y), *extra,
          L.stream_ptr(x.buf.device), nbytes=float(x.N * x.S * (x.C * (4 if res is not None else 2) + Cout * y.element_size())))
    return y


def _cg_desc(x_sp, N, Cin, Cout, k, stride, pad, transposed, output_padding, in_ctot, in_coff, out_ctot, out_coff, out_layout, out_dtype):
    sp_out = conv_out_shape(x_sp, (k,) * 3, (stride,) * 3, (pad,) * 3, transposed, (output_padding,) * 3)
    return L.ConvGatherDesc(N, Cin, Cout, x_sp[0], x_sp[1], x_sp[2], sp_out[0], sp_out[1], sp_out[2], k, stride, pad, int(transposed),
                            in_ctot, in_coff, out_ctot, out_coff, out_layout, out_dtype), sp_out


def conv_gather_tc_pack_weight(weight: torch.Tensor, k: int, stride: int, pad: int, transposed: bool) -> torch.Tensor:
    """Pack a Conv3d [Cout,Cin,k,k,k] / ConvTranspose3d [Cin,Cout,k,k,k] weight for conv_gather_tc."""
    L.require_cuda(weight)
    Cin, Cout = (weight.shape[0], weight.shape[1]) if transposed else (weight.shape[1], weight.shape[0])
    d, _ = _cg_desc((8, 8, 8), 1, Cin, Cout, k, stride, pad, transposed, stride - 1 if transposed else 0, Cin, 0, (Cout + 7) // 8 * 8, 0, 1, L.DT_F16)
    nbytes = L.load().b200_conv_gather_tc_weight_bytes(C.byref(d))
    if nbytes < 0:
        raise ValueError(f"conv_gather_tc needs Cin % 16 == 0, kernel <= 3, stride <= 2 (got Cin={Cin}, k={k}, stride={stride})")
    w32 = weight.detach().float().contiguous()
    packed = torch.empty(nbytes // 2, device=weight.device, dtype=torch.float16)
    _call("conv_gather_tc_pack_weight", C.byref(d), L.ptr(w32), L.ptr(packed), L.stream_ptr(weight.device))
    return packed


def conv_gather_tc(
    x: NC8, packed_w: torch.Tensor, Cin: int, Cout: int, k: int, stride: int, pad: int, transposed: bool = False, output_padding: int = 0,
    in_coff: int = 0, bias: torch.Tensor | None = None, out: "NC8 | torch.Tensor | None" = None, out_coff: int = 0,
    ncdhw_dtype: torch.dtype | None = None, want_stats: bool = False,
):
    """Conv3d / ConvTranspose3d on tensor cores.  Returns (NC8 | NCDHW tensor, stats)."""
    layout = 0 if ncdhw_dtype is None else 1
    d, sp_out = _cg_desc(x.sp, x.N, Cin, Cout, k, stride, pad, transposed, output_padding, x.C, in_coff,
                         (out.C if isinstance(out, NC8) else (Cout + 7) // 8 * 8), out_coff, layout, L.dt(ncdhw_dtype) if layout else L.DT_F16)
    if out is None:
        out = NC8(x.N, Cout, sp_out, x.buf.device) if layout == 0 else torch.empty((x.N, Cout, *sp_out), device=x.buf.device, dtype=ncdhw_dtype)
        d.out_ctot = out.C if layout == 0 else d.out_ctot
    stats = torch.empty((x.N * Cout, 2), device=x.buf.device, dtype=torch.float32) if want_stats else None
    b32 = _f32c(bias)
    taps = k**3 if not transposed else (k**3) / (stride**3)
    ws = _ws(L.load().b200_conv_gather_tc_workspace_bytes(C.byref(d)), x.buf.device) if want_stats else None
    _call("conv_gather_tc", C.byref(d), L.ptr(x.buf), L.ptr(packed_w), L.ptr(b32), L.ptr(out.buf if layout == 0 else out), L.ptr(stats), L.ptr(ws),
          L.stream_ptr(x.buf.device), flops=2.0 * x.N * sp_out[0] * sp_out[1] * sp_out[2] * Cin * Cout * taps,
          nbytes=float(x.N * (x.S * Cin + sp_out[0] * sp_out[1] * sp_out[2] * Cout) * 2) + _nb(packed_w))
    return out, stats


def convt3s2_head_nc8(x: NC8, Cin: int, weight: torch.Tensor, bias: torch.Tensor | None, in_coff: int = 0, out_dtype: torch.dtype = torch.float16) -> torch.Tensor:
    """ConvTranspose3d(k3, s2, p1, op1) head: NC8 features -> NCDHW logits with <= 4 channels (CUDA cores)."""
    Cout = weight.shape[1]
    y = torch.empty((x.N, Cout, *(2 * s for s in x.sp)), device=x.buf.device, dtype=out_dtype)
    _call("convt3s2_head_nc8", L.ptr(x.buf), x.N, Cin, x.sp[0], x.sp[1], x.sp[2], x.C, in_coff, L.ptr(_f32c(weight)), L.ptr(_f32c(bias)), Cout,
          L.ptr(y), L.dt(y), L.stream_ptr(x.buf.device), flops=2.0 * x.N * x.S * 27 * Cin * Cout, nbytes=float(x.N * x.S * Cin * 2) + _nb(y))
    return y
