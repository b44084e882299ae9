#!/usr/bin/env python
"""Per-shape timing of the stride-1 one-plane convolutions (kernel [1,3,3], [3,1,3] or [3,3,1]) of the anisotropic DynUNet
workloads of sliding_window_tc.py (aniso_d, aniso_w), on the three kernels that can run them:

  * conv3x3_tc:                the one-plane kernel (what the network runs);
  * conv3x3x3_tc, zero-padded: the 3x3x3 kernel with the weight zero-padded to 3x3x3 (the same bits, 3x the MMAs of axis 0);
  * conv_gather_tc:            the im2col gather kernel with the per-axis kernel, stride 1 and padding; it has no operand
                               normalisation, so a launch that normalises its input on the load is charged a norm_act_nc8 pass.

    python scripts/conv3x3_tc_shapes.py [--sw-batch 4] [--min-seconds 0.5] [--warmup 10]

Records the arguments of every conv3x3_tc call of one eager forward of sw_batch windows, then times each distinct call shape
with CUDA events, a 256 MiB L2 flush before every launch (outside the timed interval).  Every launch is also set against its
floor, max(FLOP / 989 TFLOP/s, bytes / 3.35 TB/s) (the H100 SXM data sheet: dense fp16, HBM3), with the bound that sets it.
Prints one JSON line per workload, with the card name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sw-batch", type=int, default=4)
    ap.add_argument("--min-seconds", type=float, default=0.5, help="timed launches per variant cover at least this much device time")
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("conv3x3_tc_shapes.py needs a CUDA device")
    from sliding_window_tc import _card, _nets
    from weights import fill_state_dict

    from monai_b200 import _kernels as K
    from monai_b200 import _lib as L

    dev = torch.device("cuda", 0)
    L.load()
    card = _card()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timeit(fn) -> float:
        """ms per launch: warm-up, a probe to size the run, then >= min_seconds of flushed, individually timed launches."""
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(3):
            fn()
        e1.record()
        e1.synchronize()
        reps = max(10, int(args.min_seconds * 1e3 / max(1e-3, e0.elapsed_time(e1) / 3)) + 1)
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
        for a, b in ev:
            flush.fill_(1)
            a.record()
            fn()
            b.record()
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in ev) / reps

    nets = _nets()["dynunet"]
    for name in ("dynunet_sliding_window_aniso_d", "dynunet_sliding_window_aniso_w"):
        wl = nets[name]
        net = wl["make"]()
        net.load_state_dict(fill_state_dict(net.state_dict(), wl["seed"]))
        net = net.half().eval().to(dev)
        net._graph_enabled = False   # one eager forward: every launch goes through the Python entry point
        calls, order = {}, []
        orig = K.conv3x3_tc

        def recording(x, packed_w, Cin, Cout, axis, **kw):
            key = (x.N, Cin, Cout, x.sp, axis, kw.get("in_norm") is not None)
            if key not in calls:
                calls[key] = {"count": 0, "x": x, "kw": kw}
                order.append(key)
            calls[key]["count"] += 1
            return orig(x, packed_w, Cin, Cout, axis, **kw)

        x_in = torch.randn((args.sw_batch, wl["cin"], *wl["roi"]), generator=torch.Generator().manual_seed(0)).half().to(dev)
        K.conv3x3_tc = recording
        try:
            with torch.no_grad():
                net(x_in)
        finally:
            K.conv3x3_tc = orig
        torch.cuda.synchronize()

        rows, sums = [], {"conv3x3_tc": 0.0, "conv3x3x3_tc_zero_padded": 0.0, "conv_gather_tc": 0.0}
        for key in order:
            N, cin, cout, sp, axis, norm = key
            x, kw = calls[key]["x"], calls[key]["kw"]
            k = tuple(1 if a == axis else 3 for a in range(3))
            pad = tuple((i - 1) // 2 for i in k)
            w = torch.randn((cout, cin, *k), generator=torch.Generator().manual_seed(cin + cout), device="cpu").to(dev) / (9 * cin) ** 0.5
            w27 = torch.zeros((cout, cin, 3, 3, 3), device=dev)
            w27[(slice(None), slice(None), *(slice(1, 2) if a == axis else slice(None) for a in range(3)))] = w
            p33, p27, pg = K.conv3x3_tc_pack_weight(w, axis), K.conv3x3x3_tc_pack_weight(w27), K.conv_gather_tc_pack_weight(w, k, 1, pad, False)
            in_coff = kw.get("in_coff", 0)
            common = dict(in_coff=in_coff, want_stats=kw.get("want_stats", False))
            fused = dict(in_norm=kw.get("in_norm"), in_affine=kw.get("in_affine"))
            ms = {
                "conv3x3_tc": timeit(lambda: orig(x, p33, cin, cout, axis, **common, **fused)),
                "conv3x3x3_tc_zero_padded": timeit(lambda: K.conv3x3x3_tc(x, p27, cin, cout, **common, **fused)),
                "conv_gather_tc": timeit(lambda: K.conv_gather_tc(x, pg, cin, cout, k, 1, pad, **common)),
            }
            if norm:   # the gather kernel needs the normalised operand in memory first
                st, eps, act, slope = kw["in_norm"]
                g, b = kw.get("in_affine") or (None, None)
                y = K.NC8(x.N, cin, x.sp, dev)
                ms["norm_act_nc8"] = timeit(lambda: K.norm_act_nc8(x, cin, st, x_coff=in_coff, act=act, slope=slope, out=y, eps=eps, gamma=g, beta=b))
                ms["conv_gather_tc"] += ms["norm_act_nc8"]
            S = sp[0] * sp[1] * sp[2]
            flops = 2.0 * N * S * cin * cout * 9
            nbytes = 2.0 * N * S * (cin + cout) + 2.0 * 9 * cin * cout
            floor_ms = max(flops / PEAK_FLOPS, nbytes / PEAK_BYTES) * 1e3
            per_step = calls[key]["count"] * wl_launches(wl, args.sw_batch)
            for impl in sums:
                sums[impl] += ms[impl] * per_step
            rows.append({"N": N, "Cin": cin, "Cout": cout, "sp": list(sp), "axis": axis, "NORM": norm, "launches_per_step": per_step,
                         "gflop": round(flops / 1e9, 2), "mbytes": round(nbytes / 1e6, 1),
                         "floor_ms": round(floor_ms, 4), "bound": "hbm" if nbytes / PEAK_BYTES > flops / PEAK_FLOPS else "tensor",
                         "ms": {i: round(v, 4) for i, v in ms.items()},
                         "share_of_floor": {i: round(floor_ms / ms[i], 3) for i in sums}})
        print(json.dumps({"workload": name, "card": card, "sw_batch": args.sw_batch, "l2": "256 MiB flush write before every timed launch",
                          "ms_per_step_sum": {i: round(v, 2) for i, v in sums.items()},
                          "conv3x3_tc_fastest": sums["conv3x3_tc"] < min(sums["conv3x3x3_tc_zero_padded"], sums["conv_gather_tc"]),
                          "shapes": rows}), flush=True)


def wl_launches(wl, sw_batch) -> int:
    """forwards of sw_batch windows per sliding-window step (the remainder batch counted as a full one)"""
    from sliding_window_tc import _windows

    return -(-_windows(wl["volume"], wl["roi"]) // sw_batch)


if __name__ == "__main__":
    main()
