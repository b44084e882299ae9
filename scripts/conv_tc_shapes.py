#!/usr/bin/env python
"""Per-shape timing of the 3x3x3 tensor-core convolution inside the C3 workload (bench.py swin_c3).

    python scripts/conv_tc_shapes.py [--min-seconds 1.0] [--warmup 20]

Builds SwinUNETR(feature_size=48) in fp16 with the bench weights, records the arguments of every `conv3x3x3_tc` call of one
eager forward at sw_batch 25, then times each distinct call with CUDA events (a 256 MiB L2 flush before every launch, outside
the timed interval).  For every launch that normalises its input on the operand load (NORM) the same launch without `in_norm`
and the `norm_act_nc8` pass it replaces are timed too, so the cost of the fusion shows per shape.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import torch  # noqa: E402

SW_BATCH, ROI, WINDOWS = 25, (96, 96, 96), 1000   # bench.py swin_c3


def _card() -> dict:
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_max_mhz": None}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        pl, mx = r.stdout.strip().splitlines()[0].split(", ")
        out["power_limit_w"], out["sm_max_mhz"] = float(pl), float(mx)
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        pass
    return out


def _nt(cout: int) -> int:   # conv_tc_nt() in csrc/conv_tc.cu
    if cout <= 128:
        return cout
    if cout >= 384 and cout % 64 == 0:
        return 64
    return next((nt for nt in range(128, 15, -16) if cout % nt == 0), 16)


def _bd(nt: int, depth: int, res: bool) -> int:   # dispatch_bd() in csrc/conv_tc.cu
    r = 2 if res else 1
    if nt * 4 <= 256 and (depth % 4 == 0 or depth >= 16) and 4 * nt * r <= 256:
        return 4
    if nt * 2 <= 256 and depth >= 2 and 2 * nt * r <= 256:
        return 2
    return 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=1.0, help="timed launches per variant cover at least this much device time")
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("conv_tc_shapes.py needs a CUDA device")
    from weights import fill_state_dict

    from monai_b200 import _kernels as K
    from monai_b200 import _lib as L
    from monai_b200.networks.nets import SwinUNETR

    dev = torch.device("cuda", 0)
    L.load()
    net = SwinUNETR(in_channels=1, out_channels=2, feature_size=48)
    net.load_state_dict(fill_state_dict(net.state_dict(), 1))
    net = net.eval().to(dev).half()
    net._graph_enabled = False   # one eager forward: every launch goes through the Python entry point

    calls, order = {}, []
    orig = K.conv3x3x3_tc

    def recording(x, packed_w, Cin, Cout, in_coff=0, bias=None, out=None, out_coff=0, want_stats=False, in_norm=None, res_w=None):
        key = (x.N, Cin, Cout, x.sp, in_norm is not None, res_w is not None)
        if key not in calls:
            calls[key] = {"count": 0, "kw": dict(x=x, packed_w=packed_w, Cin=Cin, Cout=Cout, in_coff=in_coff, bias=bias, out=out,
                                                 out_coff=out_coff, want_stats=want_stats, in_norm=in_norm, res_w=res_w)}
            order.append(key)
        calls[key]["count"] += 1
        return orig(x, packed_w, Cin, Cout, in_coff=in_coff, bias=bias, out=out, out_coff=out_coff, want_stats=want_stats,
                    in_norm=in_norm, res_w=res_w)

    x_in = torch.randn((SW_BATCH, 1, *ROI), generator=torch.Generator().manual_seed(0)).half().to(dev)
    K.conv3x3x3_tc = recording
    try:
        with torch.no_grad():
            net(x_in)
    finally:
        K.conv3x3x3_tc = orig
    torch.cuda.synchronize()

    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timeit(fn) -> float:
        """ms per launch: warm-up, a probe to size the run, then >= min_seconds of flushed, individually timed launches."""
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            fn()
        e1.record()
        e1.synchronize()
        reps = max(20, int(args.min_seconds * 1e3 / max(1e-3, e0.elapsed_time(e1) / 5)) + 1)
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
        for a, b in ev:
            flush.fill_(1)
            a.record()
            fn()
            b.record()
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in ev) / reps

    launches_per_step = WINDOWS // SW_BATCH
    rows, total_ms = [], 0.0
    for key in order:
        N, cin, cout, sp, norm, res = key
        kw = calls[key]["kw"]
        ms = timeit(lambda: orig(**kw))
        flops = 2.0 * N * sp[0] * sp[1] * sp[2] * cin * cout * (28 if res else 27)   # as _kernels.conv3x3x3_tc passes it
        nt = _nt(cout)
        row = {"N": N, "Cin": cin, "Cout": cout, "sp": list(sp), "NT": nt, "BD": _bd(nt, sp[0], res), "NORM": norm, "RES": res,
               "launches_per_step": calls[key]["count"] * launches_per_step, "ms_per_launch": round(ms, 4),
               "tflops": round(flops / (ms * 1e-3) / 1e12, 1)}
        total_ms += ms * row["launches_per_step"]
        if norm:
            st, eps, act, slope = kw["in_norm"]
            plain = dict(kw, in_norm=None)
            ms_plain = timeit(lambda: orig(**plain))
            x = kw["x"]
            y = K.NC8(x.N, cin, x.sp, dev)
            ms_na = timeit(lambda: K.norm_act_nc8(x, cin, st, x_coff=kw["in_coff"], act=act, slope=slope, out=y, eps=eps))
            row.update({"plain_ms_per_launch": round(ms_plain, 4), "plain_tflops": round(flops / (ms_plain * 1e-3) / 1e12, 1),
                        "norm_act_nc8_ms": round(ms_na, 4), "fused_over_plain": round(ms / ms_plain, 3),
                        "fused_over_plain_plus_norm_act": round(ms / (ms_plain + ms_na), 3)})
        rows.append(row)
    print(json.dumps({"workload": "swin_c3 conv3x3x3_tc per call shape", "card": _card(), "sw_batch": SW_BATCH,
                      "l2": "256 MiB flush write before every timed launch", "conv3x3x3_tc_ms_per_step_sum": round(total_ms, 1),
                      "shapes": rows}))


if __name__ == "__main__":
    main()
