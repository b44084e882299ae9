#!/usr/bin/env python
"""DynUNet (the nnU-Net default plan: 6 levels, filters 32 ... 320, affine instance norm, 14 classes) as the predictor of a
sliding-window inference.

    python scripts/dynunet_sliding_window.py [--sw-batch 4] [--steps 3] [--warmup 1]

A 384^3 fp16 volume, roi 128^3, overlap 0.5, gaussian blending: 125 windows per step.  Every batch shape (the full batches
and the remainder batch) is warmed up first; each timed step is bracketed by CUDA events with a 256 MiB L2 flush before it
(outside the timed interval).  A separate profiled step lists the top kernels.  Finally one forward of each batch shape
of the step (sw_batch windows, and the remainder batch) is timed on each path: `net(x)` (tensor cores) and
`net._forward_generic(x)` (the generic CUDA-core kernels), giving the speed-up per window without running 125 windows on
CUDA cores.  Prints one JSON line, with the card name and power
limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import torch  # noqa: E402

VOLUME, ROI, OVERLAP = (384, 384, 384), (128, 128, 128), 0.5


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


def window_flops(net, roi) -> float:
    """Multiply-add FLOPs (x2) of one window, from the layer shapes of DynUNet.forward (isotropic stride-2 plan)."""
    f, cin, nl = net.filters, net.in_channels, len(net.filters)
    v = [math.prod(s // 2**k for s in roi) for k in range(nl)]   # voxels at level k
    res = net.conv_block.__name__ == "UnetResBlock"

    def block(ci, co, n, skip_conv):   # two 3x3x3 convolutions (+ the 1x1x1 one of a residual block when shape or channels change)
        return 2.0 * n * 27 * (ci * co + co * co) + (2.0 * n * ci * co if res and skip_conv else 0.0)

    fl = block(cin, f[0], v[0], cin != f[0])
    for k in range(1, nl):                              # down blocks and the bottleneck (stride 2: output voxels v[k])
        fl += block(f[k - 1], f[k], v[k], True)
    for k in range(nl - 2, -1, -1):                     # up blocks: ConvTranspose3d k2 s2, then a basic block on the concat
        fl += 2.0 * v[k] * f[k + 1] * f[k] + 2.0 * v[k] * 27 * (2 * f[k] * f[k] + f[k] * f[k])
    return fl + 2.0 * v[0] * f[0] * net.out_channels


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sw-batch", type=int, default=4)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--top", type=int, default=12)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dynunet_sliding_window.py measures on a CUDA device; none is available")

    from weights import fill_state_dict

    from monai_b200 import _kernels as K
    from monai_b200.inferers import sliding_window_inference
    from monai_b200.networks.nets import DynUNet

    dev = torch.device("cuda:0")
    card = _card()
    net = DynUNet(3, 1, 14, kernel_size=[3] * 6, strides=[1, 2, 2, 2, 2, 2], upsample_kernel_size=[2] * 5)
    net.load_state_dict(fill_state_dict(net.state_dict(), 30))
    net = net.half().eval().to(dev)
    vol = torch.randn((1, 1, *VOLUME), generator=torch.Generator().manual_seed(0)).half().to(dev)
    windows = math.prod(len(range(0, s - r + 1, int(r * (1 - OVERLAP)))) + ((s - r) % int(r * (1 - OVERLAP)) != 0) for s, r in zip(VOLUME, ROI))

    def step():
        return sliding_window_inference(vol, ROI, args.sw_batch, net, OVERLAP, "gaussian")

    with torch.no_grad():
        for _ in range(max(1, args.warmup)):   # every batch shape, the remainder batch included
            step()
        torch.cuda.synchronize()
        flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
        times = []
        for _ in range(args.steps):
            flush.fill_(1)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        del flush

        K.profile_start()   # a separate, eager pass: the per-launch events slow the host down
        step()
        prof = K.profile_stop()
        prof_ms = sum(d["ms"] for d in prof.values())
        top = sorted(prof.items(), key=lambda kv: -kv[1]["ms"])[: args.top]

        # one batch of each shape of the step on each path
        def timed(fn, x, reps):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fn(x)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / reps

        per_window = {}
        for b in sorted({args.sw_batch, windows % args.sw_batch} - {0}):
            xb = torch.randn((b, 1, *ROI), generator=torch.Generator().manual_seed(b)).half().to(dev)
            net(xb)
            tc_ms = timed(net, xb, 5)
            net._forward_generic(xb)   # loads the generic kernels
            gen_ms = timed(net._forward_generic, xb, 1)
            per_window[f"batch{b}"] = {"tensor_core": round(tc_ms / b, 3), "generic": round(gen_ms / b, 3), "speedup": round(gen_ms / tc_ms, 1)}

    fl = window_flops(net, ROI)
    ms = sorted(times)[len(times) // 2]
    res = {
        "metric": "dynunet_sliding_window",
        "card": card,
        "config": {"volume": list(VOLUME), "roi": list(ROI), "overlap": OVERLAP, "mode": "gaussian", "sw_batch": args.sw_batch,
                   "windows": windows, "dtype": "float16", "net": "DynUNet(in=1, out=14, k=3x6, strides=[1,2,2,2,2,2], filters=32..320, affine IN)",
                   "l2": "256 MiB flush write between timed steps", "steps": args.steps},
        "ms_per_step": round(ms, 2), "ms_per_step_all": [round(t, 2) for t in times],
        "voxels_per_s": math.prod(VOLUME) / (ms / 1e3),
        "gflop_per_window": round(fl / 1e9, 2),
        "model_tflops": fl * windows / (ms / 1e3) / 1e12,
        "profile_ms_total": round(prof_ms, 2),
        "top_kernels": [{"name": n, "ms": round(d["ms"], 3), "share": round(d["ms"] / prof_ms, 4), "n": d["n"],
                         "tflops": round(d["flops"] / (d["ms"] / 1e3) / 1e12, 1) if d["flops"] and d["ms"] else None} for n, d in top],
        "profile_gflop_per_window": round(sum(d["flops"] for d in prof.values()) / windows / 1e9, 2),
        "per_window_ms": per_window,
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
