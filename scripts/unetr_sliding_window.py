#!/usr/bin/env python
"""UNETR (the reference's defaults: ViT-B/16, feature_size 16, 14 classes) as the predictor of a sliding-window inference.

    python scripts/unetr_sliding_window.py [--sw-batch 4] [--steps 3] [--warmup 1]

A 256^3 fp16 volume, roi 96^3, overlap 0.5, gaussian blending: 125 windows per step.  Every batch shape (the full batches
and the remainder batch) is warmed up first; each timed step is bracketed by CUDA events with a 256 MiB L2 flush before it
(outside the timed interval).  A separate profiled step lists the top kernels.  Finally one forward of a 4-window fp16
batch is timed on each path: `net(x)` (tensor cores) and `net._forward_generic(x)` (the generic CUDA-core kernels), giving
the speed-up per window without running 125 windows on CUDA cores.  Prints one JSON line, with the card name and power
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

VOLUME, ROI, OVERLAP = (256, 256, 256), (96, 96, 96), 0.5


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


def window_flops(net, roi) -> dict:
    """Multiply-add FLOPs (x2) of one window, from the layer shapes of UNETR.forward (ViT and decoder separately)."""
    hid, mlp, heads = net.hidden_size, net.mlp_dim, net.num_heads
    fs, cin = net.feature_size, net.in_channels
    v = [math.prod(s // 2**k for s in roi) for k in range(5)]   # voxels at 1, 1/2, 1/4, 1/8, 1/16 resolution
    S = v[4]
    vit = 2.0 * S * cin * 16**3 * hid
    vit += net.num_layers * (2.0 * S * hid * 3 * hid + 4.0 * heads * S * S * (hid // heads) + 2.0 * S * hid * hid + 4.0 * S * hid * mlp)

    def res(ci, co, n):      # UnetResBlock: two 3x3x3 convolutions and a 1x1x1 one when the channels change
        return 2.0 * n * 27 * (ci * co + co * co) + (2.0 * n * ci * co if ci != co else 0.0)

    def up(ci, co, n_in):    # ConvTranspose3d k2 s2
        return 2.0 * n_in * 8 * ci * co

    dec = res(cin, fs, v[0])
    dec += up(hid, 2 * fs, v[4]) + up(2 * fs, 2 * fs, v[3]) + res(2 * fs, 2 * fs, v[2]) + up(2 * fs, 2 * fs, v[2]) + res(2 * fs, 2 * fs, v[1])
    dec += up(hid, 4 * fs, v[4]) + up(4 * fs, 4 * fs, v[3]) + res(4 * fs, 4 * fs, v[2])
    dec += up(hid, 8 * fs, v[4])
    dec += up(hid, 8 * fs, v[4]) + res(16 * fs, 8 * fs, v[3])
    dec += up(8 * fs, 4 * fs, v[3]) + res(8 * fs, 4 * fs, v[2])
    dec += up(4 * fs, 2 * fs, v[2]) + res(4 * fs, 2 * fs, v[1])
    dec += up(2 * fs, fs, v[1]) + res(2 * fs, fs, v[0])
    dec += 2.0 * v[0] * fs * net.out.conv.conv.out_channels
    return {"vit": vit, "decoder": dec, "total": vit + dec}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sw-batch", type=int, default=4)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--top", type=int, default=12)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("unetr_sliding_window.py measures on a CUDA device; none is available")

    from weights import fill_state_dict

    from monai_b200 import _kernels as K
    from monai_b200.inferers import sliding_window_inference
    from monai_b200.networks.nets import UNETR

    dev = torch.device("cuda:0")
    card = _card()
    net = UNETR(in_channels=1, out_channels=14, img_size=ROI)
    net.load_state_dict(fill_state_dict(net.state_dict(), 80))
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

        # one 4-window batch on each path
        x4 = torch.randn((4, 1, *ROI), generator=torch.Generator().manual_seed(1)).half().to(dev)

        def timed(fn, reps):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fn(x4)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / reps

        net(x4)
        tc_ms = timed(net, 5)
        net._forward_generic(x4[:1])   # loads the generic kernels
        gen_ms = timed(net._forward_generic, 1)

    fl = window_flops(net, ROI)
    ms = sorted(times)[len(times) // 2]
    res = {
        "metric": "unetr_sliding_window",
        "card": card,
        "config": {"volume": list(VOLUME), "roi": list(ROI), "overlap": OVERLAP, "mode": "gaussian", "sw_batch": args.sw_batch,
                   "windows": windows, "dtype": "float16", "net": "UNETR(in=1, out=14, img=96, hidden=768, heads=12, mlp=3072, fs=16)",
                   "l2": "256 MiB flush write between timed steps", "steps": args.steps},
        "ms_per_step": round(ms, 2), "ms_per_step_all": [round(t, 2) for t in times],
        "voxels_per_s": math.prod(VOLUME) / (ms / 1e3),
        "gflop_per_window": {k: round(v / 1e9, 2) for k, v in fl.items()},
        "model_tflops": fl["total"] * windows / (ms / 1e3) / 1e12,
        "profile_ms_total": round(prof_ms, 2),
        "top_kernels": [{"name": n, "ms": round(d["ms"], 3), "share": round(d["ms"] / prof_ms, 4), "n": d["n"],
                         "tflops": round(d["flops"] / (d["ms"] / 1e3) / 1e12, 1) if d["flops"] and d["ms"] else None} for n, d in top],
        "profile_gflop_per_window": round(sum(d["flops"] for d in prof.values()) / windows / 1e9, 2),
        "per_window_ms_batch4": {"tensor_core": round(tc_ms / 4, 3), "generic": round(gen_ms / 4, 3), "speedup": round(gen_ms / tc_ms, 1)},
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
