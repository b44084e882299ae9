#!/usr/bin/env python
"""Per-shape timing of the window attention inside the C3 workload (bench.py swin_c3).

    python scripts/window_attention_shapes.py [--old-lib path/to/libmonai_b200.so] [--min-seconds 1.0] [--warmup 20]

Builds SwinUNETR(feature_size=48) in fp16 with the bench weights, records the arguments of every `window_attention_tc` call
of one eager forward at sw_batch 25 (4 stages, unshifted and shifted blocks), then times each distinct call with CUDA
events (a 256 MiB L2 flush before every launch, outside the timed interval):
  * `tc`: b200_window_attention_tc of this tree;
  * `old_tc`: b200_window_attention_tc of another build of the library (`--old-lib`, e.g. one built from an earlier
    revision), with its bias packed by that library's own b200_window_attention_tc_pack_bias;
  * `nc8`: the mma.sync kernel b200_window_attention_nc8 on the same windows and mask.
Per call it reports ms per launch, launches per step, exponentials per second against the MUFU floor (16 ex2 / clk / SM,
cc 9.0 throughput table, at the SM clock read after the timed launches), both for the n^2 exponentials the algorithm needs
and for the padded work this kernel does, and the HBM bytes per launch counted from the shapes.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

SW_BATCH, ROI, WINDOWS = 25, (96, 96, 96), 1000   # bench.py swin_c3
MUFU_PER_CLK_SM = 16
GROUP = 8   # kAtGroup in csrc/attn_tc.cu: windows per schedule group
ROWS = 192  # kAtRows in csrc/attn_tc.cu: query rows per tile (three consumer warpgroups of 64)


def _smi(fields: str) -> list[str] | None:
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0].split(", ")
    except (OSError, IndexError, subprocess.TimeoutExpired):
        return None


def _old_lib(path: str):
    lib = C.CDLL(os.path.abspath(path))
    vp, i32, i64 = C.c_void_p, C.c_int, C.c_longlong
    for name, res, args in (("b200_window_attention_tc_bias_bytes", i64, [i32, i32, i32]),
                            ("b200_window_attention_tc_pack_bias", i32, [vp, i32, i32, i32, i32, i32, vp, i32, vp, vp]),
                            ("b200_window_attention_tc", i32, [vp, i32, i32, i32, i32, i32, vp, vp, i32, vp, vp]),
                            ("b200_last_error", C.c_char_p, [])):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--old-lib", default=None, help="a second libmonai_b200.so whose b200_window_attention_tc is timed as `old_tc`")
    ap.add_argument("--min-seconds", type=float, default=1.0, help="timed launches per variant cover at least this much device time")
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("window_attention_shapes.py needs a CUDA device")
    from weights import fill_state_dict

    from monai_b200 import _kernels as K
    from monai_b200 import _lib as L
    from monai_b200.networks.nets import SwinUNETR

    dev = torch.device("cuda", 0)
    L.load()
    old = _old_lib(args.old_lib) if args.old_lib else None
    net = SwinUNETR(in_channels=1, out_channels=2, feature_size=48)
    net.load_state_dict(fill_state_dict(net.state_dict(), 1))
    net = net.eval().to(dev).half()
    net._graph_enabled = False   # one eager forward: every launch goes through the Python entry point

    packs, calls, order = {}, {}, []
    orig_pack, orig_tc = K.window_attention_tc_pack_bias, K.window_attention_tc

    def recording_pack(table, heads, n, window, region_types, ntypes):
        pb = orig_pack(table, heads, n, window, region_types, ntypes)
        packs[pb.data_ptr()] = (table, tuple(window), region_types)
        return pb

    def recording_tc(qkv, Cc, heads, nW, n, packed_bias, sched, ntypes):
        key = (qkv.N, Cc, heads, nW, n, ntypes)
        if key not in calls:
            calls[key] = {"count": 0, "args": (qkv, Cc, heads, nW, n, packed_bias, sched, ntypes)}
            order.append(key)
        calls[key]["count"] += 1
        return orig_tc(qkv, Cc, heads, nW, n, packed_bias, sched, ntypes)

    x_in = torch.randn((SW_BATCH, 1, *ROI), generator=torch.Generator().manual_seed(0)).half().to(dev)
    K.window_attention_tc_pack_bias, K.window_attention_tc = recording_pack, recording_tc
    try:
        with torch.no_grad():
            net(x_in)
    finally:
        K.window_attention_tc_pack_bias, K.window_attention_tc = orig_pack, orig_tc
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

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    steps_per_forward = WINDOWS // SW_BATCH
    rows, sums = [], {"tc": 0.0, "old_tc": 0.0, "nc8": 0.0}
    for key in order:
        N, Cc, heads, nW, n, ntypes = key
        qkv, _, _, _, _, pb, sched, _ = calls[key]["args"]
        table, window, reps = packs[pb.data_ptr()]
        stream = L.stream_ptr(dev)
        out = K.NC8(N, Cc, qkv.sp, dev)
        lib = L.load()
        ms = {"tc": timeit(lambda: L.check(lib.b200_window_attention_tc(L.ptr(qkv.buf), N, Cc, heads, nW, n, L.ptr(pb), L.ptr(sched),
                                                                          ntypes, L.ptr(out.buf), stream), "window_attention_tc"))}
        if old is not None:
            nbytes = old.b200_window_attention_tc_bias_bytes(heads, n, ntypes)
            opb = torch.empty(nbytes // 2, dtype=torch.float16, device=dev)
            tab = table.detach().float().contiguous()
            assert old.b200_window_attention_tc_pack_bias(L.ptr(tab), heads, n, *window, L.ptr(reps), ntypes, L.ptr(opb), stream) == 0

            def run_old():
                if old.b200_window_attention_tc(L.ptr(qkv.buf), N, Cc, heads, nW, n, L.ptr(opb), L.ptr(sched), ntypes, L.ptr(out.buf), stream):
                    raise RuntimeError(old.b200_last_error().decode())

            ms["old_tc"] = timeit(run_old)
        # the mma.sync kernel on the same windows: region rows rebuilt from the schedule (one representative row per type;
        # equal rows <=> equal masks), scale 1 / log2(e) so it exponentiates the same scores as the pre-scaled tc path
        region = None
        if reps is not None:
            s = sched.cpu().numpy()
            r = np.empty((nW, n), dtype=np.int32)
            rp = reps.cpu().numpy()
            for t in range(ntypes):
                r[s[16 + s[8 + t]: 16 + s[8 + t] + s[t]]] = rp[t]
            region = torch.from_numpy(r).to(dev)
        ms["nc8"] = timeit(lambda: K.window_attention_nc8(qkv, Cc, heads, nW, n, 1.0 / K.LOG2E, table, window, region))

        lps = calls[key]["count"] * steps_per_forward
        n_pad, nrt, nrt_old = (n + 31) // 32 * 32, (n + ROWS - 1) // ROWS, (n + 127) // 128
        pairs = N * nW * heads
        ex2_alg = pairs * n * n
        ex2_pad = pairs * ((n + 15) // 16 * 16) * n_pad            # warps with a valid row, padded keys
        ex2_pad_old = pairs * nrt_old * 128 * n_pad                # every warp of every 128-row tile
        tiles = pairs * nrt
        row = {"N": N, "C": Cc, "heads": heads, "nW": nW, "n": n, "mask_types": ntypes, "tiles": tiles,
               "launches_per_step": lps, "ms_per_launch": {k: round(v, 4) for k, v in ms.items()},
               "ex2_alg_per_launch": ex2_alg, "ex2_padded_per_launch": ex2_pad, "ex2_padded_per_launch_old": ex2_pad_old,
               # q, k, v read once and the output written once; the old tile order read k and v once per row tile
               "hbm_bytes_per_launch": N * nW * n * 4 * Cc * 2, "hbm_bytes_per_launch_old": N * nW * n * (2 + 2 * nrt_old) * Cc * 2,
               # bias image reloads (L2 -> shared memory): about one per schedule group and one at each CTA's start
               "bias_l2_bytes_per_launch": ((tiles // GROUP if nrt > 1 else 0) + min(tiles, sms)) * n_pad * 2 * ROWS}
        for k, v in ms.items():
            sums[k] += v * lps
        rows.append(row)

    pl = _smi("power.limit,clocks.max.sm")
    timeit(lambda: orig_tc(*calls[order[0]]["args"]))   # keep the card loaded, then read the SM clock it runs at
    clk = _smi("clocks.sm")
    sm_mhz = float(clk[0]) if clk else None
    card = {"name": torch.cuda.get_device_name(0), "sms": sms, "power_limit_w": float(pl[0]) if pl else None,
            "sm_max_mhz": float(pl[1]) if pl else None, "sm_mhz_loaded": sm_mhz}
    if sm_mhz:
        rate = MUFU_PER_CLK_SM * sms * sm_mhz * 1e6
        for row in rows:
            for k, v in row["ms_per_launch"].items():
                row.setdefault("ex2_alg_per_s", {})[k] = float(f"{row['ex2_alg_per_launch'] / (v * 1e-3):.4g}")
            row["mufu_floor_ms_alg"] = round(row["ex2_alg_per_launch"] / rate * 1e3, 4)
            row["mufu_floor_ms_padded"] = round(row["ex2_padded_per_launch"] / rate * 1e3, 4)
            row["tc_share_of_mufu_alg"] = round(row["mufu_floor_ms_alg"] / row["ms_per_launch"]["tc"], 3)
            row["tc_share_of_mufu_padded"] = round(row["mufu_floor_ms_padded"] / row["ms_per_launch"]["tc"], 3)
    print(json.dumps({"workload": "swin_c3 window attention per call shape", "card": card, "sw_batch": SW_BATCH,
                      "mufu_ex2_per_clk_per_sm": MUFU_PER_CLK_SM, "l2": "256 MiB flush write before every timed launch",
                      "ms_per_step_sum": {k: round(v, 1) for k, v in sums.items() if v}, "shapes": rows}))


if __name__ == "__main__":
    main()
