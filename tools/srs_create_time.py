#!/usr/bin/env python3
"""Time of `SRS::create(depth)` on the device: one zk_srs_generate call, which hashes g[0..depth) and h to the curve and makes g
resident.

Depths 2^16 and 2^20 on both curves, with window_bits = 0 (generation and the resident copy only) and with the default window
(plus the window table every MSM over the SRS then uses).  The host outputs are not requested, so the time is that of the device
work; the call ends in a synchronisation of the library's stream, and a host clock brackets it.  Best of REPS after WARMUP calls.
Before timing, the 2^16 prefix of each curve is checked against the generators the reference ships (tests/golden).  Prints the
card and its power limit, then one JSON document; exits non-zero without a GPU or on a mismatch."""
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEPTHS = (1 << 16, 1 << 20)
WINDOWS = (0, -1)
WARMUP, REPS = 2, 7


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


def check_prefix(ctx, zk, orc, curve, name):
    z = np.load(os.path.join(ROOT, "tests", "golden", f"{name}_srs.npz"))
    with zk.SRS.create(ctx, curve, 1 << 16) as srs:
        if not np.array_equal(ctx.compress_points(curve, srs.g), z["g_cmp"]):
            raise SystemExit(f"mismatch: {name} generators")
        if not np.array_equal(orc.from_mont(orc.BASE_FIELD[curve], srs.h.reshape(2, 4)).view(np.uint8).reshape(64), z["h_xy"]):
            raise SystemExit(f"mismatch: {name} h")


def time_create(ctx, zk, curve, depth, window_bits):
    from proof_systems_b200._lib import check
    L = zk.lib()
    times = []
    for rep in range(WARMUP + REPS):
        h = ctypes.c_void_p()
        t0 = time.perf_counter()
        check(L.zk_srs_generate(ctx._h, curve, depth, window_bits, None, None, ctypes.byref(h)))
        t1 = time.perf_counter()
        L.zk_srs_destroy(h)
        if rep >= WARMUP:
            times.append((t1 - t0) * 1e3)
    return {"depth": depth, "window_bits": window_bits, "best_ms": round(min(times), 3), "median_ms": round(sorted(times)[len(times) // 2], 3)}


def main():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device")
    import proof_systems_b200 as zk
    from oracle import oracle as orc
    orc.lib()
    print(f"card: {card()}")
    rows = []
    with zk.Context(0) as ctx:
        for curve, name in ((zk.PALLAS, "pallas"), (zk.VESTA, "vesta")):
            check_prefix(ctx, zk, orc, curve, name)
            for depth in DEPTHS:
                for wb in WINDOWS:
                    rows.append({"curve": name, **time_create(ctx, zk, curve, depth, wb)})
    print(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
