#!/usr/bin/env python3
"""Time of the recursion accumulators on the device: zk_srs_accumulator_check and zk_srs_accumulator_generate
(batch_dlog_accumulator_check / _generate, poly-commitment/src/utils.rs:204-312) over a 2^16-point SRS with the default window table.

Both curves; the check at k in {1, 16, 256, 1024} accumulators of 16 rounds, generate at k in {1, 16, 64}.  Each call ends in a
synchronisation, so a host clock brackets it (the Python call, including its argument marshalling); median and spread (min .. max)
of REPS calls after WARMUP.  Where it is cheap (k <= 16) every device result is checked against the CPU restatement
(tests/accumulator_replay.py), whose single-run host time is printed as the oracle's: Python scalars and the C oracle's MSM, not the
reference's Rust.  Prints the card and its power limit, then one JSON document; exits non-zero without a GPU or on a mismatch."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

LOG_N = 16
ROUNDS = LOG_N
CHECK_K = (1, 16, 256, 1024)
GENERATE_K = (1, 16, 64)
VERIFIED_K = 16
WARMUP, REPS = 3, 15
R = 0x1234567890ABCDEF1234567890ABCDEF


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


def timed(fn):
    times = []
    for rep in range(WARMUP + REPS):
        t0 = time.perf_counter()
        out = fn()
        t1 = time.perf_counter()
        if rep >= WARMUP:
            times.append((t1 - t0) * 1e3)
    times.sort()
    return out, {"median_ms": round(times[len(times) // 2], 3), "min_ms": round(times[0], 3), "max_ms": round(times[-1], 3)}


def main():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device")
    import accumulator_replay as acc
    import proof_systems_b200 as zk
    from oracle import oracle as orc
    orc.lib()
    print(f"card: {card()}")
    rows = []
    with zk.Context(0) as ctx:
        for curve, name in ((zk.PALLAS, "pallas"), (zk.VESTA, "vesta")):
            fid = orc.SCALAR_FIELD[curve]
            with zk.SRS.create(ctx, curve, 1 << LOG_N) as srs:
                g = srs.g
                ints = acc.random_chals(orc, fid, max(CHECK_K + GENERATE_K) * ROUNDS, seed=1)
                chals = acc.mont(orc, fid, ints)
                r = acc.mont(orc, fid, [R])[0]
                for k in GENERATE_K:
                    out, t = timed(lambda: zk.batch_dlog_accumulator_generate(srs, k, chals[: k * ROUNDS]))
                    row = {"curve": name, "call": "generate", "k": k, **t}
                    if k <= VERIFIED_K:
                        t0 = time.perf_counter()
                        want = acc.generate(orc, curve, g, k, ints[: k * ROUNDS])
                        row["oracle_restatement_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
                        if not np.array_equal(out, want):
                            raise SystemExit(f"mismatch: {name} generate k={k}")
                    rows.append(row)
                comms = zk.batch_dlog_accumulator_generate(srs, max(CHECK_K), chals[: max(CHECK_K) * ROUNDS])
                for k in CHECK_K:
                    (ok, pt), t = timed(lambda: zk.batch_dlog_accumulator_check(srs, comms[:k], chals[: k * ROUNDS], r, return_sum=True))
                    if not ok or pt.any():
                        raise SystemExit(f"an honest batch failed: {name} check k={k}")
                    row = {"curve": name, "call": "check", "k": k, **t}
                    if k <= VERIFIED_K:
                        t0 = time.perf_counter()
                        if not acc.check(orc, curve, g, comms[:k], ints[: k * ROUNDS], R):
                            raise SystemExit(f"mismatch: {name} check k={k}")
                        row["oracle_restatement_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
                    rows.append(row)
    print(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
