#!/usr/bin/env python3
"""Time of the permutation aggregation polynomial z (kimchi's ProverIndex::perm_aggreg) on device-resident inputs: one
zk_perm_aggreg_dev call.

Three shapes: d1 = 2^16 with zk_rows = 3, d1 = 2^17 with zk_rows = 5 (a two-chunk proof) and d1 = 2^20 with zk_rows = 3.  Inputs as
kimchi passes them: the 7 witness columns over d1 and permutation_coefficients8 (8 d1 evaluations per column, read at stride 8).
CUDA events bracket each call (the call itself ends in a synchronisation of the library's stream); median of REPS after WARMUP
calls.  Data are random valid Montgomery limbs, so the final-value check fails and every row's ratio is a random element; z is
written either way.  Every shape's output (z's coefficients and the flag) is checked against the Python restatement
tests/perm_replay.py at the timed size.  Prints the card and its power limit, then one JSON document; exits non-zero without a GPU
or on a mismatch."""
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CONFIGS = ((16, 3), (17, 5), (20, 3))
WARMUP, REPS = 5, 50


def rand_fe(rng, k):
    a = rng.integers(0, 2**64, size=(k, 4), dtype=np.uint64)
    a[:, 3] &= np.uint64((1 << 62) - 1)                  # < 2^254 < both moduli: a valid Montgomery representation
    return a


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


def run(ctx, zk, orc, torch, log_n, zk_rows):
    import evals_replay as ev
    import perm_replay as pr
    fid, n = zk.FP, 1 << log_n
    rng = np.random.default_rng(log_n)
    w, s8 = rand_fe(rng, 7 * n).reshape(7, n, 4), rand_fe(rng, 7 * 8 * n).reshape(7, 8 * n, 4)
    beta, gamma, shifts, rand = rand_fe(rng, 1)[0], rand_fe(rng, 1)[0], rand_fe(rng, 7), rand_fe(rng, 2)
    with ctx.buffers() as bufs:
        d_w = [bufs.put(w[k]) for k in range(7)]
        d_s = [bufs.put(s8[k]) for k in range(7)]
        d_z = bufs.alloc(n * 32)
        times = []
        for rep in range(WARMUP + REPS):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ok = ctx.perm_aggreg_dev(fid, log_n, zk_rows, d_w, d_s, 8 * n, beta, gamma, shifts, rand, d_z)
            e1.record()
            e1.synchronize()
            if rep >= WARMUP:
                times.append(e0.elapsed_time(e1))
        launches0 = ctx.launch_count
        ctx.perm_aggreg_dev(fid, log_n, zk_rows, d_w, d_s, 8 * n, beta, gamma, shifts, rand, d_z)
        launches = ctx.launch_count - launches0
        got = ctx.dev_download(d_z, (n, 4))
    # the restatement at the timed size
    ints = lambda a: ev.ints(orc, fid, a)
    _, want, want_ok = pr.perm_aggreg(orc, fid, log_n, zk_rows, [ints(w[k]) for k in range(7)], [ints(s8[k][::8]) for k in range(7)],
                                      ints(shifts), ints(beta)[0], ints(gamma)[0], ints(rand))
    if ok != want_ok or not np.array_equal(got, ev.mont(orc, fid, want)):
        raise SystemExit(f"mismatch: z (d1 = 2^{log_n}, zk_rows = {zk_rows})")
    return {"d1": n, "zk_rows": zk_rows, "launches": launches, "median_ms": round(statistics.median(times), 4), "min_ms": round(min(times), 4),
            "max_ms": round(max(times), 4), "check": "ok"}


def main():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device")
    import proof_systems_b200 as zk
    from oracle import oracle as orc
    orc.lib()
    print(f"card: {card()}")
    with zk.Context(0) as ctx:
        rows = [run(ctx, zk, orc, torch, log_n, zk_rows) for log_n, zk_rows in CONFIGS]
    print(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
