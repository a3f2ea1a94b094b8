#!/usr/bin/env python3
"""Time of the lookup argument's three device calls (kimchi's joint table, lookup::constraints::sorted and aggregation) on
device-resident inputs: zk_lookup_joint_table_dev, zk_lookup_sorted_dev and zk_lookup_aggreg_dev.

Three shapes with m = max_per_row = 4: d1 = 2^16 with zk_rows = 3, d1 = 2^17 with zk_rows = 5 and d1 = 2^20 with zk_rows = 3.  The
joint table combines 3 table columns and the table ids over d8; the sorted and aggregation calls read the witness's 15 columns and
the table at stride 8 from a valid instance of tests/lookup_replay.py (kimchi's four patterns and a synthetic one, about 70 % of
the rows with lookups).  The context runs on torch's current stream and CUDA events bracket each call there (the joint table
returns with its work queued; the sorted and aggregation calls end in a synchronisation); median of REPS after WARMUP calls.
Every output is checked against the Python restatement at the timed size (the joint table at its d1 points beyond 2^17).  Prints the card and its power limit, then one JSON document; exits non-zero without a GPU or
on a mismatch."""
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
M = 4
WARMUP, REPS = 3, 20


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


def timed(torch, call):
    times, out = [], None
    for rep in range(WARMUP + REPS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = call()
        e1.record()
        e1.synchronize()
        if rep >= WARMUP:
            times.append(e0.elapsed_time(e1))
    return out, {"median_ms": round(statistics.median(times), 4), "min_ms": round(min(times), 4), "max_ms": round(max(times), 4)}


def run(ctx, zk, orc, torch, log_n, zk_rows):
    import evals_replay as ev
    import lookup_replay as lr
    fid, n = zk.FP, 1 << log_n
    P = orc.MODULUS[fid]
    mont = lambda xs: ev.mont(orc, fid, [int(x) for x in xs])
    inst = lr.instance(P, log_n, zk_rows, M, seed=log_n)
    spec = zk.LookupSpec(fid, M)
    for pat in inst.patterns:
        spec.add_pattern([(tid, [[(None if c is None else mont([c])[0], col, nxt) for c, col, nxt in e] for e in entries]) for tid, entries in pat])
    info = spec.info(np.array(inst.row_pattern, dtype=np.uint8), *mont([inst.jc, inst.tic, inst.dummy]))
    cols8 = [orc.to_mont(fid, orc.random_scalars(fid, 8 * n, seed=k)) for k in range(4)]
    t8 = orc.to_mont(fid, orc.random_scalars(fid, 8 * n, seed=9))
    t8[::8] = mont(inst.T1)
    bufs = []

    def put(a):
        a = np.ascontiguousarray(a, dtype=np.uint64)
        p = ctx.dev_alloc(a.nbytes)
        bufs.append(p)
        ctx.dev_upload(p, a)
        return p

    row = {"d1": n, "zk_rows": zk_rows, "m": M}
    try:
        d_c = [put(c) for c in cols8[:3]]
        d_ids = put(cols8[3])
        d_o8, d_o1 = put(np.zeros((8 * n, 4))), put(np.zeros((n, 4)))
        d_w = [put(mont(c)) for c in inst.w]
        d_t = put(t8)
        d_s = [put(np.zeros((n, 4))) for _ in range(M + 1)]
        d_a = put(np.zeros((n, 4)))
        jc, tic = mont([inst.jc, inst.tic])
        b, g = mont([inst.beta, inst.gamma])
        rs, ra = mont(inst.rand_sorted), mont(inst.rand_agg)
        _, row["joint_table"] = timed(torch, lambda: ctx.lookup_joint_table_dev(fid, log_n, d_c, jc, tic, d_o8, d_ids, None, d_o1))
        bad, row["sorted"] = timed(torch, lambda: ctx.lookup_sorted_dev(fid, log_n, zk_rows, d_w, d_t, 8, info, rs, d_s))
        ok, row["aggreg"] = timed(torch, lambda: ctx.lookup_aggreg_dev(fid, log_n, zk_rows, d_w, d_t, 8, info, d_s, b, g, ra, d_a))
        got8, got1 = ctx.dev_download(d_o8, (8 * n, 4)), ctx.dev_download(d_o1, (n, 4))
        got_s = [ctx.dev_download(p, (n, 4)) for p in d_s]
        got_a = ctx.dev_download(d_a, (n, 4))
    finally:
        for p in bufs:
            ctx.dev_free(p)
    # the restatement at the timed size
    ints = lambda a: ev.ints(orc, fid, a)
    sub = slice(None) if log_n <= 17 else slice(None, None, 8)
    want8 = mont(lr.joint_table([ints(c[sub]) for c in cols8[:3]], inst.jc, inst.tic, P, ints(cols8[3][sub])))
    if not np.array_equal(got8[sub], want8) or not np.array_equal(got1, got8[::8]):
        raise SystemExit(f"mismatch: joint table (d1 = 2^{log_n})")
    s = lr.sorted_patched(inst)
    agg, want_ok = lr.aggregation(inst, s)
    if bad != -1 or any(not np.array_equal(got_s[k], mont(s[k])) for k in range(M + 1)):
        raise SystemExit(f"mismatch: sorted (d1 = 2^{log_n})")
    if ok != want_ok or not np.array_equal(got_a, mont(agg)):
        raise SystemExit(f"mismatch: aggregation (d1 = 2^{log_n})")
    row["check"] = "ok"
    return row


def main():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device")
    import proof_systems_b200 as zk
    from oracle import oracle as orc
    orc.lib()
    print(f"card: {card()}")
    ctx = zk.Context(0)
    ctx.set_stream(torch.cuda.current_stream().cuda_stream)      # the events' stream: the joint table returns with work queued
    try:
        rows = [run(ctx, zk, orc, torch, log_n, zk_rows) for log_n, zk_rows in CONFIGS]
    finally:
        ctx.close()
    print(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
