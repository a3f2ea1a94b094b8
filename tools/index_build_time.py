#!/usr/bin/env python3
"""Time of building kimchi's prover index on the device (zk_index_build: the column evaluations of constraints.rs:510-760) and of its
verifier-index commitments (zk_index_commitments: 28 + k commit_evaluations_non_hiding of verifier_index.rs:221-300), for Vesta
(scalar field Fp) over the fixture's 2^16 generators, in three shapes: d1 = 2^16 (one chunk), 2^17 and 2^20 (chunked: 2 and 16 chunks
per commitment).  The circuit has min(n - zk_rows, 2^17) gates of all 14 tags with random wires and 0 .. 20 coefficients, and every optional
selector (34 commitments).  Each call is timed on the host around the call (both end in a synchronisation); median of REPS after
WARMUP calls, with the Lagrange basis already built.  Launches are the context's counter over one call.  The CPU oracle restates the
same work (tests/index_replay.py: the columns, their FFTs and the MSMs) and its wall time is reported up to CPU_MAX_LOG; the device's
sections and commitments are checked against it there, and beyond it every section's d1 sub-sample is checked against the restated
d1 columns.  Prints the card and its power limit, then one JSON document; exits non-zero without a GPU or on a mismatch."""
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

LOGS = (16, 17, 20)
ZK_ROWS = 3
OPTIONAL = 0b111111
CPU_MAX_LOG = 17
MAX_GATES = 1 << 17        # gates past the list are padding; the device's work does not depend on the count
WARMUP, REPS = 2, 5


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


def timed(ctx, call, release=None):
    times, launches, out = [], 0, None
    for rep in range(WARMUP + REPS):
        if release and out is not None:
            release(out)
        l0 = ctx.launch_count
        t0 = time.perf_counter()
        out = call()
        times.append((time.perf_counter() - t0) * 1e3)
        launches = ctx.launch_count - l0
    return out, statistics.median(times[WARMUP:]), launches


def main():
    import torch
    if not torch.cuda.is_available():
        print("no CUDA device", file=sys.stderr)
        return 2
    import evals_replay as ev
    import index_replay as ir
    import proof_systems_b200 as zk
    from conftest import GoldenSRS
    from oracle import oracle as orc
    from test_gpu_index_build import circuit
    orc.lib()
    golden = GoldenSRS("vesta", orc)
    fid = orc.SCALAR_FIELD[golden.cid]
    print(f"card: {card()}")
    ctx = zk.Context(0)
    srs = zk.SRS(ctx, golden.cid, golden.g, golden.mont_points(golden.h_xy_canon.reshape(1, 64))[0])
    results, ok = [], True
    for log_n in LOGS:
        n = 1 << log_n
        n_gates = min(n - ZK_ROWS, MAX_GATES)
        gates, shifts = circuit(orc, fid, n, n_gates, seed=log_n)
        hdr = ir.header(zk, n, ZK_ROWS, ev.mont(orc, fid, shifts), OPTIONAL)
        g, c = ir.pruned_gates(gates), ir.gate_coeffs(orc, fid, gates)
        srs.get_lagrange_basis_from_domain_size(n)
        idx, t_build, l_build = timed(ctx, lambda: zk.IndexCache.build(ctx, fid, hdr, g, c), release=lambda i: i.close())
        comms, t_comm, l_comm = timed(ctx, lambda: srs.index_commitments(idx))
        row = {"log_n": log_n, "gates": n_gates, "chunks": comms.shape[1], "commitments": comms.shape[0], "build_ms": round(t_build, 3), "build_launches": l_build,
               "commitments_ms": round(t_comm, 3), "commitments_launches": l_comm}
        t0 = time.perf_counter()
        cols = ir.columns_d1(orc, fid, n, ZK_ROWS, gates, shifts, OPTIONAL)
        if log_n <= CPU_MAX_LOG:
            secs = {t: (cols[t] if ir.domain_mult(t) == 1 else ir.evaluate(orc, fid, cols[t], ir.domain_mult(t))) for t in cols}
            want = ir.commitments(orc, golden.cid, golden.g, srs.h, cols, OPTIONAL)
            row["cpu_oracle_s"] = round(time.perf_counter() - t0, 2)
            good = np.array_equal(comms, want)
            for t, a in secs.items():
                p, n_el, _ = idx.section(t)
                good &= np.array_equal(ctx.dev_download(p, (n_el, 4)), a)
        else:
            row["cpu_oracle_s"] = "not measured"
            good = True
            for t, a in cols.items():
                p, n_el, _ = idx.section(t)
                m = ir.domain_mult(t)
                good &= np.array_equal(ctx.dev_download(p, (n_el, 4))[::m], a)
        row["checked"] = bool(good)
        ok &= bool(good)
        results.append(row)
        idx.close()
    srs.close()
    ctx.close()
    print(json.dumps({"card": card(), "field": "Fp (Vesta scalars)", "srs": golden.g.shape[0], "zk_rows": ZK_ROWS,
                      "optional_selectors": OPTIONAL, "results": results}, indent=1))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
