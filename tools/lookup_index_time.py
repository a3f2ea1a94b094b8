#!/usr/bin/env python3
"""Time of building kimchi's lookup index on the device (zk_lookup_index_build: LookupConstraintSystem::create, lookup/index.rs:202-482)
and of its verifier-index commitments (zk_lookup_index_commitments: LookupVerifierIndex, verifier_index.rs:196-215), for Vesta (scalar
field Fp) over the fixture's 2^16 generators at d1 = 2^16 (one chunk), 2^17 and 2^20 (2 and 16 chunks per commitment).  The circuit uses
all four lookup patterns (Lookup, Xor16, RangeCheck0/1, Rot64, ForeignFieldMul gates on its first 2^16 rows), a 2^10-row user table of id
2 and one 64-row runtime table: 3 table columns, table ids, 4 selectors and the runtime selector (9 sections, 9 commitments).  Each call is
timed on the host around the call (both end in a synchronisation); median of REPS after WARMUP calls, with the Lagrange basis already
built.  Every section's d1 sub-sample is checked against the restated d1 columns (tests/lookup_index_replay.py).  Prints the card and its
power limit, then one JSON document; exits non-zero without a GPU or on a mismatch."""
import json
import os
import random
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
MAX_GATES = 1 << 16
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
    import lookup_index_replay as li
    import proof_systems_b200 as zk
    from conftest import GoldenSRS
    from oracle import oracle as orc
    from test_gpu_lookup_index import circuit, gates_of
    orc.lib()
    golden = GoldenSRS("vesta", orc)
    fid = orc.SCALAR_FIELD[golden.cid]
    P = orc.MODULUS[fid]
    print(f"card: {card()}")
    ctx = zk.Context(0)
    srs = zk.SRS(ctx, golden.cid, golden.g, golden.mont_points(golden.h_xy_canon.reshape(1, 64))[0])
    rng = random.Random(1)
    user = (2, [[rng.randrange(P) for _ in range(1 << 10)] for _ in range(2)])
    runtime = [(9, [rng.randrange(P) for _ in range(64)])]
    tables_mont = [(user[0], li.mont_table(orc, fid, user[1]))]
    runtime_mont = [(tid, ev.mont(orc, fid, c)) for tid, c in runtime]
    results, ok = [], True
    for log_n in LOGS:
        n = 1 << log_n
        tags = circuit(n, "all", seed=log_n, n_gates=min(n - ZK_ROWS - 1, MAX_GATES))
        g = gates_of(tags)
        srs.get_lagrange_basis_from_domain_size(n)
        (idx, offset), t_build, l_build = timed(ctx, lambda: zk.IndexCache.build_lookup(ctx, fid, n, ZK_ROWS, g, tables_mont, runtime_mont),
                                                release=lambda r: r[0].close())
        comms, t_comm, l_comm = timed(ctx, lambda: srs.lookup_index_commitments(idx))
        res = li.create(P, n, ZK_ROWS, tags, [user], runtime)
        good = offset == res["runtime_table_offset"] and idx.header.lookup_selectors_present == li.header_bits(res)
        p50, _, w = idx.section(0x50)
        for k, (tag, c) in enumerate(li.columns(res)):
            p = p50 + k * 8 * n * 32 if tag == 0x50 else idx.section(tag)[0]
            good &= np.array_equal(ctx.dev_download(p, (8 * n, 4))[::8], ev.mont(orc, fid, c))
        row = {"log_n": log_n, "gates": len(tags), "columns": w, "sections": idx.header.num_sections, "chunks": comms.shape[1],
               "commitments": comms.shape[0], "build_ms": round(t_build, 3), "build_launches": l_build, "commitments_ms": round(t_comm, 3),
               "commitments_launches": l_comm, "checked": bool(good)}
        ok &= bool(good)
        results.append(row)
        idx.close()
    srs.close()
    ctx.close()
    print(json.dumps({"card": card(), "field": "Fp (Vesta scalars)", "srs": golden.g.shape[0], "zk_rows": ZK_ROWS, "user_table_rows": 1 << 10,
                      "runtime_table_rows": 64, "results": results}, indent=1))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
