#!/usr/bin/env python3
"""Time of the ft polynomial of Maller's optimisation (kimchi/src/prover.rs:1147-1206) on device-resident inputs: one
zk_prover_ft_dev call.

Two prover shapes: d1 = 2^16 with max_poly_size = 2^16 (t: 7 chunks), and d1 = 2^17 with max_poly_size = 2^16 (two chunks, t: 14
chunks).  Inputs as kimchi passes them: ONE term, sigma_6 over d8 (8 d1 evaluations) with perm_scalar, and the quotient t at its
full length of 7 num_chunks max_poly_size coefficients.  CUDA events bracket each call (the call itself ends in a synchronisation
of the library's stream); median of REPS after WARMUP calls.  Data are random valid Montgomery limbs.  Every configuration's
output (the max_poly_size coefficients, ft_len and ft(zeta omega)) is checked against the Python restatement tests/ft_replay.py
at the timed size.  Prints the card and its power limit, then one JSON document; exits non-zero without a GPU or on a mismatch."""
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CONFIGS = ((16, 1 << 16), (17, 1 << 16))
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


def run(ctx, zk, orc, torch, log_n, m):
    import evals_replay as ev
    import ft_replay as fr
    fid, n = zk.FP, 1 << log_n
    P = orc.MODULUS[fid]
    nc = fr.num_chunks(n, m)
    rng = np.random.default_rng(log_n)
    s8, t = rand_fe(rng, 8 * n), rand_fe(rng, 7 * nc * m)
    perm, zeta = rand_fe(rng, 1)[0], rand_fe(rng, 1)[0]
    bufs = []

    def put(a):
        p = ctx.dev_alloc(a.nbytes)
        bufs.append(p)
        ctx.dev_upload(p, a)
        return p

    try:
        d_s8, d_t = put(s8), put(t)
        d_ft = ctx.dev_alloc(m * 32)
        bufs.append(d_ft)
        terms = [(d_s8, 8 * n, perm)]
        times = []
        for rep in range(WARMUP + REPS):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ft_len, ft_eval1 = ctx.prover_ft_dev(fid, log_n, m, terms, d_t, t.shape[0], zeta, d_ft)
            e1.record()
            e1.synchronize()
            if rep >= WARMUP:
                times.append(e0.elapsed_time(e1))
        got = ctx.dev_download(d_ft, (m, 4))
    finally:
        for p in bufs:
            ctx.dev_free(p)
    # the restatement at the timed size
    ints = lambda a: ev.ints(orc, fid, a)
    _, want, want_e1 = fr.ft(orc, fid, log_n, m, [(ints(s8), ints(perm)[0])], ints(t), ints(zeta)[0])
    if ft_len != len(want) or not np.array_equal(got[:ft_len], ev.mont(orc, fid, want)) or got[ft_len:].any():
        raise SystemExit(f"mismatch: ft coefficients (d1 = 2^{log_n}, max_poly_size = {m})")
    if not np.array_equal(ft_eval1, ev.mont(orc, fid, [want_e1])[0]):
        raise SystemExit(f"mismatch: ft(zeta omega) (d1 = 2^{log_n}, max_poly_size = {m})")
    return {"d1": n, "max_poly_size": m, "chunks": nc, "t_len": int(t.shape[0]), "ft_len": ft_len,
            "median_ms": round(statistics.median(times), 4), "min_ms": round(min(times), 4), "max_ms": round(max(times), 4), "check": "ok"}


def main():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device")
    import proof_systems_b200 as zk
    from oracle import oracle as orc
    orc.lib()
    print(f"card: {card()}")
    ctx = zk.Context(0)
    try:
        rows = [run(ctx, zk, orc, torch, log_n, m) for log_n, m in CONFIGS]
    finally:
        ctx.close()
    print(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
