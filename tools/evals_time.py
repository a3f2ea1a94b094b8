#!/usr/bin/env python3
"""Time of the prover's evaluation step at zeta and zeta*omega (kimchi/src/prover.rs:1009-1058) on device-resident columns.

Two configurations: d1 = 2^16 with max_poly_size = 2^16 (one chunk), and d1 = 2^17 with max_poly_size = 2^16 (two chunks, the
reference's chunked `heavy` configuration).  Per repetition:
  basis     two zk_lagrange_evals_dev calls (zeta, zeta*omega), then a device synchronisation
  columns   one zk_lagrange_evaluate_dev call: 22 d8 columns (7 permutation_coefficients8 + 15 coefficients8) and 6 selectors
            (generic and complete_add over d4; poseidon, mul, emul, endomul_scalar over d8) at both points
  coeffs    one zk_poly_evaluate_chunks_dev call: 17 coefficient vectors of d1 elements (15 witness, z, public) at both points,
            num_chunks = d1 / max_poly_size
Host clock around work that ends in a synchronisation; median of REPS after WARMUP repetitions.  Column data is random (valid
Montgomery limbs).  One result is checked against a Python-integer Horner evaluation (the CPU oracle converts from Montgomery
form), and the first d8 column is the FFT(8 d1) of the first coefficient vector so that its Lagrange evaluation must equal that
vector's chunk evaluations.  Prints the card and its power limit, then one JSON document; exits non-zero without a GPU or on a
mismatch."""
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = ((16, 1 << 16), (17, 1 << 16))
WARMUP, REPS = 3, 20


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


def run(ctx, zk, orc, torch, log_n, max_poly_size):
    fid, n = zk.FP, 1 << log_n
    P = orc.FP_MODULUS
    rng = np.random.default_rng(log_n)
    chunks = zk.Context.lagrange_evals_chunks(n, max_poly_size)
    bufs = []

    def put(a):
        p = ctx.dev_alloc(a.nbytes)
        bufs.append(p)
        ctx.dev_upload(p, a)
        return p

    try:
        d_coeffs = put(rand_fe(rng, 17 * n))                                     # w_0..w_14, z, public: coefficients
        d8 = put(rand_fe(rng, 22 * 8 * n))                                        # s (7) + coefficients8 (15) over d8
        ctx.ntt_dev_oop(fid, d_coeffs, n, n, d8, log_n + 3, batch=1)              # column 0 := w_0 over d8
        one = orc.fe(fid, 1)
        sel = [put(np.where(rng.integers(0, 2, size=(k * n, 1)) == 1, one, np.uint64(0)).astype(np.uint64)) for k in (4, 4, 8, 8, 8, 8)]
        sel_len = [k * n for k in (4, 4, 8, 8, 8, 8)]
        zeta = orc.fe(fid, int(rng.integers(1, 2**62)) * 2**190 + 12345)
        omega = orc.root_of_unity(fid, log_n)
        pts = np.stack([zeta, orc.fe_mul(fid, zeta, omega)])
        d_bases = [ctx.dev_alloc(chunks * n * 32) for _ in range(2)]
        bufs += d_bases
        columns = [(d8 + k * 8 * n * 32, 8 * n, False) for k in range(22)] + [(p, ln, True) for p, ln in zip(sel, sel_len)]
        polys = [(d_coeffs + j * n * 32, n) for j in range(17)]
        times = {"basis": [], "columns": [], "coeffs": [], "total": []}
        for rep in range(WARMUP + REPS):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for b, x in zip(d_bases, pts):
                ctx.lagrange_basis_evals_dev(fid, log_n, max_poly_size, x, b)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            lag = ctx.lagrange_evaluate_dev(fid, d_bases, log_n, chunks, columns)
            t2 = time.perf_counter()
            chk = ctx.poly_evaluate_chunks_dev(fid, polys, chunks, max_poly_size, pts)
            t3 = time.perf_counter()
            if rep >= WARMUP:
                for k, v in zip(("basis", "columns", "coeffs", "total"), (t1 - t0, t2 - t1, t3 - t2, t3 - t0)):
                    times[k].append(v * 1e3)
        # checks: w_0's chunks at zeta by Python Horner; its d8 column through the Lagrange path gives the same values
        w0 = ctx.dev_download(d_coeffs, (n, 4))
        raw = orc.from_mont(fid, w0).tobytes()
        c = [int.from_bytes(raw[k:k + 32], "little") for k in range(0, len(raw), 32)]
        x = orc.fe_int(fid, zeta)
        for k in range(chunks):
            acc = 0
            for v in reversed(c[k * max_poly_size:(k + 1) * max_poly_size]):
                acc = (acc * x + v) % P
            if orc.fe_int(fid, chk[0, 0, k]) != acc:
                raise SystemExit(f"mismatch: chunk {k} of w_0 at zeta (d1 = 2^{log_n})")
        if not np.array_equal(lag[0], chk[0]):
            raise SystemExit(f"mismatch: Lagrange and coefficient evaluations of w_0 (d1 = 2^{log_n})")
    finally:
        for p in bufs:
            ctx.dev_free(p)
    return {"d1": n, "max_poly_size": max_poly_size, "chunks": chunks, "columns": len(columns), "polys": len(polys), "points": 2,
            **{f"{k}_ms": round(statistics.median(v), 4) for k, v in times.items()}, "check": "ok"}


def main():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device")
    import proof_systems_b200 as zk
    from oracle import oracle as orc
    print(f"card: {card()}")
    ctx = zk.Context(0)
    try:
        rows = [run(ctx, zk, orc, torch, log_n, m) for log_n, m in CONFIGS]
    finally:
        ctx.close()
    print(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
