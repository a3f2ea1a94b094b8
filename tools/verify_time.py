#!/usr/bin/env python3
"""Time of SRS::verify through zk_srs_verify at |g| = 2^16 (the fixture's Vesta generators), batches of 1, 8 and 64 proofs.

The proofs are made once by zk_srs_open under a stand-in transcript: every challenge is SHA-256 of what was absorbed so far (the
Montgomery limbs of cip, L, R, delta) reduced below the modulus, and U is one of 32 fixture points picked by that hash, so open and
verify derive the same challenges while the Python Poseidon stays out of the timing.  Each batch is timed with a host clock around
the (synchronous) call: median of REPS after WARMUP calls.  The split comes from the library's ZKB200_TRACE_VERIFY line (it adds one
stream synchronisation after the s-vector kernels): transcript callbacks, host scalars, s-vector kernels, g MSM, proof-point MSM.
The CPU side of the comparison is the oracle's MSM of the same size as the reference's final MSM (|g| + 1 + the proof points), with
every host thread.  Prints one JSON document; exits non-zero without a GPU or if any honest batch fails to verify."""
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["ZKB200_TRACE_VERIFY"] = "1"          # read once, at the library's first verify call

LOG_N, BATCHES, WARMUP, REPS = 16, (1, 8, 64), 2, 7
FP_MODULUS = 0x40000000000000000000000000000000224698fc094cf91b992d30ed00000001


def limbs(x):
    return np.array([(x >> (64 * i)) & (2**64 - 1) for i in range(4)], dtype=np.uint64)


class Transcript:
    def __init__(self, u_points, seed):
        self.u_points, self.h = u_points, hashlib.sha256(seed.to_bytes(8, "little"))

    def _absorb(self, *arrays):
        for a in arrays:
            self.h.update(np.ascontiguousarray(a, dtype=np.uint64).tobytes())
        return int.from_bytes(self.h.digest(), "little")

    def u_base(self, cip):
        return self.u_points[self._absorb(cip) % len(self.u_points)]

    def round(self, j, l, r):
        return limbs(self._absorb(l, r) % FP_MODULUS or 1)   # any value below the modulus is a Montgomery residue

    def final(self, delta):
        return limbs(self._absorb(delta) % FP_MODULUS)


def gpu_info():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"], info["max_sm_clock_mhz"] = float(out[0]), float(out[1])
    except Exception as e:                      # the numbers are still reported, the card's limit is then unknown
        info["power_limit_w"] = f"unavailable ({e})"
    return info


def main():
    import torch
    if not torch.cuda.is_available():
        sys.exit("verify_time: no CUDA device")
    import proof_systems_b200 as zk
    from bench import splitmix64_limbs
    from oracle import oracle as orc
    n = 1 << LOG_N
    ctx = zk.Context(0)
    z = np.load(os.path.join(ROOT, "tests", "golden", "vesta_srs.npz"))
    g = ctx.decompress_points(zk.VESTA, z["g_cmp"][:n])
    h = g[3]
    srs = zk.SRS(ctx, zk.VESTA, g, h)
    u_points = g[200:232]
    poly = splitmix64_limbs(5, n).reshape(n, 4)
    bl = splitmix64_limbs(6, 1).reshape(1, 4)
    comm = srs.commit_custom(poly, 1, bl).chunks
    entries = []
    t0 = time.perf_counter()
    for i in range(max(BATCHES)):
        sc = splitmix64_limbs(100 + i, 2 * LOG_N + 6).reshape(-1, 4)
        elm, ps, es, draws = sc[:2], sc[2], sc[3], sc[4:]
        tr, seen = Transcript(u_points, i), {}

        def u_base(cip, tr=tr, seen=seen):
            seen["cip"] = cip                  # the combined inner product, as the verifier receives it
            return tr.u_base(cip)
        proof = zk.srs_open(srs, [(poly, 0, bl)], elm, ps, es, draws, u_base, tr.round, tr.final)
        entries.append((proof, elm, ps, es, seen["cip"], i))
    t_open = time.perf_counter() - t0

    def batch(B):
        out = []
        for proof, elm, ps, es, cip, seed in entries[:B]:
            tr = Transcript(u_points, seed)
            out.append(zk.BatchEvaluationProof(proof, elm, ps, es, [comm], cip, tr.u_base, tr.round, tr.final))
        return out
    rb, sgb = splitmix64_limbs(7, 2).reshape(2, 4)
    rows = {"gpu": gpu_info(), "srs": f"Vesta, |g| = 2^{LOG_N} (fixture generators), default table window",
            "proofs_made_by_zk_srs_open_s": round(t_open, 3), "batches": {}}
    ok_all = True
    pat = re.compile(r"transcript callbacks ([\d.]+) ms \| host scalars ([\d.]+) \| s-vector kernels ([\d.]+) \| g MSM ([\d.]+) \| "
                     r"proof-point MSM ([\d.]+) \| total ([\d.]+) ms")
    for B in BATCHES:
        log = tempfile.TemporaryFile(mode="w+")
        saved = os.dup(2)
        sys.stderr.flush()
        os.dup2(log.fileno(), 2)
        ts = []
        try:
            for r in range(WARMUP + REPS):
                b = batch(B)
                torch.cuda.synchronize()
                t = time.perf_counter()
                ok = zk.srs_verify(srs, b, rb, sgb)
                ts.append(time.perf_counter() - t)
                ok_all &= ok
        finally:
            sys.stderr.flush()
            os.dup2(saved, 2)
            os.close(saved)
        log.seek(0)
        parts = np.array([[float(x) for x in m.groups()] for m in pat.finditer(log.read())][WARMUP:])
        med = np.median(parts, axis=0)
        n_pts = n + 1 + B * (2 * LOG_N + 4)
        cpu_sc = splitmix64_limbs(11, n_pts).reshape(-1, 4)
        cpu_pts = np.concatenate([g, np.repeat(g[:1], n_pts - n, axis=0)])
        cpu = []
        for _ in range(3):
            t = time.perf_counter()
            orc.msm(orc.VESTA, cpu_pts, cpu_sc, threads=orc.host_threads())
            cpu.append(time.perf_counter() - t)
        rows["batches"][str(B)] = {
            "verified": bool(ok), "wall_ms_median": round(float(np.median(ts[WARMUP:])) * 1e3, 3),
            "split_ms_median": {k: round(float(v), 3) for k, v in zip(
                ("transcript_callbacks", "host_scalars", "s_vector_kernels", "g_msm", "proof_point_msm", "library_total"), med)},
            "cpu_oracle_final_msm_ms": round(float(np.median(cpu)) * 1e3, 3), "cpu_oracle_msm_points": n_pts,
            "cpu_oracle_threads": orc.host_threads()}
    l0 = ctx.launch_count
    zk.srs_verify(srs, batch(64), rb, sgb)
    rows["kernel_launches_per_verify_64"] = ctx.launch_count - l0
    print(json.dumps(rows, indent=1))
    srs.close()
    ctx.close()
    if not ok_all:
        sys.exit("verify_time: an honest batch did not verify")


if __name__ == "__main__":
    main()
