"""A plain-Python mirror of the MSM planner (proof_systems_b200/csrc/msm.cu: msm_default_window, msm_run, k_recode, k_plan), integers
only.  The tests use it in two directions: to say which pipeline a call takes (finish variant, entries per task, quads per bucket,
giant buckets, scan tiles), and to build scalars that put a chosen number of entries into chosen buckets.

The library reports (c, groups) of a call (zk_msm_partial) and its kernel launches (zk_ctx_launch_count: one more with the
thread-per-bucket finish than with the quad finish); tests/test_gpu_msm_regimes.py ties the mirror to the device through both."""
from collections import Counter, namedtuple

import numpy as np

MAX_WINDOW_BITS = 16
MAX_GIANTS = 64        # MSM_MAX_GIANTS: a longer giant list overflows and the finish kernels sum the giants themselves
MAX_BATCH = 16
PLAN_TILE = 4096       # buckets per CTA of k_plan's chained scan
TREE_QUADS = 64
GIANT_SLICES = 16      # CTAs per giant bucket in k_giant_finish
RUN = 4                # consecutive partials per thread of k_run_sum
SCALAR_LIMIT = 1 << 254   # below both scalar moduli

Plan = namedtuple("Plan", "n k c use_table nwin gpm G B NB Mmax capacity many_buckets K log_g smax run ntiles launches")
Regime = namedtuple("Regime", "s_b task_off giants overflow empty single multi tasks")


def num_windows(c):
    return (256 + c - 1) // c


def default_window(n, precomputed):
    """msm_default_window: floor(log2 n) - 1 with a table, - 4 without, kept inside [4, 16]"""
    c = max(n.bit_length() - 1, 0) - (1 if precomputed else 4)
    return min(max(c, 4), MAX_WINDOW_BITS)


def _pow2_ceil_log(x):
    l = 0
    while (1 << l) < x:
        l += 1
    return l


def plan(n, k, c_table, window_bits, sm_count, chunk=0, wave_threads=0):
    """What msm_run derives for k fused MSMs of n scalars each.  c_table: window of the resident table (0: none; what
    zk_bases_window_bits reports); window_bits: the call's choice for table-less bases (0: default)."""
    use_table = c_table != 0
    c = c_table if use_table else (window_bits or default_window(n, False))
    assert 2 <= c <= MAX_WINDOW_BITS and 1 <= k <= MAX_BATCH and n > 0
    nwin = num_windows(c)
    gpm = 1 if use_table else nwin
    G = k * gpm
    B = 1 << (c - 1)
    NB = G * B
    Mmax = n * nwin * k
    capacity = sm_count * (wave_threads or 512)
    many = NB > sm_count * TREE_QUADS
    K = chunk
    if K == 0:
        n_avg = max(1, Mmax // NB)
        k_bal = min(64, max(6, n_avg // 8)) if many else 64
        slack = min(NB // 2, capacity // 4)
        k_cap = max(4, (Mmax + capacity - slack - 1) // (capacity - slack))
        K = min(k_bal, k_cap)
    s_avg = Mmax // (K * NB) + 1
    log_g = min(3, _pow2_ceil_log((s_avg + 7) // 8))
    return Plan(n=n, k=k, c=c, use_table=use_table, nwin=nwin, gpm=gpm, G=G, B=B, NB=NB, Mmax=Mmax, capacity=capacity, many_buckets=many,
                K=K, log_g=log_g, smax=32 << log_g, run=RUN, ntiles=(NB + PLAN_TILE - 1) // PLAN_TILE, launches=8 + (1 if many else 0))


def digits(s, c):
    """k_recode: the signed base-2^c digits of s, each in (-2^(c-1), 2^(c-1)], lowest window first; a digit above 2^(c-1) becomes
    negative and carries one into the next window"""
    half, mask = 1 << (c - 1), (1 << c) - 1
    out, carry = [], 0
    for w in range(num_windows(c)):
        d = ((s >> (w * c)) & mask) + carry
        if d > half:
            d -= 1 << c
            carry = 1
        else:
            carry = 0
        out.append(d)
    assert carry == 0, "carry out of the top window"
    return out


def bucket_of(p, j, w, d):
    """index of the bucket that digit d != 0 of window w of MSM j falls into"""
    return (j * p.gpm + (0 if p.use_table else w)) * p.B + abs(d) - 1


def buckets(scalar_sets, p):
    """entries per bucket, int64 [NB]: scalar_sets[j] are the n scalars (ints) of MSM j"""
    assert len(scalar_sets) == p.k
    counts = np.zeros(p.NB, dtype=np.int64)
    for j, scalars in enumerate(scalar_sets):
        assert len(scalars) == p.n
        for s, times in Counter(int(s) for s in scalars).items():
            for w, d in enumerate(digits(s, p.c)):
                if d:
                    counts[bucket_of(p, j, w, d)] += times
    return counts


def regime(counts, p):
    """k_plan's view of a histogram: tasks per bucket s_b = ceil(n_b / K), their exclusive scan, the giant buckets (s_b > smax)
    and whether their list overflows"""
    s_b = (counts + p.K - 1) // p.K
    task_off = np.concatenate([[0], np.cumsum(s_b)])
    giants = np.flatnonzero(s_b > p.smax)
    return Regime(s_b=s_b, task_off=task_off, giants=giants, overflow=len(giants) > MAX_GIANTS, empty=int(np.sum(s_b == 0)),
                  single=int(np.sum(s_b == 1)), multi=int(np.sum((s_b >= 2) & (s_b <= p.smax))), tasks=int(task_off[-1]))


def scalar_of(window_digits, c):
    """the scalar whose signed digits are window_digits {window: digit} and zero elsewhere.  A negative digit needs a positive one
    above it: the value must not be negative."""
    half = 1 << (c - 1)
    s = 0
    for w, d in window_digits.items():
        assert -half < d <= half and d != 0 and 0 <= w < num_windows(c)
        s += d << (c * w)
    assert 0 <= s < SCALAR_LIMIT
    return s


def scalars_for(populations, c):
    """populations: (window, digit, count) triples -> count scalars per triple, in order, each with that digit in that window.
    digit v > 0 is the scalar v * 2^(c w) (bucket v - 1).  digit -v is (2^c - v) * 2^(c w): the recoding turns it into -v and
    carries, so the scalar also has digit +1 in window w + 1 (bucket 0 there)."""
    out = []
    for w, d, count in populations:
        s = scalar_of({w: d} if d > 0 else {w: d, w + 1: 1}, c)
        out += [s] * count
    return out
