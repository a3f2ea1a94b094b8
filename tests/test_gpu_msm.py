"""MSM parity: CUDA path (through the C ABI) vs the CPU oracle and vs the reference's golden vectors, bit-exact after
into_affine() (SURVEY.md "Hard parts": results are compared as canonical affine values)."""
import numpy as np
import pytest

import proof_systems_b200 as zk

pytestmark = pytest.mark.gpu

PALLAS_GY = 12418654782883325593414442427049395787963493412651469444558597405572177144507
VESTA_GY = 11426906929455361843568202299992114520848200991084027513389447476559454104162


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def lagrange_scalars(orc, fid, n, i):
    m = orc.MODULUS[fid]
    log_n = n.bit_length() - 1
    w = orc.fe_int(fid, orc.root_of_unity(fid, log_n))
    wi = pow(w, -i, m) if n > 1 else 1
    out, cur = [], pow(n, -1, m)
    for _ in range(n):
        out.append(cur)
        cur = cur * wi % m
    return orc.ints_to_limbs(out)


def test_vesta_msm_kat(ctx, orc):
    """kimchi/src/proof.rs:1163-1204"""
    cid = orc.VESTA
    G = np.concatenate([orc.fe(orc.FQ, 1), orc.fe(orc.FQ, VESTA_GY)])
    basis = np.stack([orc.scalar_mul(cid, G, i) for i in range(1, 17)])
    coeffs = [1, 7, 5, 35, 3, 21, 15, 105, 2, 14, 10, 70, 6, 42, 30, 210]   # b_poly_coefficients([2,3,5,7]), commitment.rs:869-910
    sc = orc.ints_to_limbs(coeffs)
    ex = 3756288960823668761746459900985719106126835112055076922409498125279524024429
    ey = 7540929664328976141648477194277016811781677917189411360504995258251130097840
    for wb in (0, 4, -1):
        bases = ctx.upload_bases(cid, basis, window_bits=wb)
        r = ctx.msm_affine(bases, sc)
        assert orc.fe_int(orc.FQ, r[:4]) == ex and orc.fe_int(orc.FQ, r[4:]) == ey, wb
        r = ctx.msm_affine(bases, orc.to_mont(orc.FP, sc), mont=True)       # VariableBaseMSM::msm takes field elements
        assert orc.fe_int(orc.FQ, r[:4]) == ex, wb
        bases.free()


@pytest.mark.parametrize("name", ["pallas_srs", "vesta_srs"])
def test_config1_lagrange_2048_pinned_msms(ctx, orc, request, name):
    """BASELINE config 1: 2^11-point MSMs against srs/test_*.srs; the answers are stored in the reference's file."""
    srs = request.getfixturevalue(name)
    want = srs.mont_points(srs.lag_2048_canon)
    for wb in (0, 8, 13):
        bases = ctx.upload_bases(srs.cid, srs.g[:2048], window_bits=wb)
        for i in [0, 1, 2, 1000, 2047]:
            sc = lagrange_scalars(orc, srs.scalar, 2048, i)
            assert np.array_equal(ctx.msm_affine(bases, sc), want[i]), (wb, i)
        rnd = orc.random_scalars(srs.scalar, 2048, seed=0)
        assert np.array_equal(ctx.msm_affine(bases, rnd), orc.msm(srs.cid, srs.g[:2048], rnd)), wb
        bases.free()


@pytest.mark.parametrize("name", ["pallas_srs", "vesta_srs"])
def test_edge_cases_vs_oracle(ctx, orc, request, name):
    """SURVEY.md §8d edge set: scalars 0, 1, r-1, 2^k; repeated bases (doubling); P and -P in one bucket; identity bases
    (ipa.rs:848-850); n = 1 and n not a power of two (ipa.rs:648-651); sub-slices of the resident bases."""
    srs = request.getfixturevalue(name)
    cid = srs.cid
    r = orc.MODULUS[srs.scalar]
    g = srs.g[:100].copy()
    g[5] = g[4]
    g[7] = g[6]
    g[7, 4:] = orc.fe_sub(srs.base, np.zeros(4, dtype=np.uint64), g[6, 4:])
    g[9] = 0
    g[50:60] = g[49]                  # ten copies of one point
    sc = orc.random_scalars(srs.scalar, 100, seed=3)
    sc[0] = 0
    sc[1] = orc.int_to_limbs(1)
    sc[2] = orc.int_to_limbs(r - 1)
    sc[3] = orc.int_to_limbs(1 << 200)
    sc[4] = sc[5] = orc.int_to_limbs(12345)
    sc[6] = sc[7] = orc.int_to_limbs(999)
    sc[50:60] = orc.int_to_limbs(77)  # same bucket, same point: exercises the P == Q branch of the mixed addition
    for wb in (0, 3, 6, 16):
        bases = ctx.upload_bases(cid, g, window_bits=wb)
        for n in [1, 2, 3, 7, 33, 64, 100]:
            assert np.array_equal(ctx.msm_affine(bases, sc[:n]), orc.msm(cid, g[:n], sc[:n])), (wb, n)
        # slice with an offset: msm(&g[off..off+n], ..)
        assert np.array_equal(ctx.msm_affine(bases, sc[:40], off=30), orc.msm(cid, g[30:70], sc[:40])), wb
        # explicit window choices on table-less bases
        if wb == 0:
            for c in (2, 5, 9, 13, 16):
                assert np.array_equal(ctx.msm_affine(bases, sc, window_bits=c), orc.msm(cid, g, sc)), c
        # all-zero scalars -> identity; empty MSM -> identity
        assert not np.any(ctx.msm_affine(bases, np.zeros((8, 4), dtype=np.uint64)))
        assert not np.any(ctx.msm_affine(bases, np.zeros((0, 4), dtype=np.uint64)))
        bases.free()


def test_degenerate_all_ones_witness_column(ctx, orc, pallas_srs):
    """kimchi's witness columns are {1 x 65526, 0 x 7, random x 3} (SURVEY.md §3.1): every point lands in one bucket.
    The balanced accumulation must handle it; the answer is the plain sum of the bases."""
    srs = pallas_srs
    n = 4096
    sc = np.zeros((n, 4), dtype=np.uint64)
    sc[:, 0] = 1
    sc[-10:-3] = 0
    sc[-3:] = orc.random_scalars(srs.scalar, 3, seed=1)
    bases = ctx.upload_bases(srs.cid, srs.g[:n], window_bits=-1)
    assert np.array_equal(ctx.msm_affine(bases, sc), orc.msm(srs.cid, srs.g[:n], sc))
    bases.free()


@pytest.mark.parametrize("sparsity", [0.05, 0.5, 0.99])
@pytest.mark.parametrize("bitlen", [16, 64, 128, 256])
def test_sparse_and_short_scalars(ctx, orc, vesta_srs, sparsity, bitlen):
    """The scalar distributions of the reference's `IPA Commit Evaluations` bench (poly-commitment/benches/ipa.rs:69-92):
    a fraction of the scalars non-zero, those reduced to `bitlen` bits — the high windows are empty, the low ones dense."""
    srs = vesta_srs
    n = 2048
    rng = np.random.default_rng(int(sparsity * 100) * 1000 + bitlen)
    vals = orc.limbs_to_ints(orc.random_scalars(srs.scalar, n, seed=bitlen))
    keep = rng.random(n) < sparsity
    sc = orc.ints_to_limbs([(v % (1 << bitlen)) if k else 0 for v, k in zip(vals, keep)])
    want = orc.msm(srs.cid, srs.g[:n], sc)
    for wb in (-1, 0, 7):
        bases = ctx.upload_bases(srs.cid, srs.g[:n], window_bits=wb)
        assert np.array_equal(ctx.msm_affine(bases, sc), want), wb
        bases.free()


@pytest.mark.parametrize("wb", [-1, 0, 9])
def test_random_and_all_ones_scalars_vs_oracle(ctx, orc, vesta_srs, wb):
    """random scalars and the degenerate one-bucket column against the oracle: the default table, plain bases and a window-9 table"""
    srs = vesta_srs
    n = 3000
    sc = orc.random_scalars(srs.scalar, n, seed=77)
    ones = np.zeros((n, 4), dtype=np.uint64); ones[:, 0] = 1
    with ctx.upload_bases(srs.cid, srs.g[:n], window_bits=wb) as bases:
        for scal in (sc, ones):
            assert np.array_equal(ctx.msm_affine(bases, scal), orc.msm(srs.cid, srs.g[:n], scal))


def test_config2_2_16_pallas(ctx, orc, pallas_srs):
    """BASELINE config 2: 2^16-point Pallas MSM on the real SRS, w = 16 table and the tuned window; one answer is
    pinned by srs/test_pallas.srs (lagrange_bases[65536][i]), the random-scalar answer by the oracle."""
    srs = pallas_srs
    n = 1 << 16
    rnd = orc.random_scalars(srs.scalar, n, seed=1)
    want_rnd = orc.msm(srs.cid, srs.g, rnd)
    want_lag = srs.mont_points(srs.lag_65536_canon)
    lag_sc = lagrange_scalars(orc, srs.scalar, n, int(srs.lag_65536_idx[1]))
    for wb in (16, -1, 0):
        bases = ctx.upload_bases(srs.cid, srs.g, window_bits=wb)
        assert np.array_equal(ctx.msm_affine(bases, rnd), want_rnd), wb
        assert np.array_equal(ctx.msm_affine(bases, lag_sc), want_lag[1]), wb
        # linearity / split property (ipa.rs:652-662: msm(g[..n/2]) + msm(g[n/2..]) == msm(g))
        lo = ctx.msm(bases, rnd[: n // 2])
        hi = ctx.msm(bases, rnd[n // 2:], off=n // 2)
        assert np.array_equal(zk.jacobian_to_affine(srs.cid, zk.jacobian_sum(srs.cid, np.stack([lo, hi]))), want_rnd), wb
        bases.free()


def test_batch_shares_bases(ctx, orc, vesta_srs):
    """the 7 chunks of t (ipa.rs:663-676) / 15 witness columns: k scalar vectors against the same resident bases."""
    srs = vesta_srs
    n, k = 2048, 5
    bases = ctx.upload_bases(srs.cid, srs.g[:n], window_bits=-1)
    sc = orc.random_scalars(srs.scalar, n * k, seed=11).reshape(k, n, 4)
    out = ctx.msm_batch(bases, sc)
    for j in range(k):
        assert np.array_equal(zk.jacobian_to_affine(srs.cid, out[j]), orc.msm(srs.cid, srs.g[:n], sc[j])), j
    bases.free()


def test_config4_2_20_vesta_sharded(ctx, orc, vesta_srs):
    """BASELINE config 4: 2^20-point Vesta MSM (fixture generators extended deterministically, SURVEY.md §8d), uniform
    Fp scalars seed 3.  The full MSM must match the oracle, and the per-shard partials of a 1/2/4/8-way split by points
    (what ranks compute before the all-gather) must sum to the identical affine point."""
    srs = vesta_srs
    n = 1 << 20
    g = orc.extend_bases(srs.cid, srs.g, n)
    sc = orc.random_scalars(srs.scalar, n, seed=3)
    want = orc.msm(srs.cid, g, sc)
    bases = ctx.upload_bases(srs.cid, g, window_bits=-1)
    assert bases.window_bits == 16
    assert np.array_equal(ctx.msm_affine(bases, sc), want)
    from proof_systems_b200.parallel import shard_bounds
    for world in (2, 4, 8):
        parts = []
        for r in range(world):
            lo, hi = shard_bounds(n, world, r)
            parts.append(ctx.msm(bases, sc[lo:hi], off=lo))
        assert np.array_equal(zk.jacobian_to_affine(srs.cid, zk.jacobian_sum(srs.cid, np.stack(parts))), want), world
    bases.free()


def test_pinned_scalars_zero_copy(ctx, orc, pallas_srs):
    import torch
    srs = pallas_srs
    n = 3000
    sc = orc.random_scalars(srs.scalar, n, seed=13)
    pinned = torch.from_numpy(sc.view(np.int64).copy()).pin_memory().numpy().view(np.uint64)
    bases = ctx.upload_bases(srs.cid, srs.g[:n], window_bits=-1)
    assert np.array_equal(ctx.msm_affine(bases, pinned), orc.msm(srs.cid, srs.g[:n], sc))
    bases.free()


def test_concurrent_callers_share_one_context(ctx, orc, vesta_srs):
    """kimchi commits its 15 witness columns from 15 rayon workers against one Arc<SRS> (kimchi/src/prover.rs:329-351;
    SRS: Sync + Send, poly-commitment/src/lib.rs:61): the C ABI must be re-entrant.  Eight Python threads (ctypes
    releases the GIL during the call) hammer one context with different scalar vectors."""
    import threading
    srs = vesta_srs
    n = 1024
    bases = ctx.upload_bases(srs.cid, srs.g[:n], window_bits=-1)
    scs = [orc.random_scalars(srs.scalar, n, seed=100 + t) for t in range(8)]
    want = [orc.msm(srs.cid, srs.g[:n], s) for s in scs]
    got, errs = [None] * 8, []

    def work(t):
        try:
            for _ in range(5):
                got[t] = ctx.msm_affine(bases, scs[t])
        except Exception as e:  # pragma: no cover
            errs.append(e)

    th = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errs
    for t in range(8):
        assert np.array_equal(got[t], want[t]), t
    bases.free()


def test_error_codes(ctx, orc, pallas_srs):
    """invalid arguments come back as error codes with a message, never as a crash"""
    srs = pallas_srs
    bases = ctx.upload_bases(srs.cid, srs.g[:64], window_bits=0)
    sc = orc.random_scalars(srs.scalar, 64, seed=1)
    with pytest.raises(zk.ZkError) as e:
        ctx.msm(bases, sc, off=10)                     # slice [10, 74) outside the 64 resident bases
    assert e.value.code == -1 and "outside" in str(e.value)
    with pytest.raises(zk.ZkError):
        ctx.msm(bases, sc, window_bits=17)
    with pytest.raises(zk.ZkError):
        ctx.upload_bases(7, srs.g[:4])                 # unknown curve id
    with pytest.raises(zk.ZkError):
        ctx.ntt(5, np.zeros((4, 4), dtype=np.uint64))  # unknown field id
    with pytest.raises(zk.ZkError):
        ctx.ntt_dev(zk.FP, 0, 21)                      # log_n beyond the two-pass plan
    with pytest.raises(zk.ZkError):
        ctx.set_option("msm_tma", 1)                   # unknown option
    other = zk.Context(0)
    with pytest.raises(zk.ZkError):
        other.msm(bases, sc)                           # bases belong to another context
    other.close()
    bases.free()


def test_partial_and_finish_gathered_emulate_two_ranks(ctx, orc, vesta_srs):
    """The multi-GPU exchange without the collective (SURVEY.md §8e): two zk_msm_partial calls on the two halves of the points
    write their slice sums next to each other — exactly what an all_gather over two ranks produces — and
    zk_msm_finish_gathered(world = 2) must return the MSM over all points; world = 1 must equal zk_msm."""
    import torch
    srs = vesta_srs
    n = 2048
    sc = orc.random_scalars(srs.scalar, n, seed=41)
    want = orc.msm(srs.cid, srs.g[:n], sc)
    d_sc = torch.from_numpy(sc.view(np.int64)).cuda()
    h_sc = torch.from_numpy(sc.view(np.int64).copy()).pin_memory()
    for wb in (-1, 0):
        bases = ctx.upload_bases(srs.cid, srs.g[:n], window_bits=wb)
        d_all = torch.zeros((2, 4096, 16), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()       # torch fills on ITS stream; the context runs on its own
        w = 0 if wb else 7             # without a table the default window depends on the slice length: ranks must agree on one
        c, g = ctx.msm_partial(bases, d_sc.data_ptr(), n, d_all.data_ptr(), 4096, window_bits=w)
        one = ctx.msm_finish_gathered(srs.cid, d_all.data_ptr(), 1, c, g)
        assert np.array_equal(zk.jacobian_to_affine(srs.cid, one), want), wb
        cnt = c * g
        packed = torch.zeros((2, cnt, 16), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        half = n // 2
        assert ctx.msm_partial(bases, d_sc.data_ptr(), half, packed[0].data_ptr(), cnt, window_bits=w) == (c, g)
        # second "rank": page-locked host scalars, read over PCIe
        assert ctx.msm_partial(bases, h_sc.data_ptr() + 32 * half, half, packed[1].data_ptr(), cnt, off=half, window_bits=w) == (c, g)
        two = ctx.msm_finish_gathered(srs.cid, packed.data_ptr(), 2, c, g)
        assert np.array_equal(zk.jacobian_to_affine(srs.cid, two), want), wb
        launched = ctx.launch_count
        with pytest.raises(zk.ZkError):
            ctx.msm_partial(bases, d_sc.data_ptr(), n, d_all.data_ptr(), 1)      # buffer too small for the slice sums
        assert ctx.launch_count == launched                                       # refused before anything runs
        bases.free()


def test_synthetic_points_are_on_the_curve_and_deterministic(ctx, orc):
    """zk_points_synthetic (inputs of BASELINE config 4 in bench.py): every point satisfies y^2 = x^3 + 5, the sequence depends only
    on (curve, seed, index), and an MSM over them agrees with the oracle."""
    for cid in (zk.PALLAS, zk.VESTA):
        fid = orc.BASE_FIELD[cid]
        p = ctx.synthetic_points(cid, 3000, seed=9)
        assert np.array_equal(p, ctx.synthetic_points(cid, 3000, seed=9))
        assert np.array_equal(p[:1000], ctx.synthetic_points(cid, 1000, seed=9))
        assert not np.array_equal(p[:8], ctx.synthetic_points(cid, 8, seed=10))
        x, y = np.ascontiguousarray(p[:, :4]), np.ascontiguousarray(p[:, 4:])
        five = orc.to_mont(fid, orc.ints_to_limbs([5] * len(p)))
        lhs = ctx.field_op(fid, "mul", y, y)
        rhs = ctx.field_op(fid, "add", ctx.field_op(fid, "mul", ctx.field_op(fid, "mul", x, x), x), five)
        assert np.array_equal(lhs, rhs)
        assert len({bytes(r) for r in x}) == len(p)                      # distinct points
        sc = orc.random_scalars(orc.SCALAR_FIELD[cid], len(p), seed=11)
        b = ctx.upload_bases(cid, p, window_bits=-1)
        assert np.array_equal(ctx.msm_affine(b, sc), orc.msm(cid, p, sc))
        b.free()


def test_concurrent_host_callers_overlap_on_the_lane_pool():
    """kimchi/src/prover.rs:329-351: 15 rayon workers call commit_evaluations_non_hiding at once on ONE shared SRS.  A context is a
    pool of lanes (csrc/ctx.hpp): independent host-pointer calls from different threads run concurrently on the device — every
    result equals the serial one, and the 15 calls take clearly less wall-clock time than one after the other.
    The measurement runs in a fresh interpreter: late in a long test session the threaded calls time slower than the serial ones
    for reasons of the session (its threads, heap and contexts), not of the library."""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path[:0] = [{here!r}, {os.path.dirname(here)!r}]\n"
            "from oracle import oracle as orc\nfrom conftest import GoldenSRS\nimport test_gpu_msm as t\n"
            "orc.lib()\nt._lane_pool_overlap(orc, GoldenSRS('pallas', orc))\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]


def _lane_pool_overlap(orc, G):
    import gc
    import threading
    import time
    n, k = 1 << 14, 15
    c = zk.Context(0)
    try:
        bases = c.upload_bases(zk.PALLAS, G.g[:n], window_bits=-1)
        sc = [orc.random_scalars(G.scalar, n, seed=300 + j) for j in range(k)]
        aff = lambda r: zk.jacobian_to_affine(zk.PALLAS, r)     # (Jacobian coordinates depend on the order the sort's atomics hand out)
        serial = [aff(c.msm(bases, sc[j])) for j in range(k)]                 # also warms every code path up
        # both arms are the best of three rounds: on a shared host one ~5 ms window is at the mercy of the other tenants; and, like
        # timeit, with the garbage collector off (a collection over a whole test session's heap stalls every thread for milliseconds)
        gc.collect()
        gc.disable()
        c.set_option("ctx_lanes", 1)
        t_serial = float("inf")
        for _ in range(3):
            t0 = time.perf_counter()
            for j in range(k):
                c.msm(bases, sc[j])
            t_serial = min(t_serial, time.perf_counter() - t0)
        c.set_option("ctx_lanes", 4)
        out = [None] * k
        t_pool = float("inf")
        # the threads are started first and released together: the window times the 15 calls, not thread creation (which can
        # take as long as the serial calls themselves on a busy host)
        for rnd in range(4):                                                  # round 0 creates the lanes and their scratch: untimed
            go = threading.Barrier(k + 1)

            def work(j):
                go.wait()
                out[j] = c.msm(bases, sc[j])          # the serial arm times the calls alone too: made affine below
            th = [threading.Thread(target=work, args=(j,)) for j in range(k)]
            for t in th:
                t.start()
            go.wait()
            t0 = time.perf_counter()
            for t in th:
                t.join()
            if rnd:
                t_pool = min(t_pool, time.perf_counter() - t0)
        gc.enable()
        out = [aff(r) for r in out]
        for j in range(k):
            assert np.array_equal(out[j], serial[j]), j
            assert np.array_equal(out[j], orc.msm(zk.PALLAS, G.g[:n], sc[j])), j
        assert t_pool < 0.8 * t_serial, (t_pool, t_serial)
        bases.free()
    finally:
        gc.enable()
        c.close()


def test_library_owned_communicator_single_rank(ctx, orc, pallas_srs):
    """zk_comm_* / zk_msm_sharded with a world of one: the NCCL communicator is created inside the library (csrc/comm.cu) and the
    sharded entry point returns the plain MSM."""
    from proof_systems_b200.parallel import LibraryComm
    G = pallas_srs
    n = 4096
    comm = LibraryComm(ctx)
    try:
        bases = ctx.upload_bases(zk.PALLAS, G.g[:n], window_bits=-1)
        sc = orc.random_scalars(G.scalar, n, seed=77)
        got = zk.jacobian_to_affine(zk.PALLAS, comm.msm(bases, sc.ctypes.data, n))
        assert np.array_equal(got, orc.msm(zk.PALLAS, G.g[:n], sc))
        bases.free()
    finally:
        comm.close()
