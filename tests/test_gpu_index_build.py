"""The prover index built on the device (zk_index_build) and the commitments of its verifier index (zk_index_commitments), bit for bit
against tests/index_replay.py, the restatement of kimchi's ConstraintSystem::evaluated_column_coefficients / column_evaluations
(constraints.rs:510-760) and ProverIndex::verifier_index (verifier_index.rs:221-300).  The built index also equals the loaded cache
file of the same circuit, and the resident chain runs on it: z of a wired circuit ends at 1 and its quotient vanishes on d1, and the
generic-gate constraint of a satisfied circuit is zero on d1."""
import ctypes
import random
import threading

import numpy as np
import pytest
import torch

import evals_replay as ev
import gate_programs as gp
import index_replay as ir
import perm_replay as pr
import proof_systems_b200 as zk
from index_cache_writer import write_cache
from test_gpu_perm_aggreg import vanishing_coeffs

pytestmark = pytest.mark.gpu

ALL_OPTIONAL = 0b111111


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def circuit(orc, fid, n, n_gates, seed, tags=range(14), max_row=None):
    """n_gates gates cycling through `tags`, random wires into rows < max_row (default n), 0 .. 20 coefficients; random shifts"""
    rng = random.Random(seed)
    P = orc.MODULUS[fid]
    tags = list(tags)
    max_row = max_row or n
    gates = []
    for r in range(n_gates):
        wires = [(rng.randrange(max_row), rng.randrange(7)) for _ in range(7)]
        gates.append((tags[r % len(tags)], wires, [rng.randrange(P) for _ in range(rng.choice([0, 1, 3, 15, 20]))]))
    shifts = [1] + [rng.randrange(2, P) for _ in range(6)]
    return gates, shifts


def build(ctx, orc, fid, n, zk_rows, gates, shifts, optional=0, zero_selectors=False, **kw):
    h = ir.header(zk, n, zk_rows, ev.mont(orc, fid, shifts), optional, **kw)
    return zk.IndexCache.build(ctx, fid, h, ir.pruned_gates(gates), ir.gate_coeffs(orc, fid, gates), zero_selectors)


def section(ctx, idx, tag):
    p, n_el, dom = idx.section(tag)
    return ctx.dev_download(p, (n_el, 4)), dom


def view(ptr, n_el) -> torch.Tensor:
    """a device section as a torch tensor [n_el, 4] (int64 bits), without a copy"""
    class A:
        __cuda_array_interface__ = {"shape": (n_el, 4), "typestr": "<i8", "data": (ptr, False), "version": 3}
    return torch.as_tensor(A(), device="cuda")


# ---------------------------------------------------------------------------------------------------------------- 1, 2: sections
CASES = [(4, 3, 16, 0), (4, 15, 9, ALL_OPTIONAL), (10, 5, 1000, ALL_OPTIONAL), (10, 3, 1024, 0b010101), (10, 1023, 14, 0b100010),
         (16, 3, 40000, ALL_OPTIONAL)]


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,zk_rows,n_gates,optional", CASES)
def test_sections_match_the_restatement(ctx, orc, fid, log_n, zk_rows, n_gates, optional):
    n = 1 << log_n
    gates, shifts = circuit(orc, fid, n, n_gates, seed=log_n * 100 + zk_rows + fid)
    endo = ev.mont(orc, fid, [12345])[0]
    kw = dict(public_inputs=3, prev_challenges=2, max_poly_size=1 << 16, feature_flags=0x41, lookup_selectors_present=0,
              disable_gates_checks=1, has_verifier_index_digest=1, endo=endo, verifier_index_digest=[1, 2, 3, 4], identifier=b"circuit-7")
    idx = build(ctx, orc, fid, n, zk_rows, gates, shifts, optional, **kw)
    try:
        want = ir.sections(orc, fid, n, zk_rows, gates, shifts, optional)
        h = idx.header
        assert h.num_sections == len(want) == 29 + bin(optional).count("1")
        assert (h.domain_d1_size, h.zk_rows, h.optional_selectors_present) == (n, zk_rows, optional)
        assert (h.public_inputs, h.prev_challenges, h.max_poly_size, h.feature_flags, h.disable_gates_checks, h.has_verifier_index_digest) == \
            (3, 2, 1 << 16, 0x41, 1, 1)
        assert list(h.endo) == [int(x) for x in endo] and list(h.verifier_index_digest) == [1, 2, 3, 4] and h.identifier == b"circuit-7"
        assert [list(r) for r in h.shift] == [[int(x) for x in r] for r in ev.mont(orc, fid, shifts)]
        for tag, (payload, dom) in want.items():
            got, d = section(ctx, idx, tag)
            assert d == dom and np.array_equal(got, payload), hex(tag)
        for tag in (0x02, 0x03, 0x50):
            with pytest.raises(zk.ZkError):
                idx.section(tag)
        for b in range(6):
            if not optional >> b & 1:
                with pytest.raises(zk.ZkError):
                    idx.section(0x40 + b)
    finally:
        idx.close()


@pytest.mark.parametrize("fid", [0, 1])
def test_zero_selectors(ctx, orc, fid):
    n, zk_rows = 256, 4
    gates, shifts = circuit(orc, fid, n, 200, seed=5 + fid)
    idx = build(ctx, orc, fid, n, zk_rows, gates, shifts, ALL_OPTIONAL, zero_selectors=True)
    try:
        want = ir.sections(orc, fid, n, zk_rows, gates, shifts, ALL_OPTIONAL, zero_selectors=True)
        zeroed = set(ir.selector_tags(ALL_OPTIONAL))
        assert zeroed == {0x22, 0x23, 0x24, 0x25} | {0x40 + b for b in range(6)}
        for tag, (payload, dom) in want.items():
            got, d = section(ctx, idx, tag)
            assert d == dom and np.array_equal(got, payload), hex(tag)
            assert (not got.any()) == (tag in zeroed), hex(tag)
    finally:
        idx.close()


# ---------------------------------------------------------------------------------------------------------------- 3: built == loaded
def cache_image(orc, fid, n, zk_rows, gates, shifts, optional, endo):
    secs = ir.sections(orc, fid, n, zk_rows, gates, shifts, optional)
    hdr = {"public": 1, "prev_challenges": 0, "zk_rows": zk_rows, "max_poly_size": n, "domain_d1_size": n, "optional_selectors_present": optional,
           "endo_limbs": [int(x) for x in endo], "shift_limbs": [[int(x) for x in r] for r in ev.mont(orc, fid, shifts)]}
    sections = [(0x02, ir.pruned_gates(ir.padded(gates, n)), 0), (0x03, ir.gate_coeffs(orc, fid, ir.padded(gates, n)), 0)]
    sections += [(tag, a.astype("<u8").tobytes(), dom) for tag, (a, dom) in secs.items()]
    return write_cache("vk", hdr, sections)


@pytest.mark.parametrize("fid", [0, 1])
def test_built_index_equals_the_loaded_file(ctx, orc, fid):
    n, zk_rows, optional = 512, 6, 0b001100
    gates, shifts = circuit(orc, fid, n, 300, seed=11 + fid)
    endo = ev.mont(orc, fid, [77])[0]
    loaded = zk.IndexCache(ctx, cache_image(orc, fid, n, zk_rows, gates, shifts, optional, endo))
    built = build(ctx, orc, fid, n, zk_rows, gates, shifts, optional, public_inputs=1, max_poly_size=n, endo=endo, identifier=b"vk")
    try:
        hb, hl = built.header, loaded.header
        for f, _ in zk.IndexHeader._fields_:
            if f not in ("num_sections", "shift", "endo", "verifier_index_digest"):
                assert getattr(hb, f) == getattr(hl, f), f
        assert [list(r) for r in hb.shift] == [list(r) for r in hl.shift] and list(hb.endo) == list(hl.endo)
        assert hl.num_sections == hb.num_sections + 2                    # the file also holds the gates and their coefficients
        for tag in [0x01] + ir.commitment_tags(optional):
            a, da = section(ctx, built, tag)
            b, db = section(ctx, loaded, tag)
            assert da == db and np.array_equal(a, b), hex(tag)
    finally:
        built.close()
        loaded.close()


# ---------------------------------------------------------------------------------------------------------------- 4: 2^21 rows
def test_two_to_the_21_rows(ctx, orc):
    """omega^row needs the third table factor (row >= 2^20): wires point anywhere in the domain"""
    fid, log_n, zk_rows = 0, 21, 3
    n = 1 << log_n
    gates, shifts = circuit(orc, fid, n, 3000, seed=21)
    gates[0] = (ir.GENERIC, [(n - 1, 6), ((1 << 20) + 5, 0), ((1 << 20) + 1023, 3), (1 << 20, 1), (n - 2, 2), (3 << 19, 4), (7, 5)], [5])
    cols = ir.columns_d1(orc, fid, n, zk_rows, gates, shifts)
    idx = build(ctx, orc, fid, n, zk_rows, gates, shifts)
    try:
        assert idx.header.num_sections == len(cols) == 29
        for tag, c in cols.items():
            p, n_el, dom = idx.section(tag)
            m = ir.domain_mult(tag)
            assert n_el == dom == m * n
            got = view(p, n_el)[::m].cpu().numpy().view(np.uint64)
            assert np.array_equal(got, c), hex(tag)
        for tag in (0x30, 0x23):
            p, n_el, _ = idx.section(tag)
            assert np.array_equal(view(p, n_el).cpu().numpy().view(np.uint64), ir.evaluate(orc, fid, cols[tag], 8)), hex(tag)
    finally:
        idx.close()
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------- 5: commitments
def srs_of(ctx, golden, m):
    return zk.SRS(ctx, golden.cid, golden.g[:m], golden.mont_points(golden.h_xy_canon.reshape(1, 64))[0])


@pytest.mark.parametrize("curve,log_n,m", [("pallas", 10, 1 << 16), ("vesta", 10, 1 << 16), ("vesta", 16, 1 << 16), ("vesta", 17, 1 << 16)])
def test_commitments(ctx, orc, pallas_srs, vesta_srs, curve, log_n, m):
    golden = pallas_srs if curve == "pallas" else vesta_srs
    fid = orc.SCALAR_FIELD[golden.cid]
    n, zk_rows, optional = 1 << log_n, 5, 0b100101
    gates, shifts = circuit(orc, fid, n, min(n, 3000), seed=log_n + fid)
    srs = srs_of(ctx, golden, m)
    idx = build(ctx, orc, fid, n, zk_rows, gates, shifts, optional)
    try:
        got = srs.index_commitments(idx)
        chunks = max(1, n // m)
        assert got.shape == (28 + 3, chunks, 8)
        cols = ir.columns_d1(orc, fid, n, zk_rows, gates, shifts, optional)
        want = ir.commitments(orc, golden.cid, golden.g[:m], srs.h, cols, optional)
        assert np.array_equal(got, want)
        # the masked ones are h away from commit_evaluations_non_hiding
        plain = srs.commit_evaluations_non_hiding(n, cols[0x21]).chunks
        assert np.array_equal(got[23], np.stack([orc.affine_add(golden.cid, p, srs.h) for p in plain]))
        if log_n == 10:          # a loaded cache of the same circuit commits to the same points
            endo = ev.mont(orc, fid, [1])[0]
            loaded = zk.IndexCache(ctx, cache_image(orc, fid, n, zk_rows, gates, shifts, optional, endo))
            try:
                assert np.array_equal(srs.index_commitments(loaded), got)
            finally:
                loaded.close()
    finally:
        idx.close()
        srs.close()


# ---------------------------------------------------------------------------------------------------------------- 6: the resident chain
def wired_circuit(orc, fid, log_n, zk_rows, seed):
    """random cycles of 1 to 4 cells among the cells of rows < n - zk_rows, encoded as gate wires (wire k of row j = the next cell of
    (k, j)'s cycle); the witness is constant on each cycle and random elsewhere"""
    P, n = orc.MODULUS[fid], 1 << log_n
    rng = random.Random(seed)
    last = n - zk_rows
    cells = [(k, j) for j in range(last) for k in range(7)]
    rng.shuffle(cells)
    wires = {}
    w = [[rng.randrange(P) for _ in range(n)] for _ in range(7)]
    i = 0
    while i < len(cells):
        cyc = cells[i:i + rng.randint(1, 4)]
        i += len(cyc)
        v = rng.randrange(P)
        for a, b in zip(cyc, cyc[1:] + cyc[:1]):
            wires[a] = (b[1], b[0])                                # (row, col) of the next cell
            w[a[0]][a[1]] = v
    gates = [(ir.GENERIC, [wires[(k, j)] for k in range(7)], []) for j in range(last)]
    shifts = [1] + [rng.randrange(2, P) for _ in range(6)]
    return gates, shifts, w


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,zk_rows", [(10, 5), (12, 3)])
def test_permutation_on_a_built_index(ctx, orc, fid, log_n, zk_rows):
    P, n = orc.MODULUS[fid], 1 << log_n
    m8 = 8 * n
    gates, shifts, w = wired_circuit(orc, fid, log_n, zk_rows, seed=fid + log_n)
    rng = random.Random(log_n)
    beta, gamma, alpha0, r0, r1 = (rng.randrange(1, P) for _ in range(5))
    mont = lambda xs: ev.mont(orc, fid, xs)
    idx = build(ctx, orc, fid, n, zk_rows, gates, shifts)
    bufs = []

    def put(a):
        a = np.ascontiguousarray(a, dtype=np.uint64)
        p = ctx.dev_alloc(a.nbytes)
        bufs.append(p)
        ctx.dev_upload(p, a)
        return p
    try:
        d_s = [idx.section(0x30 + k)[0] for k in range(7)]
        d_wev = put(np.concatenate([mont(w[k]) for k in range(7)]))
        d_w = [d_wev + k * n * 32 for k in range(7)]
        d_z = put(np.zeros((n, 4), dtype=np.uint64))
        b, g, sh, rn = mont([beta])[0], mont([gamma])[0], mont(shifts), mont([r0, r1])
        assert ctx.perm_aggreg_dev(fid, log_n, zk_rows, d_w, d_s, m8, b, g, sh, rn, d_z) is True
        sigma = [ev.ints(orc, fid, c) for t, c in sorted(ir.columns_d1(orc, fid, n, zk_rows, gates, shifts).items()) if 0x30 <= t <= 0x36]
        _, z_coeffs, ok = pr.perm_aggreg(orc, fid, log_n, zk_rows, w, sigma, shifts, beta, gamma, [r0, r1])
        assert ok and np.array_equal(ctx.dev_download(d_z, (n, 4)), mont(z_coeffs))
        d_wc, d_w8, d_z8, d_zk8, d_out = (put(np.zeros((k, 4), dtype=np.uint64)) for k in (7 * n, 7 * m8, m8, m8, m8))
        ctx.ntt_dev_oop(fid, d_wev, n, n, d_wc, log_n, batch=7, inverse=True)
        ctx.ntt_dev_oop(fid, d_wc, n, n, d_w8, log_n + 3, batch=7)
        ctx.ntt_dev_oop(fid, d_z, n, n, d_z8, log_n + 3)
        d_zk = put(mont(vanishing_coeffs(orc, fid, log_n, zk_rows)))
        ctx.ntt_dev_oop(fid, d_zk, 4, 4, d_zk8, log_n + 3)
        ctx.perm_quotient_dev(fid, log_n + 3, [d_w8 + k * m8 * 32 for k in range(7)], d_z8, d_s, d_zk8, b, g, mont([alpha0])[0], sh, d_out)
        out = ctx.dev_download(d_out, (m8, 4))
        assert not out[::8].any() and out.any()
    finally:
        for p in bufs:
            ctx.dev_free(p)
        idx.close()


@pytest.mark.parametrize("fid,log_n", [(0, 8), (1, 11)])
def test_generic_gates_on_a_built_index(ctx, orc, fid, log_n):
    """rows < n - 3 are Generic gates with random coefficients and a witness solving both halves for o; zk_expr_eval_dev over the
    built coefficients8 and generic_selector4 is zero at every point of d1 and not everywhere on d4"""
    P, n = orc.MODULUS[fid], 1 << log_n
    rng = random.Random(fid + log_n)
    w = [[rng.randrange(P) for _ in range(n)] for _ in range(15)]
    gates = []
    for j in range(n - 3):
        c = [rng.randrange(P) for _ in range(10)]
        for h in range(2):
            l, r = w[3 * h][j], w[3 * h + 1][j]
            cl, cr, co, cm, cc = c[5 * h:5 * h + 5]
            w[3 * h + 2][j] = -(cl * l + cr * r + cm * l * r + cc) * pow(co, P - 2, P) % P
        gates.append((ir.GENERIC, [(j, k) for k in range(7)], c))
    shifts = [1] + [rng.randrange(2, P) for _ in range(6)]
    idx = build(ctx, orc, fid, n, 3, gates, shifts)
    bufs = []
    try:
        d_w1 = ctx.dev_alloc(15 * n * 32)
        d_w8 = ctx.dev_alloc(15 * 8 * n * 32)
        d_out = ctx.dev_alloc(4 * n * 32)
        bufs += [d_w1, d_w8, d_out]
        ctx.dev_upload(d_w1, np.concatenate([ev.mont(orc, fid, c) for c in w]))
        ctx.ntt_dev(fid, d_w1, log_n, batch=15, inverse=True)
        ctx.ntt_dev_oop(fid, d_w1, n, n, d_w8, log_n + 3, batch=15)
        cols = [(d_w8 + k * 8 * n * 32, 8 * n, 8) for k in range(15)]
        cols += [(idx.section(0x10 + i)[0], 8 * n, 8) for i in range(15)] + [(idx.section(0x20)[0], 4 * n, 4)]
        alphas = orc.to_mont(fid, orc.random_scalars(fid, 2, seed=fid))
        gp.generic_gate(zk.ExprProgram(), alphas).evaluations(ctx, fid, cols, 4 * n, 4, d_out)
        out = ctx.dev_download(d_out, (4 * n, 4))
        assert not out[::4].any() and out.any()
    finally:
        for p in bufs:
            ctx.dev_free(p)
        idx.close()


# ---------------------------------------------------------------------------------------------------------------- 7: refusals
def raw_build(ctx, fid, h, g, c, zero=0, n_gates=None):
    out = ctypes.c_void_p(0xdead)
    rc = zk.lib().zk_index_build(ctx._h, fid, ctypes.byref(h) if h is not None else None, g or None, len(g) // 60 if n_gates is None else n_gates,
                                 c or None, len(c), zero, ctypes.byref(out))
    return rc, out.value


def test_refusals(ctx, orc):
    fid, n = 0, 64
    P = orc.MODULUS[fid]
    gates, shifts = circuit(orc, fid, n, 10, seed=9)
    g, c = ir.pruned_gates(gates), ir.gate_coeffs(orc, fid, gates)
    hdr = lambda **kw: ir.header(zk, kw.pop("n", n), kw.pop("zk_rows", 3), ev.mont(orc, fid, shifts), kw.pop("optional", 0), **kw)
    ok_rc, ok_ptr = raw_build(ctx, fid, hdr(), g, c)
    assert ok_rc == 0 and ok_ptr
    zk.lib().zk_index_cache_free(ctypes.c_void_p(ok_ptr))
    bad_tag = bytearray(g)
    bad_tag[60 * 3] = 14
    bad_row = bytearray(g)
    bad_row[60 * 2 + 4 + 8 * 5:60 * 2 + 8 + 8 * 5] = n.to_bytes(4, "little")
    bad_col = bytearray(g)
    bad_col[60 * 4 + 8 + 8 * 6:60 * 4 + 12 + 8 * 6] = (7).to_bytes(4, "little")
    over = [(ir.ZERO, [(0, 0)] * 7, [])]                              # one gate whose coefficient equals the modulus
    c_over = bytearray(ir.gate_coeffs(orc, fid, [(ir.ZERO, [(0, 0)] * 7, [1])]))
    c_over[4:36] = P.to_bytes(32, "little")
    sh_bad = hdr()
    for j in range(4):
        sh_bad.shift[3][j] = (P >> (64 * j)) & (2 ** 64 - 1)
    cases = {
        "null header": (fid, None, g, c),
        "unknown field": (2, hdr(), g, c),
        "n not a power of two": (fid, hdr(n=48), g, c),
        "n beyond 2^27": (fid, hdr(n=1 << 28), g, c),
        "zk_rows 2": (fid, hdr(zk_rows=2), g, c),
        "zk_rows n": (fid, hdr(zk_rows=n), g, c),
        "more gates than rows": (fid, hdr(n=8), g, c),
        "tag 14": (fid, hdr(), bytes(bad_tag), c),
        "wire row n": (fid, hdr(), bytes(bad_row), c),
        "wire col 7": (fid, hdr(), bytes(bad_col), c),
        "coefficients short": (fid, hdr(), g, c[:-1]),
        "coefficients long": (fid, hdr(), g, c + bytes(4)),
        "a record too few": (fid, hdr(), g + ir.pruned_gates(gates[:1]), c),
        "optional bit 6": (fid, hdr(optional=1 << 6), g, c),
        "shift not canonical": (fid, sh_bad, g, c),
        "coefficient not canonical": (fid, hdr(), ir.pruned_gates(over), bytes(c_over)),
    }
    for name, (f, h, gg, cc) in cases.items():
        rc, p = raw_build(ctx, f, h, gg, cc)
        assert (rc, p) == (-1, None), name
    assert raw_build(ctx, fid, hdr(), b"", b"", n_gates=3) == (-1, None)     # gates null with a count


def test_commitment_refusals(ctx, orc, vesta_srs):
    fid, n = 0, 64                                                             # Vesta's scalars: Fp
    gates, shifts = circuit(orc, fid, n, 10, seed=10)
    srs = srs_of(ctx, vesta_srs, 1 << 10)
    other = build(ctx, orc, 1, n, 3, gates, shifts)                            # over Fq
    endo = ev.mont(orc, fid, [1])[0]
    image = lambda secs, optional=0: write_cache("vk", {"public": 0, "prev_challenges": 0, "zk_rows": 3, "max_poly_size": n, "domain_d1_size": n,
                                                        "optional_selectors_present": optional, "endo_limbs": [int(x) for x in endo],
                                                        "shift_limbs": [[0] * 4] * 7}, secs)
    full = [(t, a.astype("<u8").tobytes(), d) for t, (a, d) in ir.sections(orc, fid, n, 3, gates, shifts).items()]
    missing = zk.IndexCache(ctx, image([s for s in full if s[0] != 0x22]))
    short = zk.IndexCache(ctx, image([s if s[0] != 0x24 else (0x24, s[1][:32 * 40], 0) for s in full]))
    no_opt = zk.IndexCache(ctx, image(full, optional=0b10))
    good = build(ctx, orc, fid, n, 3, gates, shifts)
    try:
        out = np.zeros((64, 8), dtype=np.uint64)
        k = ctypes.c_size_t()
        call = lambda idx, cap=64: zk.lib().zk_index_commitments(srs._h, idx._h if idx else None, out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)), cap, ctypes.byref(k))
        for name, idx in {"null index": None, "other field": other, "missing section": missing, "short section": short, "header bit": no_opt}.items():
            assert call(idx) == -1, name
        assert call(good, cap=27) == -1 and k.value == 28
        assert call(good) == 0 and k.value == 28
    finally:
        for h in (other, missing, short, no_opt, good, srs):
            h.close()


# ---------------------------------------------------------------------------------------------------------------- 8: streams, threads
def test_on_a_callers_stream(orc, vesta_srs):
    """both calls on a caller's stream, queued behind a spin kernel: the uploads of the gates and the gathers follow it"""
    fid, n, zk_rows = 0, 1 << 12, 4
    gates, shifts = circuit(orc, fid, n, 4000, seed=12)
    want = ir.sections(orc, fid, n, zk_rows, gates, shifts, 0b1)
    stream = torch.cuda.Stream()
    c = zk.Context(0)
    try:
        c.set_stream(stream.cuda_stream)
        srs = srs_of(c, vesta_srs, 1 << 16)
        srs.get_lagrange_basis_from_domain_size(n)
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            torch.cuda._sleep(20_000_000)
            idx = build(c, orc, fid, n, zk_rows, gates, shifts, 0b1)
            torch.cuda._sleep(20_000_000)
            got = srs.index_commitments(idx)
        for tag, (payload, dom) in want.items():
            assert np.array_equal(section(c, idx, tag)[0], payload), hex(tag)
        cols = {t: (a[::ir.domain_mult(t)]) for t, (a, _) in want.items()}
        assert np.array_equal(got, ir.commitments(orc, vesta_srs.cid, vesta_srs.g[:1 << 16], srs.h, cols, 0b1))
        idx.close()
        srs.close()
    finally:
        c.close()


def test_two_threads_share_a_context(ctx, orc):
    fid, n = 1, 1 << 10
    work = [circuit(orc, fid, n, 700 + t, seed=30 + t) for t in range(2)]
    want = [ir.sections(orc, fid, n, 5, g, s, 0b11) for g, s in work]
    errors = []

    def run(t):
        try:
            for _ in range(3):
                idx = build(ctx, orc, fid, n, 5, *work[t], 0b11)
                for tag, (payload, _) in want[t].items():
                    assert np.array_equal(section(ctx, idx, tag)[0], payload), hex(tag)
                idx.close()
        except Exception as e:             # noqa: BLE001 - reported below
            errors.append(e)
    th = [threading.Thread(target=run, args=(t,)) for t in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
