"""SRS::verify (poly-commitment/src/ipa.rs:301-502) restated on the CPU oracle, and the batches its tests verify.

`oracle_verify` builds the reference's one big MSM — h || g || padding, then per proof sg, U, L_j, R_j, the commitment chunks, U,
delta — with Python integers for every scalar and the oracle's MSM, and returns the accumulated point (the batch verifies iff it is
the identity).  `reference_batch` replays the reference's randomised batch-verification test (poly-commitment/tests/commitment.rs:
119-257) on the StdRng([0; 32]) stream of tests/open_replay.py: 7 aggregated proofs over SRS::create(128), each with 7 evaluation
points and 11 random polynomials committed with blinders, a fresh Poseidon sponge per proof, then rand_base and sg_rand_base.  The
openings come from a backend: the oracle restatement of SRS::open below, or the device (zk_srs_open).  `HashTranscript` is a cheap
deterministic stand-in for the sponge (challenges are a hash of what was absorbed), for batches where Poseidon would dominate.
Test infrastructure only."""
import copy
import hashlib
from dataclasses import dataclass, field

import numpy as np

from kimchi_transcript import FP, FQ, BWGroupMap, DefaultFqSponge, endo_coefficient, scalar_challenge_to_field
from open_replay import GENERATOR_Y_VESTA, SRS_LEN, OracleRounds, Points, draw_fp
from rust_rng import StdRng

ZERO_PT = np.zeros(8, dtype=np.uint64)


@dataclass
class Opening:
    """ipa::OpeningProof with canonical integer scalars and affine Montgomery points"""
    lr: list
    delta: np.ndarray
    z1: int
    z2: int
    sg: np.ndarray


@dataclass
class Entry:
    """one BatchEvaluationProof: `transcript()` makes the proof's fresh sponge (an object with u_base(cip) -> U, round(j, L, R) -> u,
    final(delta) -> c); comms: one uint64 [chunks, 8] array per evaluation (0 chunks = an empty PolyComm)"""
    opening: Opening
    elm: list
    polyscale: int
    evalscale: int
    comms: list
    cip: int
    transcript: object
    extra: dict = field(default_factory=dict)


def b_poly(chals, x, m):
    """commitment.rs:426-436"""
    k = len(chals)
    pw = [x]
    for _ in range(1, k):
        pw.append(pw[-1] * pw[-1] % m)
    r = 1
    for i in range(k):
        r = r * (1 + chals[i] * pw[k - 1 - i]) % m
    return r


def b_poly_coefficients(chals, m):
    """commitment.rs:464-476: s[i] = prod over set bits t of i of chals[k-1-t]"""
    k = len(chals)
    s = [1] * (1 << k)
    for i in range(1, 1 << k):
        t = i.bit_length() - 1
        s[i] = s[i - (1 << t)] * chals[k - 1 - t] % m
    return s


def oracle_verify(orc, cid, g, h, batch, rand_base, sg_rand_base):
    """SRS::verify up to the comparison with zero: the accumulated point, affine [8] (zeros = the identity)"""
    m = orc.MODULUS[orc.SCALAR_FIELD[cid]]
    n = g.shape[0]
    padded = 1 << (n - 1).bit_length()
    points = [h] + list(g) + [ZERO_PT] * (padded - n)
    scalars = [0] * (padded + 1)
    r_i = w_i = 1
    for e in batch:
        op, tr = e.opening, e.transcript()
        u_base = tr.u_base(e.cip)
        chal = [tr.round(j, l, r) for j, (l, r) in enumerate(op.lr)]
        chal_inv = [pow(u, -1, m) if u else 0 for u in chal]          # ark_ff::batch_inversion leaves zeros alone
        c = tr.final(op.delta)
        b0, sc = 0, 1
        for x in e.elm:
            b0 = (b0 + sc * b_poly(chal, x, m)) % m
            sc = sc * e.evalscale % m
        s = b_poly_coefficients(chal, m)
        points.append(op.sg)
        scalars.append(-r_i * op.z1 - w_i)
        for i, v in enumerate(s):
            scalars[i + 1] += w_i * v                                  # IndexError past the padded length, as the reference panics
        scalars[0] -= r_i * op.z2
        points.append(u_base)
        scalars.append(-r_i * op.z1 * b0)
        rc = c * r_i % m
        for (l, r), ui, u in zip(op.lr, chal_inv, chal):
            points += [l, r]
            scalars += [rc * ui, rc * u]
        ps = 1
        for comm in e.comms:                                           # combine_commitments: empty ones are skipped
            for ch in comm:
                points.append(ch)
                scalars.append(rc * ps)
                ps = ps * e.polyscale % m
        points.append(u_base)
        scalars.append(rc * e.cip)
        points.append(op.delta)
        scalars.append(r_i)
        r_i = r_i * rand_base % m
        w_i = w_i * sg_rand_base % m
    return orc.msm(cid, np.stack(points), orc.ints_to_limbs([x % m for x in scalars]))


# ---------------------------------------------------------------------------------------------- transcripts
def vesta_endo_r(orc):
    """ipa.rs:214-231: the endo coefficient of the scalar field that matches the curve's endomorphism"""
    P = Points(orc)
    endo_q, endo_r = endo_coefficient(FQ), endo_coefficient(FP)
    gen = P.from_xy(1, GENERATOR_Y_VESTA)
    if not np.array_equal(P.mul(gen, endo_r), P.from_xy(endo_q % FQ, GENERATOR_Y_VESTA)):
        endo_r = endo_r * endo_r % FP
    return endo_r


class PoseidonTranscript:
    """DefaultFqSponge over Vesta with the BW group map: the reference's transcript of SRS::open / SRS::verify (ipa.rs:372-383)"""

    def __init__(self, orc, endo_r):
        self.P, self.endo_r = Points(orc), endo_r
        self.sponge = DefaultFqSponge("fq")

    def u_base(self, cip):
        self.sponge.absorb_fr([(cip - (pow(2, 255, FP) + 1)) * pow(2, -1, FP) % FP])     # shift_scalar (commitment.rs:273-288)
        return self.P.from_xy(*BWGroupMap(FQ).to_group(self.sponge.challenge_fq()))

    def round(self, j, l, r):
        self.sponge.absorb_g([self.P.xy(l)])
        self.sponge.absorb_g([self.P.xy(r)])
        return scalar_challenge_to_field(self.sponge.challenge(), self.endo_r, FP)

    def final(self, delta):
        self.sponge.absorb_g([self.P.xy(delta)])
        return scalar_challenge_to_field(self.sponge.challenge(), self.endo_r, FP)


class HashTranscript:
    """Stand-in sponge: every challenge is SHA-256 of everything absorbed so far (mod the scalar modulus); U is one of `u_points`
    picked by that hash.  Open and verify absorb the same values, so they derive the same challenges.  zero_round: that round's
    challenge is 0 (a transcript the reference's verifier accepts as input)."""

    def __init__(self, m, u_points, seed=0, zero_round=None):
        self.m, self.u_points, self.zero_round = m, u_points, zero_round
        self.h = hashlib.sha256(seed.to_bytes(8, "little"))

    def _absorb(self, *arrays):
        for a in arrays:
            self.h.update(np.ascontiguousarray(a, dtype=np.uint64).tobytes())
        return int.from_bytes(self.h.digest(), "little")

    def u_base(self, cip):
        return self.u_points[self._absorb(np.array([cip % (1 << 64), cip >> 64 & (2**64 - 1), cip >> 128 & (2**64 - 1), cip >> 192], dtype=np.uint64))
                             % len(self.u_points)]

    def round(self, j, l, r):
        u = self._absorb(l, r) % self.m
        return 0 if j == self.zero_round else (u or 1)

    def final(self, delta):
        return self._absorb(delta) % self.m


# ---------------------------------------------------------------------------------------------- openings
def oracle_open(orc, g, h, polys, elm, polyscale, evalscale, draws, tr):
    """SRS::open (ipa.rs:823-1061) for Vesta coefficient-form polynomials, restated as in tests/open_replay.py with the rounds on the
    oracle; polys: (coeffs, blinders) integer lists; draws: rand_l, rand_r per round, then d, r_delta"""
    P = Points(orc)
    n = g.shape[0]
    a = [0] * n
    blinding_factor, scale = 0, 1
    for coeffs, blinders in polys:
        off = 0
        for bl in blinders:
            for i, c in enumerate(coeffs[off:off + n]):
                a[i] = (a[i] + scale * c) % FP
            blinding_factor = (blinding_factor + bl * scale) % FP
            scale = scale * polyscale % FP
            off += n
    b, scale = [0] * n, 1
    for e in elm:
        t = 1
        for i in range(n):
            b[i] = (b[i] + scale * t) % FP
            t = t * e % FP
        scale = scale * evalscale % FP
    cip = sum(x * y for x, y in zip(a, b)) % FP
    u_base = tr.u_base(cip)
    rounds = OracleRounds(orc, g, a, b)
    k = (n - 1).bit_length()
    lr, chals, chal_invs = [], [], []
    for j in range(k):
        rand_l, rand_r = draws[2 * j], draws[2 * j + 1]
        l_part, r_part, ip_l, ip_r = rounds.lr()
        l = P.add(P.add(l_part, P.mul(h, rand_l)), P.mul(u_base, ip_l))
        r = P.add(P.add(r_part, P.mul(h, rand_r)), P.mul(u_base, ip_r))
        lr.append((l, r))
        u = tr.round(j, l, r)
        chals.append(u)
        chal_invs.append(pow(u, -1, FP))
        rounds.fold(u, chal_invs[-1])
    a0, b0, g0 = rounds.finish()
    r_prime = blinding_factor
    for j in range(k):
        r_prime = (r_prime + draws[2 * j] * chal_invs[j] + draws[2 * j + 1] * chals[j]) % FP
    d, r_delta = draws[2 * k], draws[2 * k + 1]
    delta = P.add(P.mul(P.add(g0, P.mul(u_base, b0)), d), P.mul(h, r_delta))
    c = tr.final(delta)
    return Opening(lr, delta, (a0 * c + d) % FP, (r_prime * c + r_delta) % FP, g0)


def device_open(zk, orc, srs, sfid, polys_mont, elm, polyscale, evalscale, draws, tr):
    """the same through zk_srs_open; polys_mont: (coeffs [len, 4], blinders [k, 4]) Montgomery arrays, scalars integers.
    Returns (Opening, the combined inner product the library passed to u_base)"""
    mont = lambda xs: orc.to_mont(sfid, orc.ints_to_limbs(list(xs)))
    fe_int = lambda limbs: orc.fe_int(sfid, np.ascontiguousarray(limbs, dtype=np.uint64).reshape(4))
    seen = {}

    def u_base(cip):
        seen["cip"] = fe_int(cip)
        return tr.u_base(seen["cip"])

    proof = zk.srs_open(srs, [(c, 0, bl) for c, bl in polys_mont], mont(elm), mont([polyscale])[0], mont([evalscale])[0], mont(draws), u_base,
                        lambda j, l, r: mont([tr.round(j, l, r)])[0], lambda d: mont([tr.final(d)])[0])
    op = Opening([(l.copy(), r.copy()) for l, r in proof.lr], proof.delta, fe_int(proof.z1), fe_int(proof.z2), proof.sg)
    return op, seen["cip"]


def to_device(zk, orc, sfid, e):
    """Entry -> zk.BatchEvaluationProof with a fresh transcript behind limb-level callbacks"""
    mont = lambda xs: orc.to_mont(sfid, orc.ints_to_limbs(list(xs))) if len(xs) else np.zeros((0, 4), dtype=np.uint64)
    fe_int = lambda limbs: orc.fe_int(sfid, np.ascontiguousarray(limbs, dtype=np.uint64).reshape(4))
    op, tr = e.opening, e.transcript()
    opening = zk.OpeningProof(np.array([[l, r] for l, r in op.lr], dtype=np.uint64).reshape(-1, 2, 8), op.delta, mont([op.z1])[0],
                              mont([op.z2])[0], op.sg)
    return zk.BatchEvaluationProof(opening, mont(e.elm), mont([e.polyscale])[0], mont([e.evalscale])[0], e.comms, mont([e.cip])[0],
                                   lambda cip: tr.u_base(fe_int(cip)), lambda j, l, r: mont([tr.round(j, l, r)])[0],
                                   lambda d: mont([tr.final(d)])[0])


# ---------------------------------------------------------------------------------------------- the reference's batch
def commit(orc, g, h, coeffs, blinders):
    """srs.commit(poly, 1, rng) with the drawn blinders: commit_non_hiding (ipa.rs:638-683) then mask_custom (ipa.rs:605-622)"""
    P, n = Points(orc), g.shape[0]
    chunks = [orc.msm(orc.VESTA, g[:len(coeffs[o:o + n])], orc.ints_to_limbs(coeffs[o:o + n])) for o in range(0, len(coeffs), n)] or [ZERO_PT]
    return np.stack([P.add(c, P.mul(h, bl)) if c.any() else P.mul(h, bl) for c, bl in zip(chunks, blinders)])


def combined_inner_product(coeff_lists, elm, polyscale, evalscale, n):
    """commitment.rs:622-657 over the chunked evaluations of the polynomials (to_chunked_polynomial(num_chunks, n).evaluate_chunks)"""
    res, ps = 0, 1
    for coeffs in coeff_lists:
        for o in range(0, max(1, len(coeffs)), n):
            chunk, acc, es = coeffs[o:o + n], 0, 1
            for x in elm:
                ev = 0
                for c in reversed(chunk):
                    ev = (ev * x + c) % FP
                acc = (acc + es * ev) % FP
                es = es * evalscale % FP
            res = (res + ps * acc) % FP
            ps = ps * polyscale % FP
    return res


def reference_batch(orc, vesta_srs, opener):
    """(entries, rand_base, sg_rand_base, g, h) of commitment.rs:119-257; opener(polys, elm, polyscale, evalscale, draws, transcript) ->
    Opening makes each proof (oracle_open or device_open on SRS::create(128))"""
    g = vesta_srs.g[:SRS_LEN]
    h = vesta_srs.mont_points(vesta_srs.h_xy_canon)[0]
    endo_r = vesta_endo_r(orc)
    rng = StdRng(bytes(32))
    entries = []
    for _ in range(7):
        elm = [draw_fp(rng) for _ in range(7)]
        polys, comms = [], []
        for _ in range(11):
            ln = rng.next_u64() % 500                                          # `let len: usize = rng.gen(); len % 500`
            coeffs = [draw_fp(rng) for _ in range(ln + 1)] if ln else []       # DensePolynomial::rand(len): len + 1 coefficients
            blinders = [draw_fp(rng) for _ in range(max(1, -(-len(coeffs) // SRS_LEN)))]
            polys.append((coeffs, blinders))
            comms.append(commit(orc, g, h, coeffs, blinders))
        polyscale, evalscale = draw_fp(rng), draw_fp(rng)
        draws = [draw_fp(rng) for _ in range(2 * 7 + 2)]                        # rand_l, rand_r per round, then d, r_delta
        make_tr = lambda: PoseidonTranscript(orc, endo_r)
        opening = opener(polys, elm, polyscale, evalscale, draws, make_tr())
        cip = combined_inner_product([c for c, _ in polys], elm, polyscale, evalscale, SRS_LEN)
        entries.append(Entry(opening, elm, polyscale, evalscale, comms, cip, make_tr))
    rand_base, sg_rand_base = draw_fp(rng), draw_fp(rng)                        # SRS::verify's draws (ipa.rs:357-358)
    return entries, rand_base, sg_rand_base, g, h


def opening_bytes(orc, op) -> bytes:
    """rmp-serde of OpeningProof{lr, delta, z1, z2, sg} (ipa.rs:1175-1191), Vesta"""
    P = Points(orc)
    pt = lambda p: b"\xc4\x21" + P.compress(p)
    fe = lambda x: b"\xc4\x20" + x.to_bytes(32, "little")
    return (b"\x95" + bytes([0x90 | len(op.lr)]) + b"".join(b"\x92" + pt(l) + pt(r) for l, r in op.lr) + pt(op.delta) + fe(op.z1) + fe(op.z2)
            + pt(op.sg))


TAMPERINGS = ["z1", "z2", "swap_lr", "chunk", "cip", "sg", "bad_proof"]


def tamper(entries, kind, m, other_point, at=2):
    """a copy of the batch with one change to entry `at`"""
    out = [copy.copy(e) for e in entries]
    e = out[at]
    op = copy.copy(e.opening)
    e.opening = op
    if kind == "z1":
        op.z1 = (op.z1 + 1) % m
    elif kind == "z2":
        op.z2 = (op.z2 + 1) % m
    elif kind == "swap_lr":
        op.lr = list(op.lr)
        op.lr[1] = (op.lr[1][1], op.lr[1][0])
    elif kind == "chunk":
        e.comms = list(e.comms)
        q = next(i for i, c in enumerate(e.comms) if c.shape[0])
        e.comms[q] = e.comms[q].copy()
        e.comms[q][0] = other_point
    elif kind == "cip":
        e.cip = (e.cip + 1) % m
    elif kind == "sg":
        op.sg = other_point
    elif kind == "bad_proof":
        e.opening = entries[(at + 1) % len(entries)].opening
    else:
        raise ValueError(kind)
    return out
