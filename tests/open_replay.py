"""Replay of the reference's `ser_regression_canonical_opening_proof` (poly-commitment/tests/commitment.rs:119-229, 388-443): the
first proof of `generate_random_opening_proof(StdRng seed [0; 32], group_map, SRS::<Vesta>::create(128))`, i.e. SRS::open
(ipa.rs:823-1061) on 11 random polynomials at 7 points.  Everything the reference does on the host around the folding rounds
(random stream, combine_polys utils.rs:103-202, b_init, sponge, group map, challenges, delta / z1 / z2, msgpack) is restated
here with Python integers (tests/rust_rng.py, tests/kimchi_transcript.py); the ROUNDS — the two MSMs, the inner products, the
folds of a, b and g — come from a backend: the CPU oracle (explicit point-by-point folding) or the device (`zk.IpaRounds`).
Test infrastructure only."""
import numpy as np

from kimchi_transcript import FP, FQ, BWGroupMap, DefaultFqSponge, endo_coefficient, scalar_challenge_to_field
from rust_rng import StdRng

GENERATOR_Y_VESTA = 11426906929455361843568202299992114520848200991084027513389447476559454104162
R_INV_FP = pow(1 << 256, -1, FP)
SRS_LEN = 128


def draw_fp(rng) -> int:
    """Fp::rand -> canonical integer (the drawn limbs are the Montgomery representation)"""
    limbs = rng.field_mont_limbs(FP)
    return sum(l << (64 * i) for i, l in enumerate(limbs)) * R_INV_FP % FP


class Points:
    """Vesta points as the oracle's affine Montgomery arrays <-> canonical integer coordinates"""

    def __init__(self, orc):
        self.orc, self.cid, self.fid = orc, orc.VESTA, orc.FQ

    def from_xy(self, x, y):
        return self.orc.to_mont(self.fid, self.orc.ints_to_limbs([x, y])).reshape(8)

    def xy(self, pt):
        if not np.any(pt):
            return None
        x, y = self.orc.limbs_to_ints(self.orc.from_mont(self.fid, np.ascontiguousarray(pt).reshape(2, 4)))
        return x, y

    def add(self, p, q):
        return self.orc.affine_add(self.cid, p, q)

    def mul(self, p, k):
        return self.orc.scalar_mul(self.cid, p, k % FP) if k % FP else np.zeros(8, dtype=np.uint64)

    def compress(self, pt) -> bytes:
        xy = self.xy(pt)
        if xy is None:
            return bytes(32) + b"\x40"
        return xy[0].to_bytes(32, "little") + bytes([0x80 if xy[1] > FQ - xy[1] else 0])


class OracleRounds:
    """the folding rounds exactly as ipa.rs:929-1007 writes them, bases folded point by point on the CPU oracle"""

    def __init__(self, orc, g, a, b):
        self.orc, self.g, self.a, self.b = orc, g.copy(), list(a), list(b)

    def lr(self):
        h = len(self.a) // 2
        a, b, g, orc = self.a, self.b, self.g, self.orc
        l = orc.msm(orc.VESTA, g[:h], orc.ints_to_limbs(a[h:]))
        r = orc.msm(orc.VESTA, g[h:], orc.ints_to_limbs(a[:h]))
        return l, r, sum(x * y for x, y in zip(a[h:], b[:h])) % FP, sum(x * y for x, y in zip(a[:h], b[h:])) % FP

    def fold(self, u, u_inv):
        h = len(self.a) // 2
        orc = self.orc
        self.a = [(self.a[i] + u_inv * self.a[i + h]) % FP for i in range(h)]
        self.b = [(self.b[i] + u * self.b[i + h]) % FP for i in range(h)]
        self.g = np.stack([orc.affine_add(orc.VESTA, self.g[i], orc.scalar_mul(orc.VESTA, self.g[i + h], u)) for i in range(h)])

    def finish(self):
        return self.a[0], self.b[0], self.g[0]


class DeviceRounds:
    """the same rounds on the device: proof_systems_b200.IpaRounds over the resident SRS table (csrc/ipa.cu)"""

    def __init__(self, orc, zk, ctx, g, a, b):
        self.orc, self.zk = orc, zk
        self.bases = ctx.upload_bases(zk.VESTA, g)
        mont = lambda xs: orc.to_mont(orc.FP, orc.ints_to_limbs(xs))
        self.rounds = zk.IpaRounds(ctx, self.bases, mont(a), mont(b))

    def lr(self):
        l, r, ipl, ipr = self.rounds.lr()
        aff = lambda p: self.zk.jacobian_to_affine(self.zk.VESTA, p)
        return aff(l), aff(r), self.orc.fe_int(self.orc.FP, ipl), self.orc.fe_int(self.orc.FP, ipr)

    def fold(self, u, u_inv):
        mont = lambda x: self.orc.to_mont(self.orc.FP, self.orc.ints_to_limbs([x]))[0]
        self.rounds.fold(mont(u), mont(u_inv))

    def finish(self):
        a0, b0 = self.rounds.state()
        sg = self.zk.jacobian_to_affine(self.zk.VESTA, self.rounds.sg())
        self.rounds.close()
        self.bases.free()
        return self.orc.fe_int(self.orc.FP, a0[0]), self.orc.fe_int(self.orc.FP, b0[0]), sg


def first_opening_proof_bytes(orc, vesta_srs, make_rounds) -> bytes:
    """make_rounds(g [128, 8], a [128 ints], b [128 ints]) -> a rounds backend; returns rmp-serde's bytes of the OpeningProof"""
    P = Points(orc)
    g = vesta_srs.g[:SRS_LEN]
    h = vesta_srs.mont_points(vesta_srs.h_xy_canon)[0]
    rng = StdRng(bytes(32))
    # ---- generate_random_opening_proof, first iteration (commitment.rs:135-203): only what `open` consumes; the commitments
    #      themselves are not part of the proof, but their blinders are drawn from the same stream
    elm = [draw_fp(rng) for _ in range(7)]
    polys = []
    for _ in range(11):
        ln = rng.next_u64() % 500                                         # `let len: usize = rng.gen(); len % 500`
        coeffs = [draw_fp(rng) for _ in range(ln + 1)] if ln else []       # DensePolynomial::rand(len, rng): len + 1 coefficients
        chunks = max(1, -(-len(coeffs) // SRS_LEN))                        # commit_non_hiding(poly, 1): ipa.rs:638-683
        polys.append((coeffs, [draw_fp(rng) for _ in range(chunks)]))      # srs.commit: one blinder per chunk (ipa.rs:686-693)
    polyscale, evalscale = draw_fp(rng), draw_fp(rng)

    # ---- SRS::open (ipa.rs:823-1061)
    endo_q = endo_coefficient(FQ)
    endo_r = endo_coefficient(FP)
    gen = P.from_xy(1, GENERATOR_Y_VESTA)
    if not np.array_equal(P.mul(gen, endo_r), P.from_xy(endo_q % FQ, GENERATOR_Y_VESTA)):     # ipa.rs:214-231
        endo_r = endo_r * endo_r % FP
    # combine_polys (utils.rs:103-202), coefficient-form polynomials only
    a = [0] * SRS_LEN
    blinding_factor, scale = 0, 1
    for coeffs, blinders in polys:
        off = 0
        for bl in blinders:
            for i, c in enumerate(coeffs[off:off + SRS_LEN]):
                a[i] = (a[i] + scale * c) % FP
            blinding_factor = (blinding_factor + bl * scale) % FP
            scale = scale * polyscale % FP
            off += SRS_LEN
    b, scale = [0] * SRS_LEN, 1
    for e in elm:                                                          # b_init (ipa.rs:848-861)
        t = 1
        for i in range(SRS_LEN):
            b[i] = (b[i] + scale * t) % FP
            t = t * e % FP
        scale = scale * evalscale % FP
    cip = sum(x * y for x, y in zip(a, b)) % FP
    sponge = DefaultFqSponge("fq")
    sponge.absorb_fr([(cip - (pow(2, 255, FP) + 1)) * pow(2, -1, FP) % FP])    # shift_scalar (commitment.rs:273-288): Fp < Fq
    u_base = P.from_xy(*BWGroupMap(FQ).to_group(sponge.challenge_fq()))
    rounds = make_rounds(g, a, b)
    lr, blinders, chals, chal_invs = [], [], [], []
    for _ in range(7):
        rand_l, rand_r = draw_fp(rng), draw_fp(rng)
        l_part, r_part, ip_l, ip_r = rounds.lr()
        l = P.add(P.add(l_part, P.mul(h, rand_l)), P.mul(u_base, ip_l))    # ipa.rs:938-948
        r = P.add(P.add(r_part, P.mul(h, rand_r)), P.mul(u_base, ip_r))    # ipa.rs:950-960
        lr.append((l, r))
        blinders.append((rand_l, rand_r))
        sponge.absorb_g([P.xy(l)])
        sponge.absorb_g([P.xy(r)])
        u = scalar_challenge_to_field(sponge.challenge(), endo_r, FP)
        u_inv = pow(u, -1, FP)
        chals.append(u)
        chal_invs.append(u_inv)
        rounds.fold(u, u_inv)
    a0, b0, g0 = rounds.finish()
    r_prime = blinding_factor
    for (rl, rr), u, ui in zip(blinders, chals, chal_invs):
        r_prime = (r_prime + rl * ui + rr * u) % FP
    d, r_delta = draw_fp(rng), draw_fp(rng)
    delta = P.add(P.mul(P.add(g0, P.mul(u_base, b0)), d), P.mul(h, r_delta))
    sponge.absorb_g([P.xy(delta)])
    c = scalar_challenge_to_field(sponge.challenge(), endo_r, FP)
    z1, z2 = (a0 * c + d) % FP, (r_prime * c + r_delta) % FP

    # ---- rmp-serde of OpeningProof{lr, delta, z1, z2, sg} (ipa.rs:1175-1191)
    pt = lambda p: b"\xc4\x21" + P.compress(p)
    fe = lambda x: b"\xc4\x20" + x.to_bytes(32, "little")
    return b"\x95" + bytes([0x90 | len(lr)]) + b"".join(b"\x92" + pt(l) + pt(r) for l, r in lr) + pt(delta) + fe(z1) + fe(z2) + pt(g0)


def opening_proof_bytes_product_level(orc, zk, ctx, vesta_srs) -> bytes:
    """The same proof through the PRODUCT-LEVEL entry point zk_srs_open (csrc/open.cu): combine_polys, b_init, the combined inner
    product, the rounds (h and U inside the MSMs), r_prime, delta, z1, z2 all run in the library; this function only draws the
    random stream in the reference's order and plays the transcript (sponge, group map, endo challenges) behind the callbacks."""
    P = Points(orc)
    g = vesta_srs.g[:SRS_LEN]
    h = vesta_srs.mont_points(vesta_srs.h_xy_canon)[0]
    rng = StdRng(bytes(32))
    elm = [draw_fp(rng) for _ in range(7)]
    polys = []
    for _ in range(11):
        ln = rng.next_u64() % 500
        coeffs = [draw_fp(rng) for _ in range(ln + 1)] if ln else []
        chunks = max(1, -(-len(coeffs) // SRS_LEN))
        polys.append((coeffs, [draw_fp(rng) for _ in range(chunks)]))
    polyscale, evalscale = draw_fp(rng), draw_fp(rng)
    draws = [draw_fp(rng) for _ in range(2 * 7 + 2)]                      # rand_l, rand_r per round, then d, r_delta (ipa.rs:936-937, 1027-1028)

    endo_q, endo_r = endo_coefficient(FQ), endo_coefficient(FP)
    gen = P.from_xy(1, GENERATOR_Y_VESTA)
    if not np.array_equal(P.mul(gen, endo_r), P.from_xy(endo_q % FQ, GENERATOR_Y_VESTA)):
        endo_r = endo_r * endo_r % FP
    mont = lambda xs: orc.to_mont(orc.FP, orc.ints_to_limbs(list(xs))) if len(xs) else np.zeros((0, 4), dtype=np.uint64)
    fe_int = lambda limbs: orc.fe_int(orc.FP, np.ascontiguousarray(limbs, dtype=np.uint64).reshape(4))
    sponge = DefaultFqSponge("fq")

    def u_base(cip):
        sponge.absorb_fr([(fe_int(cip) - (pow(2, 255, FP) + 1)) * pow(2, -1, FP) % FP])      # shift_scalar (commitment.rs:273-288)
        return P.from_xy(*BWGroupMap(FQ).to_group(sponge.challenge_fq()))

    def round_challenge(i, l, r):
        sponge.absorb_g([P.xy(l)])
        sponge.absorb_g([P.xy(r)])
        return mont([scalar_challenge_to_field(sponge.challenge(), endo_r, FP)])[0]

    def final_challenge(delta):
        sponge.absorb_g([P.xy(delta)])
        return mont([scalar_challenge_to_field(sponge.challenge(), endo_r, FP)])[0]

    with zk.SRS(ctx, zk.VESTA, g, h) as srs:
        plnms = [(mont(c), 0, mont(bl)) for c, bl in polys]
        proof = zk.srs_open(srs, plnms, mont(elm), mont([polyscale])[0], mont([evalscale])[0], mont(draws), u_base, round_challenge, final_challenge)
    pt = lambda p: b"\xc4\x21" + P.compress(p)
    fe = lambda x: b"\xc4\x20" + fe_int(x).to_bytes(32, "little")
    lr = proof.lr
    return (b"\x95" + bytes([0x90 | len(lr)]) + b"".join(b"\x92" + pt(l) + pt(r) for l, r in lr) + pt(proof.delta) + fe(proof.z1) + fe(proof.z2)
            + pt(proof.sg))
