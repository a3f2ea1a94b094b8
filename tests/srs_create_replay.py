"""Restatement (test infrastructure, Python integers) of `SRS::create(depth)` (poly-commitment/src/ipa.rs:234-265, 561-590,
751-778) for the curves y^2 = x^3 + 5 over the Pasta fields:

  g[i] = point_of_random_bytes(Blake2b512(u32_be(i)))          i = 0 .. depth - 1
  h    = point_of_random_bytes(Blake2b512(b"srs_misc" || u32_be(0)))

point_of_random_bytes takes digest bytes 0..30 as bits `bits[8i + j] = (d[i] >> j) & 1` and reads them with
BigInt::from_bits_be (bits[0] is the most significant bit): every byte bit-reversed, the bytes big-endian.  That integer
t < 2^248 is an element of the curve's base field, fed to the BW group map (groupmap/src/lib.rs, `kimchi_transcript.BWGroupMap`);
the Pasta cofactor is 1, so the map's point is the generator.  Pure Python: about 3 ms per point, so tests sample indices."""
import hashlib

from kimchi_transcript import FP, FQ, BWGroupMap

PALLAS, VESTA = 0, 1
BASE_MODULUS = {PALLAS: FP, VESTA: FQ}
_MAPS = {}


def group_map(curve: int) -> BWGroupMap:
    if curve not in _MAPS:
        _MAPS[curve] = BWGroupMap(BASE_MODULUS[curve])
    return _MAPS[curve]


def digest(msg: bytes) -> bytes:
    return hashlib.blake2b(msg, digest_size=64).digest()


def rev8(b: int) -> int:
    return int(format(b, "08b")[::-1], 2)


def pack(d: bytes) -> int:
    """digest -> t: bytes 0..30, each bit-reversed, read big-endian"""
    return int.from_bytes(bytes(rev8(b) for b in d[:31]), "big")


def point_of_random_bytes(curve: int, msg: bytes):
    """(x, y) canonical integers"""
    return group_map(curve).to_group(pack(digest(msg)))


def generator(curve: int, i: int):
    return point_of_random_bytes(curve, i.to_bytes(4, "big"))


def blinder(curve: int):
    return point_of_random_bytes(curve, b"srs_misc" + (0).to_bytes(4, "big"))


def compress(curve: int, pt) -> bytes:
    """ark-serialize's 33-byte compressed form: x little-endian, flag bit 7 when y is the larger of {y, p - y}"""
    x, y = pt
    p = BASE_MODULUS[curve]
    return x.to_bytes(32, "little") + bytes([0x80 if y > p - y else 0])


def xy_bytes(pt) -> bytes:
    """64 bytes canonical little-endian x || y (the fixtures' h_xy layout)"""
    return pt[0].to_bytes(32, "little") + pt[1].to_bytes(32, "little")
