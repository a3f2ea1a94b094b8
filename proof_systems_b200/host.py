"""Host-side mirrors of the reference interfaces on the MSM/NTT path, over the C ABI (srs.cu holds the policy code).

Names, argument meaning and error behaviour follow the reference so that the parity tests read like its own:
  poly_commitment::SRS / ipa::SRS<G>                  poly-commitment/src/lib.rs:61-241, ipa.rs:56-75,596-800
  poly_commitment::PolyComm<C>{chunks}                poly-commitment/src/commitment.rs:47-50
  poly_commitment::error::CommitmentError             poly-commitment/src/error.rs:3-9
  ark_poly::Radix2EvaluationDomain<F>                 used as `D` in kimchi/src/prover.rs:39-42, circuits/domains.rs:24-33
"""
from __future__ import annotations

import ctypes
import os
from dataclasses import dataclass

import numpy as np

from ._lib import (BASE_FIELD, FINAL_CB, FP, FQ, ROUND_CB, SCALAR_FIELD, U_BASE_CB, Context, Handle, IndexHeader, LookupInfo, LookupJoint,
                   LookupTable, LookupTerm, OpenPoly, OpenTranscript, RuntimeTableCfg, VerifyProof, ZkError, _fe, _np_u64, _ptr, _u64p, check,
                   jacobian_to_affine, lib)


class LookupIndexError(ZkError):
    """LookupError of LookupConstraintSystem::create (kimchi/src/circuits/lookup/index.rs:23-36): kind is ID_COLLISION
    (LookupTableIdCollision), TABLE_ID_ZERO (TableIDZeroMustHaveZeroEntry) or TOO_LONG (LookupTableTooLong); message the reference's"""
    ID_COLLISION, TABLE_ID_ZERO, TOO_LONG = 1, 2, 3

    def __init__(self, kind: int, message: str):
        super().__init__(-1, message)
        self.kind, self.message = kind, message


class BlindersDontMatch(ValueError):
    """CommitmentError::BlindersDontMatch(blinders_len, commitment_len)"""


@dataclass
class PolyComm:
    """chunks: uint64 [k, 8] affine points (identity = zeros)"""
    chunks: np.ndarray

    def __len__(self):
        return self.chunks.shape[0]


class SRS(Handle):
    """ipa::SRS<G>{g, h, lagrange_bases} with g (and every registered Lagrange basis) resident on the device."""

    def __init__(self, ctx: Context, curve: int, g, h, window_bits: int = -1, _create=None):
        """_create(g, h, out): the library call that writes the handle, and g and h with it (SRS.create); by default zk_srs_create
        of g and h"""
        self.ctx, self.curve = ctx, curve
        self.g = _np_u64(g, (8,))
        self.h = _fe(h, 8)
        if _create is None:
            _create = lambda g, h, out: lib().zk_srs_create(ctx._h, curve, _ptr(g), g.shape[0], h.ctypes.data_as(_u64p), window_bits, out)
        self._h = ctypes.c_void_p()
        check(_create(self.g, self.h, ctypes.byref(self._h)))

    # fn create(depth: usize) -> Self
    @classmethod
    def create(cls, ctx: Context, curve: int, depth: int, window_bits: int = -1) -> "SRS":
        """SRS::create (ipa.rs:751-778): g[0..depth) and h hashed to the curve on the device (zk_srs_generate), bit-exact with the
        reference; `g` and `h` are the host copies of the points the handle holds."""
        return cls(ctx, curve, np.empty((depth, 8), dtype=np.uint64), np.empty(8, dtype=np.uint64), _create=lambda g, h, out: lib().zk_srs_generate(
            ctx._h, curve, depth, window_bits, g.ctypes.data_as(_u64p), h.ctypes.data_as(_u64p), out))

    @classmethod
    def from_file(cls, ctx: Context, curve: int, path: str, window_bits: int = -1, lagrange: bool = True) -> "SRS":
        """Load srs/{pallas,vesta}.srs or srs/test_{pallas,vesta}.srs (precomputed_srs.rs:76-91 get_srs / get_srs_test): the points
        are decoded on the device; the Lagrange bases stored in a test file populate the cache (single-chunk bases only)."""
        from . import srs_file
        f = srs_file.read_srs(path)
        dec = ctx.decompress_points if f.compressed else ctx.points_from_uncompressed
        srs = cls(ctx, curve, dec(curve, f.g), dec(curve, f.h.reshape(1, -1))[0], window_bits)
        if lagrange:
            for n, basis in f.lagrange_bases.items():
                if basis.shape[1] == 1:
                    srs.add_lagrange_basis(n, ctx.points_from_uncompressed(curve, basis[:, 0]))
        return srs

    def _release(self, h):
        lib().zk_srs_destroy(h)

    # fn max_poly_size(&self) -> usize  /  fn size(&self)
    def max_poly_size(self) -> int:
        return int(lib().zk_srs_max_poly_size(self._h))

    size = max_poly_size

    def blinding_commitment(self) -> np.ndarray:
        return self.h

    def add_lagrange_basis(self, domain_size: int, basis, window_bits: int = -1):
        """Populate the cache behind get_lagrange_basis(domain) (ipa.rs:780-795) with a precomputed basis."""
        b = _np_u64(basis, (8,))
        assert b.shape[0] == domain_size * self.lagrange_basis_chunks(domain_size)      # chunk-major for domains larger than the SRS
        check(lib().zk_srs_add_lagrange_basis(self._h, domain_size, _ptr(b), window_bits))

    def lagrange_basis_chunks(self, domain_size: int) -> int:
        """chunks per basis element: ceil(domain / |g|) (ipa.rs:1145)"""
        return int(lib().zk_srs_lagrange_basis_chunks(self._h, domain_size))

    # fn get_lagrange_basis_from_domain_size(&self, domain_size: usize) -> &Vec<PolyComm<G>>
    def get_lagrange_basis_from_domain_size(self, domain_size: int, window_bits: int = -1) -> np.ndarray:
        """Computes (once) the basis on the device — SRS::lagrange_basis, ipa.rs:1065-1172 — and returns it: [n, 8] affine, or
        [chunks, n, 8] (chunk-major: PolyComm i of the reference is out[:, i]) when the domain is larger than the SRS."""
        check(lib().zk_srs_lagrange_basis(self._h, domain_size, window_bits))
        chunks = self.lagrange_basis_chunks(domain_size)
        out = np.empty((chunks * domain_size, 8), dtype=np.uint64)
        check(lib().zk_srs_get_lagrange_basis(self._h, domain_size, out.ctypes.data_as(_u64p), chunks * domain_size))
        return out if chunks == 1 else out.reshape(chunks, domain_size, 8)

    # fn commit_non_hiding(&self, plnm: &DensePolynomial<F>, num_chunks: usize) -> PolyComm<G>
    def commit_non_hiding(self, coeffs, num_chunks: int) -> PolyComm:
        c = _np_u64(coeffs, (4,)) if len(coeffs) else np.zeros((0, 4), dtype=np.uint64)
        cap = max(num_chunks, (c.shape[0] + self.g.shape[0] - 1) // self.g.shape[0], 1)
        out = np.zeros((cap, 8), dtype=np.uint64)
        k = ctypes.c_size_t()
        check(lib().zk_srs_commit_non_hiding(self._h, _ptr(c) if c.size else None, c.shape[0], num_chunks,
                                             out.ctypes.data_as(_u64p), cap, ctypes.byref(k)))
        return PolyComm(out[: k.value])

    # fn commit_evaluations_non_hiding(&self, domain: D<F>, plnm: &Evaluations<F, D<F>>) -> PolyComm<G>
    def commit_evaluations_non_hiding(self, domain_size: int, evals) -> PolyComm:
        e = _np_u64(evals, (4,))
        out = np.zeros((max(1, self.lagrange_basis_chunks(domain_size)), 8), dtype=np.uint64)
        check(lib().zk_srs_commit_evaluations_non_hiding(self._h, domain_size, _ptr(e), e.shape[0], out.ctypes.data_as(_u64p)))
        return PolyComm(out)

    def commit_evaluations_non_hiding_batch(self, domain_size: int, evals) -> list:
        """[commit_evaluations_non_hiding(domain, e) for e in evals] in one call: evals uint64 [k, domain_size, 4].  The
        reference computes the witness commitments concurrently (kimchi/src/prover.rs:329-351); here the k MSMs share lanes."""
        e = np.ascontiguousarray(evals, dtype=np.uint64)
        if e.ndim != 3 or e.shape[1:] != (domain_size, 4):
            raise ValueError("expected uint64 [k, domain_size, 4]")
        out = np.zeros((e.shape[0], 8), dtype=np.uint64)
        check(lib().zk_srs_commit_evaluations_batch(self._h, domain_size, _ptr(e), e.shape[0], out.ctypes.data_as(_u64p)))
        return [PolyComm(out[j:j + 1]) for j in range(e.shape[0])]

    # fn mask_custom(&self, com: PolyComm<G>, blinders: &PolyComm<F>) -> Result<BlindedCommitment<G>, CommitmentError>
    def mask_custom(self, com: PolyComm, blinders) -> PolyComm:
        b = _np_u64(blinders, (4,))
        out = np.zeros_like(com.chunks)
        try:
            check(lib().zk_srs_mask_custom(self._h, _ptr(com.chunks), len(com), _ptr(b), b.shape[0], out.ctypes.data_as(_u64p)))
        except ZkError as e:
            if e.code == -4:
                raise BlindersDontMatch(b.shape[0], len(com)) from e
            raise
        return PolyComm(out)

    def commit_custom(self, coeffs, num_chunks: int, blinders) -> PolyComm:
        return self.mask_custom(self.commit_non_hiding(coeffs, num_chunks), blinders)

    def commit_evaluations_custom(self, domain_size: int, evals, blinders) -> PolyComm:
        return self.mask_custom(self.commit_evaluations_non_hiding(domain_size, evals), blinders)

    def index_commitments(self, index: "IndexCache") -> np.ndarray:
        """zk_index_commitments: the commitments of ProverIndex::verifier_index (kimchi/src/verifier_index.rs:221-300) of a built or
        loaded index, uint64 [count, chunks, 8] affine: sigma 0..6, coefficients 0..14, generic, psm, complete_add, mul, emul,
        endomul_scalar (those six masked with blinder one), then the present optional selectors in bit order."""
        n = index.header.domain_d1_size
        chunks = self.lagrange_basis_chunks(n)
        count = 7 + 15 + 6 + bin(index.header.optional_selectors_present).count("1")
        out = np.zeros((count * chunks, 8), dtype=np.uint64)
        k = ctypes.c_size_t()
        check(lib().zk_index_commitments(self._h, index._h, out.ctypes.data_as(_u64p), out.shape[0], ctypes.byref(k)))
        return out[: k.value].reshape(-1, chunks, 8)


    def lookup_index_commitments(self, index: "IndexCache") -> np.ndarray:
        """zk_lookup_index_commitments: the commitments of LookupVerifierIndex (kimchi/src/verifier_index.rs:196-215), uint64
        [count, chunks, 8] affine: lookup_table[0 .. w) and table_ids (masked with blinder one), then the present selectors xor,
        lookup, range_check, ffmul and runtime_tables_selector."""
        n = index.header.domain_d1_size
        chunks = self.lagrange_basis_chunks(n)
        count = index.section(0x50)[2] + bin(index.header.lookup_selectors_present & 0x3F).count("1")
        out = np.zeros((count * chunks, 8), dtype=np.uint64)
        k = ctypes.c_size_t()
        check(lib().zk_lookup_index_commitments(self._h, index._h, out.ctypes.data_as(_u64p), out.shape[0], ctypes.byref(k)))
        return out[: k.value].reshape(-1, chunks, 8)


class IndexCache(Handle):
    """A cached prover index (kimchi/src/cached_prover_index.rs:26-56, "MINAPK01") resident on the device: zk_index_cache_load parses the
    header and the section table and copies the payload as it lies in the file — raw Montgomery limbs are the device format."""

    def __init__(self, ctx: Context, image: bytes | None = None, expect_identifier: str | None = None, _create=None):
        """_create(out): the library call that writes the handle (IndexCache.build); by default zk_index_cache_load of image"""
        if _create is None:
            buf = np.frombuffer(image, dtype=np.uint8)
            ident = expect_identifier.encode() if expect_identifier is not None else None
            _create = lambda out: lib().zk_index_cache_load(ctx._h, ctypes.c_void_p(buf.ctypes.data), buf.size, ident, out)
        self.ctx, self._h = ctx, ctypes.c_void_p()
        check(_create(ctypes.byref(self._h)))
        self.header = IndexHeader()
        if self._h:                     # IndexCache.build_lookup: no handle when the circuit has no lookup
            check(lib().zk_index_cache_header(self._h, ctypes.byref(self.header)))

    @classmethod
    def build(cls, ctx: Context, fid: int, header, gates: bytes, gate_coeffs: bytes, zero_selectors: bool = False) -> "IndexCache":
        """zk_index_build: the prover index's column evaluations (constraints.rs:510-760) built on the device from the circuit's gates
        in the cache file's encodings — `gates` the PrunedGate records (60 bytes each), `gate_coeffs` the GateCoeffs records — and an
        IndexHeader with domain_d1_size, zk_rows, shift and optional_selectors_present set.  zero_selectors: the reference's
        `cfg!(debug_assertions) && disable_gates_checks`."""
        g, c = bytes(gates), bytes(gate_coeffs)
        if len(g) % 60:
            raise ValueError("gates: a whole number of 60-byte PrunedGate records expected")
        return cls(ctx, _create=lambda out: lib().zk_index_build(ctx._h, fid, ctypes.byref(header), g or None, len(g) // 60, c or None, len(c),
                                                                int(zero_selectors), out))

    @classmethod
    def build_lookup(cls, ctx: Context, fid: int, n: int, zk_rows: int, gates: bytes, tables, runtime=None):
        """zk_lookup_index_build: LookupConstraintSystem::create (kimchi/src/circuits/lookup/index.rs:202-482) on the device.  gates:
        PrunedGate records as for build; tables: the fixed LookupTables as (id, data), data Montgomery uint64 [width, len, 4] (its
        columns); runtime: None or the RuntimeTableCfgs as (id, first_column), first_column Montgomery uint64 [len, 4].  Returns
        (IndexCache, runtime_table_offset or None), or (None, None) when no gate uses a lookup; raises LookupIndexError for the
        reference's LookupErrors."""
        g = bytes(gates)
        if len(g) % 60:
            raise ValueError("gates: a whole number of 60-byte PrunedGate records expected")
        keep = []                       # the arrays the structures point into, alive until the call returns
        fixed = (LookupTable * max(1, len(tables)))()
        for k, (tid, data) in enumerate(tables):
            d = np.ascontiguousarray(data, dtype=np.uint64)
            if d.ndim != 3 or d.shape[2] != 4:
                raise ValueError("a table's data: uint64 [width, len, 4] expected")
            keep.append(d)
            fixed[k] = LookupTable(tid, d.shape[0], d.shape[1], d.ctypes.data if d.size else None)
        rts = runtime or []
        rt = (RuntimeTableCfg * max(1, len(rts)))()
        for k, (tid, col) in enumerate(rts):
            c = _np_u64(col, (4,)) if len(col) else np.zeros((0, 4), dtype=np.uint64)
            keep.append(c)
            rt[k] = RuntimeTableCfg(tid, c.shape[0], c.ctypes.data if c.size else None)
        err, off = ctypes.c_int(), ctypes.c_uint64()

        def create(out):
            rc = lib().zk_lookup_index_build(ctx._h, fid, n, zk_rows, g or None, len(g) // 60, fixed, len(tables), rt, len(rts),
                                             int(runtime is not None), ctypes.byref(err), ctypes.byref(off), out)
            if rc and err.value:
                raise LookupIndexError(err.value, lib().zk_last_error().decode(errors="replace"))
            return rc
        idx = cls(ctx, _create=create)
        if not idx._h:
            return None, None
        return idx, (off.value if runtime is not None else None)

    @classmethod
    def from_file(cls, ctx: Context, path: str, expect_identifier: str | None = None) -> "IndexCache":
        import mmap
        with open(path, "rb") as f:
            mm = mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ)
        return cls(ctx, mm, expect_identifier)

    def section(self, tag: int):
        """(device pointer, element count, declared domain size) of a field-element section"""
        p, n, d = ctypes.c_void_p(), ctypes.c_size_t(), ctypes.c_uint32()
        check(lib().zk_index_cache_section(self._h, tag, ctypes.byref(p), ctypes.byref(n), ctypes.byref(d)))
        return p.value or 0, n.value, d.value

    def _release(self, h):
        lib().zk_index_cache_free(h)


class OpeningProof:
    """poly_commitment::ipa::OpeningProof (ipa.rs:1175-1191): lr [rounds, 2, 8], delta [8], z1 [4], z2 [4], sg [8] — points affine,
    everything in Montgomery limbs"""

    def __init__(self, lr, delta, z1, z2, sg):
        self.lr, self.delta, self.z1, self.z2, self.sg = lr, delta, z1, z2, sg


class _Transcript:
    """The caller's transcript callables u_base(cip [4]) -> U [8], round_challenge(i, l [8], r [8]) -> u [4] and
    final_challenge(delta [8]) -> c [4] as a zk_open_transcript (`struct`).  An exception never unwinds through the C frames: the
    first one is kept, the callback returns 1 so that the library fails the call, and reraise() raises it once the call is back."""

    def __init__(self, u_base, round_challenge, final_challenge):
        self.error = None
        self.callbacks = (U_BASE_CB(self.guard(lambda cip, out: _put(out, u_base(_view(cip, 4)), 8))),
                          ROUND_CB(self.guard(lambda i, l, r, out: _put(out, round_challenge(int(i), _view(l, 8), _view(r, 8)), 4))),
                          FINAL_CB(self.guard(lambda d, out: _put(out, final_challenge(_view(d, 8)), 4))))
        self.struct = OpenTranscript(None, *self.callbacks)

    def guard(self, fn):
        def wrapped(user, *args):
            try:
                fn(*args)
                return 0
            except Exception as e:
                if self.error is None:
                    self.error = e
                return 1
        return wrapped

    def reraise(self):
        if self.error is not None:
            raise self.error


def _view(p, n):
    return np.ctypeslib.as_array(p, shape=(n,)).copy()


def _put(p, v, n):
    np.ctypeslib.as_array(p, shape=(n,))[:] = np.ascontiguousarray(v, dtype=np.uint64).reshape(n)


def srs_open(srs, plnms, elm, polyscale, evalscale, rng_scalars, u_base, round_challenge, final_challenge) -> OpeningProof:
    """SRS::open (ipa.rs:823-1061) through zk_srs_open.
    plnms: list of (data [len, 4] Montgomery numpy array OR (device_ptr, len), domain_size (0 = coefficients), blinders [k, 4]);
    elm [m, 4]; rng_scalars [2 * rounds + 2, 4] = rand_l, rand_r per round, then d, r_delta; the three callables are the caller's
    transcript: u_base(cip [4]) -> U [8]; round_challenge(i, l [8], r [8]) -> u [4]; final_challenge(delta [8]) -> c [4]."""
    keep, arr = [], (OpenPoly * max(1, len(plnms)))()
    for i, (data, dom, blinders) in enumerate(plnms):
        if isinstance(data, tuple):
            ptr, ln = data
        else:
            d = _np_u64(data, (4,))
            keep.append(d)
            ptr, ln = d.ctypes.data, d.shape[0]
        bl = _np_u64(blinders, (4,))
        keep.append(bl)
        arr[i] = OpenPoly(ptr, ln, dom, bl.ctypes.data, bl.shape[0])
    elm = _np_u64(elm, (4,))
    rng = _np_u64(rng_scalars, (4,))
    ps, es = _fe(polyscale), _fe(evalscale)
    tr = _Transcript(u_base, round_challenge, final_challenge)
    rounds_cap = 64
    lr = np.zeros((rounds_cap, 2, 8), dtype=np.uint64)
    delta, sg = np.zeros(8, dtype=np.uint64), np.zeros(8, dtype=np.uint64)
    z1, z2 = np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.uint64)
    rounds = ctypes.c_size_t(0)
    rc = lib().zk_srs_open(srs._h, arr, len(plnms), _ptr(elm), elm.shape[0], _ptr(ps), _ptr(es), _ptr(rng), rng.shape[0], ctypes.byref(tr.struct),
                           _ptr(lr), rounds_cap, ctypes.byref(rounds), _ptr(delta), _ptr(z1), _ptr(z2), _ptr(sg))
    tr.reraise()
    check(rc)
    return OpeningProof(lr[: rounds.value].copy(), delta, z1, z2, sg)


@dataclass
class BatchEvaluationProof:
    """One element of the batch of SRS::verify (commitment.rs:682-700): the opening, its evaluation points and scales, the commitments
    of `evaluations` (each uint64 [chunks, 8]; zero chunks = an empty PolyComm), the combined inner product, and the proof's own
    transcript — the same three callables as srs_open: u_base(cip [4]) -> U [8]; round_challenge(i, l [8], r [8]) -> u [4];
    final_challenge(delta [8]) -> c [4].  Everything in Montgomery limbs."""
    opening: OpeningProof
    elm: np.ndarray
    polyscale: np.ndarray
    evalscale: np.ndarray
    commitments: list
    combined_inner_product: np.ndarray
    u_base: object
    round_challenge: object
    final_challenge: object


def srs_verify(srs, batch, rand_base, sg_rand_base, return_sum: bool = False):
    """SRS::verify (ipa.rs:301-502) through zk_srs_verify: True iff the batch of BatchEvaluationProof verifies.  rand_base and
    sg_rand_base are the two scalars the reference draws from its rng (Montgomery [4]).  With return_sum, also the affine point [8]
    the reference compares with zero.  An exception raised by a callback aborts the call and is re-raised here."""
    keep, transcripts = [], []

    def arr(a, tail):
        a = _np_u64(a, tail) if np.size(a) else np.zeros((0,) + tail, dtype=np.uint64)
        keep.append(a)
        return a

    descs = (VerifyProof * max(1, len(batch)))()
    for i, e in enumerate(batch):
        op = e.opening
        lr = arr(op.lr, (2, 8))
        delta, sg, z1, z2 = arr(op.delta, (8,)), arr(op.sg, (8,)), arr(op.z1, (4,)), arr(op.z2, (4,))
        elm, ps, es, cip = arr(e.elm, (4,)), arr(e.polyscale, (4,)), arr(e.evalscale, (4,)), arr(e.combined_inner_product, (4,))
        comms = [arr(c, (8,)) for c in e.commitments]
        cxy = arr(np.concatenate(comms) if comms else np.zeros((0, 8), dtype=np.uint64), (8,))
        chunks = (ctypes.c_size_t * max(1, len(comms)))(*[c.shape[0] for c in comms])
        tr = _Transcript(e.u_base, e.round_challenge, e.final_challenge)
        transcripts.append(tr)
        keep.append(chunks)
        p = lambda a: a.ctypes.data if a.size else None
        descs[i] = VerifyProof(p(lr), lr.shape[0], p(delta), p(z1), p(z2), p(sg), p(elm), elm.shape[0], p(ps), p(es), p(cxy), chunks,
                               len(comms), p(cip), ctypes.pointer(tr.struct))
    rng = np.concatenate([_fe(rand_base), _fe(sg_rand_base)])
    ok = ctypes.c_int(0)
    out = np.zeros(12, dtype=np.uint64)
    rc = lib().zk_srs_verify(srs._h, descs, len(batch), _ptr(rng), ctypes.byref(ok), _ptr(out))
    for tr in transcripts:
        tr.reraise()
    check(rc)
    if not return_sum:
        return bool(ok.value)
    return bool(ok.value), jacobian_to_affine(srs.curve, out)


# the scalar fields' moduli (curves/src/pasta/fields/fp.rs, fq.rs)
_MODULUS = {FP: 0x40000000000000000000000000000000224698fc094cf91b992d30ed00000001,
            FQ: 0x40000000000000000000000000000000224698fc0994a8dd8c46eb2100000001}


def _os_scalar(field: int) -> np.ndarray:
    """F::rand(&mut OsRng): uniform below the modulus by rejection, from the OS's randomness.  Montgomery limbs [4]: the Montgomery
    form of a uniform element is itself uniform below the modulus."""
    m = _MODULUS[field]
    while True:
        x = int.from_bytes(os.urandom(32), "little") >> 1
        if x < m:
            return np.array([(x >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)


def _rows(a, tail):
    """a as contiguous uint64 [-1, *tail], also when empty"""
    return _np_u64(a, tail) if np.size(a) else np.zeros((0,) + tail, dtype=np.uint64)


def batch_dlog_accumulator_check(srs, comms, chals, r=None, return_sum: bool = False):
    """batch_dlog_accumulator_check (poly-commitment/src/utils.rs:212-273) through zk_srs_accumulator_check: True iff the k
    accumulators comms [k, 8] equal <b_poly_coefficients(chals_i), g> for the first k chunks of `rounds = len(chals) / k`
    challenges (chals [n, 4], Montgomery).  r: the scalar the reference draws from OsRng (Montgomery [4]); None draws one from the
    OS's randomness.  With return_sum, also the affine point [8] the check compares with zero.  Where the reference panics the
    library refuses, raised as ZkError."""
    c, ch = _rows(comms, (8,)), _rows(chals, (4,))
    rr = _os_scalar(SCALAR_FIELD[srs.curve]) if r is None else _fe(r)
    ok = ctypes.c_int(0)
    out = np.zeros(12, dtype=np.uint64)
    check(lib().zk_srs_accumulator_check(srs._h, _ptr(c) if c.size else None, c.shape[0], _ptr(ch) if ch.size else None, ch.shape[0],
                                         _ptr(rr), ctypes.byref(ok), _ptr(out)))
    if not return_sum:
        return bool(ok.value)
    return bool(ok.value), jacobian_to_affine(srs.curve, out)


def batch_dlog_accumulator_generate(srs, num_comms: int, chals) -> np.ndarray:
    """batch_dlog_accumulator_generate (poly-commitment/src/utils.rs:275-312) through zk_srs_accumulator_generate: one accumulator
    <b_poly_coefficients(chunk), g> per chunk of `rounds = len(chals) / num_comms` challenges (chals [n, 4], Montgomery), as uint64
    [n / rounds, 8] affine.  Where the reference panics the library refuses, raised as ZkError."""
    ch = _rows(chals, (4,))
    n = ch.shape[0]
    cap = n // (n // num_comms) if num_comms and n >= num_comms else 0
    out = np.zeros((max(cap, 1), 8), dtype=np.uint64)
    got = ctypes.c_size_t(0)
    check(lib().zk_srs_accumulator_generate(srs._h, num_comms, _ptr(ch) if ch.size else None, n, _ptr(out), cap, ctypes.byref(got)))
    return out[: got.value]


class IpaRounds(Handle):
    """The folding loop of SRS::open (poly-commitment/src/ipa.rs:929-1007) with a and b resident on the device and the bases
    taken from the resident SRS table (`bases` = ctx.upload_bases(curve, srs.g)); see csrc/ipa.cu.

    The caller owns the sponge: per round it takes `lr()` -> (<a_hi,g_lo>, <a_lo,g_hi>, <a_hi,b_lo>, <a_lo,b_hi>), finishes
    L and R with its blinders (rand_l * h + <a_hi,b_lo> * u_base, ipa.rs:943-961), absorbs them, squeezes u and calls
    `fold(u, u_inv)`.  After log2(n) rounds `state()` is (a0, b0) and `sg()` the folded base g0."""

    def __init__(self, ctx: Context, bases, a_mont, b_mont):
        a, b = _np_u64(a_mont, (4,)), _np_u64(b_mont, (4,))
        n = 1 << max(1, (len(bases) - 1).bit_length())          # ipa.rs:848-850: padded_length
        if a.shape[0] > n or b.shape[0] > n:
            raise ValueError("a and b must not be longer than the padded SRS")
        pad = lambda v: np.concatenate([v, np.zeros((n - v.shape[0], 4), dtype=np.uint64)]) if v.shape[0] < n else v
        a, b = pad(a), pad(b)                                    # ipa.rs:858-862: a padded with zeros
        self.ctx, self.curve, self.bases = ctx, bases.curve, bases
        self._h = ctypes.c_void_p()
        check(lib().zk_ipa_begin(ctx._h, bases._h, _ptr(a), _ptr(b), n, ctypes.byref(self._h)))

    def __len__(self):
        return int(lib().zk_ipa_len(self._h))

    def lr(self):
        l, r = np.zeros(12, dtype=np.uint64), np.zeros(12, dtype=np.uint64)
        ipl, ipr = np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.uint64)
        check(lib().zk_ipa_round_lr(self._h, l.ctypes.data_as(_u64p), r.ctypes.data_as(_u64p), ipl.ctypes.data_as(_u64p), ipr.ctypes.data_as(_u64p)))
        return l, r, ipl, ipr

    def fold(self, u_mont, u_inv_mont):
        u, ui = _fe(u_mont), _fe(u_inv_mont)
        check(lib().zk_ipa_round_fold(self._h, u.ctypes.data_as(_u64p), ui.ctypes.data_as(_u64p)))

    def state(self):
        n = len(self)
        a, b = np.zeros((n, 4), dtype=np.uint64), np.zeros((n, 4), dtype=np.uint64)
        check(lib().zk_ipa_read(self._h, _ptr(a), _ptr(b), n, None))
        return a, b

    def sg(self) -> np.ndarray:
        """g0 after the last fold, Jacobian [12]"""
        out = np.zeros(12, dtype=np.uint64)
        check(lib().zk_ipa_read(self._h, None, None, 0, out.ctypes.data_as(_u64p)))
        return out

    def _release(self, h):
        lib().zk_ipa_free(h)


class ExprProgram:
    """Builder of the RPN programs zk_expr_eval_dev runs — kimchi's `PolishToken` list (kimchi/src/circuits/expr.rs:819-836) with the
    Challenge / Constant terms already literal.  Methods are the reference's token names; `evaluations` is Expr::evaluations
    (expr.rs:1938-1990) on the device.  Opcode numbers are include/zkb200.h's ZK_EXPR_*."""
    CONST, CELL, DUP, POW, ADD, MUL, SUB, STORE, LOAD = range(9)

    def __init__(self):
        self.tokens: list[tuple[int, int]] = []
        self.constants: list[np.ndarray] = []
        self.n_cached = 0

    def literal(self, x_mont):
        self.constants.append(_fe(x_mont))
        self.tokens.append((self.CONST, len(self.constants) - 1)); return self

    def cell(self, col: int, next_row: bool = False):
        self.tokens.append((self.CELL, col | (0x80000000 if next_row else 0))); return self

    def dup(self): self.tokens.append((self.DUP, 0)); return self
    def pow(self, n: int): self.tokens.append((self.POW, n)); return self
    def add(self): self.tokens.append((self.ADD, 0)); return self
    def mul(self): self.tokens.append((self.MUL, 0)); return self
    def sub(self): self.tokens.append((self.SUB, 0)); return self

    def store(self) -> int:
        """Store: the top of the stack also goes to the next cache slot; returns the slot for load()"""
        self.tokens.append((self.STORE, 0)); self.n_cached += 1; return self.n_cached - 1

    def load(self, slot: int): self.tokens.append((self.LOAD, slot)); return self

    def evaluations(self, ctx: Context, field: int, cols, out_len: int, out_domain_mult: int, d_out: int, accumulate: bool = False):
        """cols: [(device pointer, len, domain_mult)] in the order the program's cell() indices refer to"""
        ctx.expr_eval_dev(field, self.tokens, np.array(self.constants, dtype=np.uint64).reshape(-1, 4), cols, out_len, out_domain_mult, d_out, accumulate)


_MONT_ONE = {FP: (0x34786d38fffffffd, 0x992c350be41914ad, 0xffffffffffffffff, 0x3fffffffffffffff),    # R mod p (host_field.hpp)
             FQ: (0x5b2b3e9cfffffffd, 0x992c350be3420567, 0xffffffffffffffff, 0x3fffffffffffffff)}


class LookupSpec:
    """kimchi's LookupInfo lowered for zk_lookup_sorted_dev / zk_lookup_aggreg_dev: patterns of joint lookups (JointLookupSpec,
    kimchi/src/circuits/lookup/lookups.rs:312-409) and, per call, each row's pattern (LookupInfo::by_row, :286-299).

    A joint lookup is (table_id, entries): table_id an int (LookupTableID::Constant) or ("witness", column) (WitnessColumn, read at
    the current row); entries up to 4 linear combinations (SingleLookup), each a list of terms (coeff, column, next_row) with coeff
    Montgomery limbs [4] or None for one."""
    XOR_TABLE_ID, RANGE_CHECK_TABLE_ID = 0, 1          # kimchi/src/circuits/lookup/tables/mod.rs:15-18
    KIMCHI_PATTERNS = ("xor", "lookup", "range_check", "foreign_field_mul")

    def __init__(self, field: int, max_per_row: int):
        self.field, self.max_per_row = field, max_per_row
        self.terms: list[tuple] = []
        self.lookups: list[tuple] = []
        self.patterns: list[tuple[int, int]] = []

    @classmethod
    def kimchi_lookups(cls, pattern: str) -> list:
        """LookupPattern::lookups() (lookups.rs:448-528) of "xor", "lookup", "range_check" or "foreign_field_mul".  ForeignFieldMul
        applies to its gate's row and the next one; that is the row mapping's business (by_row), not the pattern's."""
        one = lambda col: [(None, col, False)]
        if pattern == "xor":
            return [(cls.XOR_TABLE_ID, [one(3 + i), one(7 + i), one(11 + i)]) for i in range(4)]
        if pattern == "lookup":
            return [(("witness", 0), [one(2 * i + 1), one(2 * i + 2)]) for i in range(3)]
        if pattern == "range_check":
            return [(cls.RANGE_CHECK_TABLE_ID, [one(c)]) for c in range(3, 7)]
        if pattern == "foreign_field_mul":
            return [(cls.RANGE_CHECK_TABLE_ID, [one(c)]) for c in range(7, 11)]
        raise ValueError(f"unknown lookup pattern {pattern!r}")

    def add_pattern(self, lookups) -> int:
        """Appends a pattern (a list of joint lookups); returns its index p — rows using it carry p + 1 in row_pattern"""
        first = len(self.lookups)
        for table_id, entries in lookups:
            first_term = len(self.terms)
            counts = []
            for entry in entries:
                for coeff, col, nxt in entry:
                    self.terms.append((_MONT_ONE[self.field] if coeff is None else tuple(int(x) for x in np.asarray(coeff, dtype=np.uint64).reshape(4)),
                                       int(col), int(bool(nxt))))
                counts.append(len(entry))
            tid, tcol = (0, int(table_id[1])) if isinstance(table_id, tuple) else (int(table_id), -1)
            self.lookups.append((tid, tcol, counts, first_term))
        self.patterns.append((first, len(lookups)))
        return len(self.patterns) - 1

    def add_kimchi_pattern(self, pattern: str) -> int:
        return self.add_pattern(self.kimchi_lookups(pattern))

    def info(self, row_pattern, joint_combiner, table_id_combiner, dummy) -> "LookupInfo":
        """The zk_lookup_info of these patterns for rows row_pattern (uint8 [lookup_rows]: 0 none, p + 1 pattern p); scalars Montgomery"""
        terms = (LookupTerm * max(1, len(self.terms)))()
        for k, (c, col, nxt) in enumerate(self.terms):
            terms[k].coeff[:] = list(c)
            terms[k].column, terms[k].next = col, nxt
        joints = (LookupJoint * max(1, len(self.lookups)))()
        for k, (tid, tcol, counts, first_term) in enumerate(self.lookups):
            joints[k].table_id, joints[k].table_id_column, joints[k].first_term = tid, tcol, first_term
            joints[k].n_entries = len(counts)                    # more than 4: the library refuses the call
            for e, cnt in enumerate(counts[:4]):
                joints[k].entry_terms[e] = cnt
        first = (ctypes.c_uint32 * max(1, len(self.patterns)))(*[p[0] for p in self.patterns])
        count = (ctypes.c_uint32 * max(1, len(self.patterns)))(*[p[1] for p in self.patterns])
        rows = np.ascontiguousarray(row_pattern, dtype=np.uint8)
        s = LookupInfo()
        s.terms, s.n_terms = ctypes.cast(terms, ctypes.POINTER(LookupTerm)), len(self.terms)
        s.lookups, s.n_lookups = ctypes.cast(joints, ctypes.POINTER(LookupJoint)), len(self.lookups)
        s.pattern_first, s.pattern_count, s.n_patterns = ctypes.cast(first, ctypes.POINTER(ctypes.c_uint32)), ctypes.cast(count, ctypes.POINTER(ctypes.c_uint32)), len(self.patterns)
        s.row_pattern = rows.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8))
        s.max_per_row = self.max_per_row
        for name, v in (("joint_combiner", joint_combiner), ("table_id_combiner", table_id_combiner), ("dummy", dummy)):
            getattr(s, name)[:] = [int(x) for x in np.asarray(v, dtype=np.uint64).reshape(4)]
        s._keep = (terms, joints, first, count, rows)          # the arrays the structure points into
        return s


class LagrangeBasisEvaluations(Handle):
    """kimchi::lagrange_basis_evaluations::LagrangeBasisEvaluations (lagrange_basis_evaluations.rs:24-258) resident on the device: the
    chunks x n basis values at x live in a device buffer this object owns (close() frees it).  Columns are (device pointer, len) pairs
    of Montgomery evaluations whose length is a multiple of domain_size()."""

    def __init__(self, ctx: Context, field: int, max_poly_size: int, log_n: int, x):
        self.ctx, self.field, self.log_n = ctx, field, log_n
        self.chunks = Context.lagrange_evals_chunks(1 << log_n, max_poly_size)
        self._h = ctx.buffers()
        self.ptr = self._h.alloc(max(1, self.chunks) << (log_n + 5))
        try:
            ctx.lagrange_basis_evals_dev(field, log_n, max_poly_size, x, self.ptr)
        except Exception:
            self.close()
            raise

    # pub fn new(max_poly_size: usize, domain: D<F>, x: F) -> LagrangeBasisEvaluations<F>
    @classmethod
    def new(cls, ctx: Context, field: int, max_poly_size: int, log_n: int, x) -> "LagrangeBasisEvaluations":
        return cls(ctx, field, max_poly_size, log_n, x)

    def domain_size(self) -> int:
        return 1 << self.log_n

    # pub fn evaluate<D: EvaluationDomain<F>>(&self, p: &Evaluations<F, D>) -> Vec<F>
    def evaluate(self, column) -> np.ndarray:
        """[chunks, 4]: chunk k is sum_i p[stride i] l_k[i]"""
        return self.ctx.lagrange_evaluate_dev(self.field, [self.ptr], self.log_n, self.chunks, [(column[0], column[1], False)])[0, 0]

    # pub fn evaluate_boolean<D: EvaluationDomain<F>>(&self, p: &Evaluations<F, D>) -> Vec<F>
    def evaluate_boolean(self, column) -> np.ndarray:
        """[chunks, 4]: chunk k is the sum of l_k[i] over every i with p[stride i] != 0"""
        return self.ctx.lagrange_evaluate_dev(self.field, [self.ptr], self.log_n, self.chunks, [(column[0], column[1], True)])[0, 0]

    @staticmethod
    def evaluate_all(points, columns) -> np.ndarray:
        """evaluate / evaluate_boolean of every column at every point in one call: points = LagrangeBasisEvaluations of one domain,
        columns = [(device pointer, len, boolean)] -> [n_cols, n_points, chunks, 4]"""
        p0 = points[0]
        if any(p.log_n != p0.log_n or p.chunks != p0.chunks or p.field != p0.field for p in points):
            raise ValueError("the bases must share field, domain and chunk count")
        return p0.ctx.lagrange_evaluate_dev(p0.field, [p.ptr for p in points], p0.log_n, p0.chunks, columns)

    def evals(self) -> np.ndarray:
        """the basis values [chunks, n, 4] (downloaded)"""
        return self.ctx.dev_download(self.ptr, (self.chunks, self.domain_size(), 4))

    def _release(self, bufs):
        bufs.close()


class Radix2EvaluationDomain:
    """ark_poly::Radix2EvaluationDomain::<F>::new(size) on the device.  `field` is ZK_FP or ZK_FQ."""

    def __init__(self, ctx: Context, field: int, size: int):
        if size <= 0:
            raise ValueError("domain size must be positive")
        log_n = (size - 1).bit_length()  # new(n) rounds up to the next power of two
        self.ctx, self.field, self.log_size_of_group, self.size = ctx, field, log_n, 1 << log_n

    def _run(self, a, inverse, coset):
        a = _np_u64(a, (4,))
        if a.shape[0] > self.size:
            raise ValueError("more coefficients than the domain size")  # ark reduces mod X^n - 1; callers on the path never do
        buf = np.zeros((self.size, 4), dtype=np.uint64)
        buf[: a.shape[0]] = a
        return self.ctx.ntt(self.field, buf, inverse=inverse, coset=coset, in_len=a.shape[0] if not inverse else 0)

    def fft(self, coeffs) -> np.ndarray:
        return self._run(coeffs, False, False)

    def ifft(self, evals) -> np.ndarray:
        return self._run(evals, True, False)

    def coset_fft(self, coeffs) -> np.ndarray:
        return self._run(coeffs, False, True)

    def coset_ifft(self, evals) -> np.ndarray:
        return self._run(evals, True, True)
