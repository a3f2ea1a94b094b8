"""ctypes bindings of libzkb200.so (include/zkb200.h).  No fallback: a missing library is an ImportError."""
from __future__ import annotations

import ctypes
import os

import numpy as np

FP, FQ = 0, 1
PALLAS, VESTA = 0, 1
BASE_FIELD = {PALLAS: FP, VESTA: FQ}
SCALAR_FIELD = {PALLAS: FQ, VESTA: FP}
CUDA_STREAM_LEGACY = 0x1             # cudaStreamLegacy (cuda_runtime_api.h)

_HERE = os.path.dirname(os.path.abspath(__file__))
# ZKB200_LIB: an alternative BUILD of the same CUDA library (tools/mul_variants.sh times the field-product variants
# libzkb200_k<K>.so against the shipped one); never a different implementation — there is no CPU fallback to select.
_SO = os.environ.get("ZKB200_LIB") or os.path.join(_HERE, "libzkb200.so")


def library_path() -> str:
    return _SO


class ZkError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"zkb200 error {code}: {msg}")
        self.code = code


_lib = None
_u64p = ctypes.POINTER(ctypes.c_uint64)


def lib() -> ctypes.CDLL:
    """Load the CUDA library.  Raises ImportError if it was not built (python __graft_entry__.py / make -C csrc)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_SO):
        raise ImportError(
            f"{_SO} is missing: build the CUDA extension first (python -c 'import __graft_entry__ as g; g.build()'). "
            "proof_systems_b200 has no CPU fallback.")
    L = ctypes.CDLL(_SO)
    vp, sz, i, u = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_uint
    L.zk_last_error.restype = ctypes.c_char_p
    L.zk_device_count.restype = i
    L.zk_ctx_create.argtypes = [i, ctypes.POINTER(vp)]
    L.zk_ctx_destroy.argtypes = [vp]
    L.zk_ctx_destroy.restype = None
    L.zk_ctx_set_stream.argtypes = [vp, vp]
    L.zk_ctx_launch_count.argtypes = [vp]
    L.zk_ctx_launch_count.restype = ctypes.c_uint64
    L.zk_ctx_set_profile.argtypes = [vp, i]
    L.zk_ctx_set_option.argtypes = [vp, ctypes.c_char_p, ctypes.c_long]
    L.zk_ctx_last_stage_ms.argtypes = [vp, ctypes.POINTER(ctypes.c_float), sz]
    L.zk_bases_upload.argtypes = [vp, i, vp, sz, i, i, ctypes.POINTER(vp)]
    L.zk_bases_free.argtypes = [vp]
    L.zk_bases_free.restype = None
    L.zk_bases_len.argtypes = [vp]
    L.zk_bases_len.restype = sz
    L.zk_bases_window_bits.argtypes = [vp]
    L.zk_points_decompress.argtypes = [vp, i, vp, sz, _u64p]
    L.zk_points_from_uncompressed.argtypes = [vp, i, vp, sz, _u64p]
    L.zk_points_compress.argtypes = [vp, i, vp, sz, vp]
    L.zk_msm.argtypes = [vp, vp, sz, sz, vp, i, i, _u64p]
    L.zk_msm_dev.argtypes = [vp, vp, sz, sz, vp, i, i, _u64p]
    L.zk_msm_batch.argtypes = [vp, vp, sz, sz, vp, sz, i, i, _u64p]
    L.zk_msm_partial.argtypes = [vp, vp, sz, sz, vp, i, i, vp, sz, ctypes.POINTER(u), ctypes.POINTER(u)]
    L.zk_msm_finish_gathered.argtypes = [vp, i, vp, sz, u, u, _u64p]
    L.zk_jacobian_to_affine.argtypes = [i, _u64p, _u64p]
    L.zk_jacobian_add.argtypes = [i, _u64p, _u64p, _u64p]
    L.zk_jacobian_sum.argtypes = [i, _u64p, sz, _u64p]
    L.zk_ntt.argtypes = [vp, i, vp, u, i, i]
    L.zk_ntt_batch.argtypes = [vp, i, vp, u, sz, sz, i, i]
    L.zk_ntt_dev.argtypes = [vp, i, vp, u, sz, sz, i, i]
    L.zk_srs_create.argtypes = [vp, i, vp, sz, _u64p, i, ctypes.POINTER(vp)]
    L.zk_srs_destroy.argtypes = [vp]
    L.zk_srs_destroy.restype = None
    L.zk_srs_max_poly_size.argtypes = [vp]
    L.zk_srs_max_poly_size.restype = sz
    L.zk_srs_add_lagrange_basis.argtypes = [vp, sz, vp, i]
    L.zk_srs_lagrange_basis.argtypes = [vp, sz, i]
    L.zk_srs_get_lagrange_basis.argtypes = [vp, sz, _u64p, sz]
    L.zk_srs_lagrange_basis_chunks.argtypes = [vp, sz]
    L.zk_srs_lagrange_basis_chunks.restype = sz
    L.zk_srs_commit_non_hiding.argtypes = [vp, vp, sz, sz, _u64p, sz, ctypes.POINTER(sz)]
    L.zk_srs_commit_evaluations_non_hiding.argtypes = [vp, sz, vp, sz, _u64p]
    L.zk_srs_commit_evaluations_batch.argtypes = [vp, sz, vp, sz, _u64p]
    L.zk_srs_mask_custom.argtypes = [vp, vp, sz, vp, sz, _u64p]
    L.zk_ipa_begin.argtypes = [vp, vp, vp, vp, sz, ctypes.POINTER(vp)]
    L.zk_ipa_free.argtypes = [vp]
    L.zk_ipa_free.restype = None
    L.zk_ipa_len.argtypes = [vp]
    L.zk_ipa_len.restype = sz
    L.zk_ipa_round_lr.argtypes = [vp, _u64p, _u64p, _u64p, _u64p]
    L.zk_ipa_round_fold.argtypes = [vp, _u64p, _u64p]
    L.zk_ipa_read.argtypes = [vp, vp, vp, sz, _u64p]
    L.zk_debug_field_op.argtypes = [vp, i, i, vp, vp, vp, sz]
    L.zk_debug_mul_throughput.argtypes = [vp, i, u, ctypes.POINTER(ctypes.c_double)]
    L.zk_debug_op_throughput.argtypes = [vp, i, i, u, u, u, ctypes.POINTER(ctypes.c_double)]
    _lib = L
    if os.environ.get("ZKB200_LIB") and not hasattr(L, "zk_points_synthetic"):
        return L      # an A/B build of an older tree (tools/build_variants.sh): the newest entry points are absent
    L.zk_points_synthetic.argtypes = [vp, i, ctypes.c_uint64, sz, vp]
    L.zk_ntt_dev_oop.argtypes = [vp, i, vp, sz, sz, vp, u, sz, i, i]
    L.zk_dev_alloc.argtypes = [vp, sz, ctypes.POINTER(vp)]
    L.zk_dev_free.argtypes = [vp, vp]
    L.zk_dev_upload.argtypes = [vp, vp, vp, sz]
    L.zk_dev_download.argtypes = [vp, vp, vp, sz]
    L.zk_perm_quotient_dev.argtypes = [vp, i, u, vp, vp, vp, vp, vp, vp, vp, vp, u, vp]
    L.zk_points_fold_dev.argtypes = [vp, i, vp, sz, vp, vp]
    L.zk_poly_add_dev.argtypes = [vp, i, vp, vp, sz]
    L.zk_poly_divide_by_vanishing_dev.argtypes = [vp, i, vp, sz, u, vp, ctypes.POINTER(ctypes.c_int)]
    L.zk_expr_eval_dev.argtypes = [vp, i, vp, sz, vp, sz, vp, sz, ctypes.c_uint64, u, i, vp]
    L.zk_index_cache_load.argtypes = [vp, vp, sz, ctypes.c_char_p, ctypes.POINTER(vp)]
    L.zk_index_cache_free.argtypes = [vp]
    L.zk_index_cache_free.restype = None
    L.zk_index_cache_header.argtypes = [vp, ctypes.POINTER(IndexHeader)]
    L.zk_index_cache_section.argtypes = [vp, ctypes.c_uint32, ctypes.POINTER(vp), ctypes.POINTER(sz), ctypes.POINTER(ctypes.c_uint32)]
    L.zk_index_build.argtypes = [vp, i, ctypes.POINTER(IndexHeader), vp, sz, vp, sz, i, ctypes.POINTER(vp)]
    L.zk_index_commitments.argtypes = [vp, vp, _u64p, sz, ctypes.POINTER(sz)]
    L.zk_comm_unique_id.argtypes = [vp]
    L.zk_comm_init_rank.argtypes = [vp, vp, i, i, ctypes.POINTER(vp)]
    L.zk_comm_destroy.argtypes = [vp]
    L.zk_comm_destroy.restype = None
    L.zk_msm_sharded.argtypes = [vp, vp, sz, sz, vp, i, i, vp]
    L.zk_srs_open.argtypes = [vp, ctypes.POINTER(OpenPoly), sz, vp, sz, vp, vp, vp, sz, ctypes.POINTER(OpenTranscript), vp, sz,
                              ctypes.POINTER(sz), vp, vp, vp, vp]
    L.zk_srs_verify.argtypes = [vp, ctypes.POINTER(VerifyProof), sz, vp, ctypes.POINTER(i), vp]
    L.zk_lagrange_evals_chunks.argtypes = [sz, sz]
    L.zk_lagrange_evals_chunks.restype = sz
    L.zk_lagrange_evals_dev.argtypes = [vp, i, u, sz, vp, vp]
    L.zk_lagrange_evaluate_dev.argtypes = [vp, i, ctypes.POINTER(vp), sz, u, sz, ctypes.POINTER(EvalColumn), sz, vp]
    L.zk_poly_evaluate_chunks_dev.argtypes = [vp, i, ctypes.POINTER(DevPoly), sz, sz, sz, vp, sz, vp]
    L.zk_prover_ft_dev.argtypes = [vp, i, u, sz, ctypes.POINTER(LinTerm), sz, vp, sz, vp, vp, ctypes.POINTER(sz), vp]
    L.zk_perm_aggreg_dev.argtypes = [vp, i, u, sz, ctypes.POINTER(vp), ctypes.POINTER(vp), ctypes.c_uint64, vp, vp, vp, vp, vp, ctypes.POINTER(i)]
    L.zk_lookup_joint_table_dev.argtypes = [vp, i, u, ctypes.POINTER(vp), sz, vp, vp, vp, vp, vp, vp]
    L.zk_lookup_sorted_dev.argtypes = [vp, i, u, sz, ctypes.POINTER(vp), vp, u, ctypes.POINTER(LookupInfo), vp, ctypes.POINTER(vp),
                                       ctypes.POINTER(ctypes.c_int64)]
    L.zk_lookup_aggreg_dev.argtypes = [vp, i, u, sz, ctypes.POINTER(vp), vp, u, ctypes.POINTER(LookupInfo), ctypes.POINTER(vp), vp, vp, vp, vp,
                                       ctypes.POINTER(i)]
    return L


class IndexHeader(ctypes.Structure):
    """zk_index_header (include/zkb200.h)"""
    _fields_ = [("public_inputs", ctypes.c_uint32), ("prev_challenges", ctypes.c_uint32), ("zk_rows", ctypes.c_uint64), ("max_poly_size", ctypes.c_uint64),
                ("domain_d1_size", ctypes.c_uint64), ("feature_flags", ctypes.c_uint32), ("optional_selectors_present", ctypes.c_uint32),
                ("lookup_selectors_present", ctypes.c_uint32), ("num_sections", ctypes.c_uint32), ("disable_gates_checks", ctypes.c_int),
                ("has_verifier_index_digest", ctypes.c_int), ("endo", ctypes.c_uint64 * 4), ("shift", (ctypes.c_uint64 * 4) * 7),
                ("verifier_index_digest", ctypes.c_uint64 * 4), ("identifier", ctypes.c_char * 512)]


class ExprToken(ctypes.Structure):
    """zk_expr_token (include/zkb200.h)"""
    _fields_ = [("op", ctypes.c_uint32), ("arg", ctypes.c_uint32)]


class ExprColumn(ctypes.Structure):
    """zk_expr_column (include/zkb200.h)"""
    _fields_ = [("d_evals", ctypes.c_void_p), ("len", ctypes.c_uint64), ("domain_mult", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


class EvalColumn(ctypes.Structure):
    """zk_eval_column (include/zkb200.h)"""
    _fields_ = [("d_evals", ctypes.c_void_p), ("len", ctypes.c_uint64), ("boolean", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


class DevPoly(ctypes.Structure):
    """zk_dev_poly (include/zkb200.h)"""
    _fields_ = [("d_coeffs", ctypes.c_void_p), ("len", ctypes.c_uint64)]


class LinTerm(ctypes.Structure):
    """zk_lin_term (include/zkb200.h)"""
    _fields_ = [("d_evals", ctypes.c_void_p), ("len", ctypes.c_uint64), ("coeff", ctypes.c_uint64 * 4)]


class LookupTerm(ctypes.Structure):
    """zk_lookup_term (include/zkb200.h)"""
    _fields_ = [("coeff", ctypes.c_uint64 * 4), ("column", ctypes.c_uint32), ("next", ctypes.c_uint32)]


class LookupJoint(ctypes.Structure):
    """zk_lookup_joint (include/zkb200.h)"""
    _fields_ = [("table_id", ctypes.c_int32), ("table_id_column", ctypes.c_int32), ("n_entries", ctypes.c_uint32),
                ("entry_terms", ctypes.c_uint32 * 4), ("first_term", ctypes.c_uint32)]


class LookupInfo(ctypes.Structure):
    """zk_lookup_info (include/zkb200.h); host.LookupSpec builds one"""
    _fields_ = [("terms", ctypes.POINTER(LookupTerm)), ("n_terms", ctypes.c_size_t), ("lookups", ctypes.POINTER(LookupJoint)),
                ("n_lookups", ctypes.c_size_t), ("pattern_first", ctypes.POINTER(ctypes.c_uint32)), ("pattern_count", ctypes.POINTER(ctypes.c_uint32)),
                ("n_patterns", ctypes.c_size_t), ("row_pattern", ctypes.POINTER(ctypes.c_uint8)), ("max_per_row", ctypes.c_uint),
                ("joint_combiner", ctypes.c_uint64 * 4), ("table_id_combiner", ctypes.c_uint64 * 4), ("dummy", ctypes.c_uint64 * 4)]


class OpenPoly(ctypes.Structure):
    """zk_open_poly (include/zkb200.h)"""
    _fields_ = [("data", ctypes.c_void_p), ("len", ctypes.c_size_t), ("domain_size", ctypes.c_size_t),
                ("blinders", ctypes.c_void_p), ("n_blinders", ctypes.c_size_t)]


U_BASE_CB = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint64))
ROUND_CB = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_uint, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint64),
                            ctypes.POINTER(ctypes.c_uint64))
FINAL_CB = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint64))


class OpenTranscript(ctypes.Structure):
    """zk_open_transcript (include/zkb200.h)"""
    _fields_ = [("user", ctypes.c_void_p), ("u_base", U_BASE_CB), ("round", ROUND_CB), ("final_challenge", FINAL_CB)]


class VerifyProof(ctypes.Structure):
    """zk_verify_proof (include/zkb200.h)"""
    _fields_ = [("lr_xy", ctypes.c_void_p), ("n_rounds", ctypes.c_size_t), ("delta_xy", ctypes.c_void_p), ("z1", ctypes.c_void_p),
                ("z2", ctypes.c_void_p), ("sg_xy", ctypes.c_void_p), ("elm", ctypes.c_void_p), ("n_elm", ctypes.c_size_t),
                ("polyscale", ctypes.c_void_p), ("evalscale", ctypes.c_void_p), ("comm_xy", ctypes.c_void_p),
                ("comm_chunks", ctypes.POINTER(ctypes.c_size_t)), ("n_comms", ctypes.c_size_t), ("combined_inner_product", ctypes.c_void_p),
                ("transcript", ctypes.POINTER(OpenTranscript))]


def check(rc: int):
    if rc != 0:
        raise ZkError(rc, lib().zk_last_error().decode(errors="replace"))


def _np_u64(a, shape_tail):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    assert a.size % int(np.prod(shape_tail)) == 0
    return a.reshape((-1,) + tuple(shape_tail))


def _ptr(a: np.ndarray):
    return ctypes.c_void_p(a.ctypes.data)


def _out(n):
    return np.empty(n, dtype=np.uint64)


def jacobian_to_affine(curve: int, xyz) -> np.ndarray:
    """Projective::into_affine()"""
    xyz = np.ascontiguousarray(xyz, dtype=np.uint64)
    out = _out(8)
    check(lib().zk_jacobian_to_affine(curve, xyz.ctypes.data_as(_u64p), out.ctypes.data_as(_u64p)))
    return out


def jacobian_sum(curve: int, pts) -> np.ndarray:
    pts = _np_u64(pts, (12,))
    out = _out(12)
    check(lib().zk_jacobian_sum(curve, pts.ctypes.data_as(_u64p), pts.shape[0], out.ctypes.data_as(_u64p)))
    return out


class Context:
    """One CUDA device (one per process/rank)."""

    def __init__(self, device: int = 0):
        self._h = ctypes.c_void_p()
        check(lib().zk_ctx_create(device, ctypes.byref(self._h)))
        self.device = device

    def close(self):
        if getattr(self, "_h", None):
            lib().zk_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, cuda_stream: int | None):
        """None: the library's own stream.  An integer is a cudaStream_t handle, 0 included: 0 is the legacy default stream (torch's
        default stream reports 0 as its cuda_stream) and reaches the C ABI as cudaStreamLegacy, whose NULL means the own stream."""
        handle = None if cuda_stream is None else (int(cuda_stream) or CUDA_STREAM_LEGACY)
        check(lib().zk_ctx_set_stream(self._h, ctypes.c_void_p(handle)))

    @property
    def launch_count(self) -> int:
        return int(lib().zk_ctx_launch_count(self._h))

    def set_profile(self, enabled: bool):
        check(lib().zk_ctx_set_profile(self._h, int(enabled)))

    def set_option(self, name: str, value: int):
        check(lib().zk_ctx_set_option(self._h, name.encode(), value))

    def last_stage_ms(self) -> dict:
        buf = (ctypes.c_float * 8)()
        check(lib().zk_ctx_last_stage_ms(self._h, buf, 8))
        names = ["recode", "plan", "scatter", "accumulate", "finish", "bitsum", "ntt"]
        return {k: float(buf[i]) for i, k in enumerate(names)}

    def decompress_points(self, curve: int, raw33) -> np.ndarray:
        """ark-serialize compressed points (bytes or uint8 [n, 33], the srs/*.srs form) -> affine Montgomery [n, 8]"""
        buf = np.frombuffer(raw33, dtype=np.uint8) if isinstance(raw33, (bytes, bytearray)) else np.ascontiguousarray(raw33, dtype=np.uint8).reshape(-1)
        n = buf.size // 33
        out = np.empty((n, 8), dtype=np.uint64)
        check(lib().zk_points_decompress(self._h, curve, ctypes.c_void_p(buf.ctypes.data), n, out.ctypes.data_as(_u64p)))
        return out

    # ------------------------------------------------------------------ MSM
    def points_from_uncompressed(self, curve: int, raw65) -> np.ndarray:
        """uint8 [n, 65] ark uncompressed points (the srs/test_*.srs form) -> uint64 [n, 8] affine Montgomery"""
        raw = np.ascontiguousarray(raw65, dtype=np.uint8)
        if raw.ndim != 2 or raw.shape[1] != 65:
            raise ValueError("expected uint8 [n, 65]")
        out = np.zeros((raw.shape[0], 8), dtype=np.uint64)
        check(lib().zk_points_from_uncompressed(self._h, curve, _ptr(raw), raw.shape[0], out.ctypes.data_as(_u64p)))
        return out

    def compress_points(self, curve: int, points) -> np.ndarray:
        """uint64 [n, 8] affine Montgomery -> uint8 [n, 33] ark compressed points (what PolyComm / OpeningProof serialise to)"""
        pts = _np_u64(points, (8,))
        out = np.zeros((pts.shape[0], 33), dtype=np.uint8)
        check(lib().zk_points_compress(self._h, curve, _ptr(pts), pts.shape[0], _ptr(out)))
        return out

    def synthetic_points(self, curve: int, n: int, seed: int = 0) -> np.ndarray:
        """n deterministic on-curve points [n, 8] (zk_points_synthetic): inputs for workloads larger than the shipped SRS"""
        out = np.empty((n, 8), dtype=np.uint64)
        check(lib().zk_points_synthetic(self._h, curve, ctypes.c_uint64(seed), n, out.ctypes.data_as(_u64p)))
        return out

    def upload_bases(self, curve: int, points, window_bits: int = -1) -> "Bases":
        return Bases(self, curve, points, window_bits)

    def msm(self, bases: "Bases", scalars, off: int = 0, mont: bool = False, window_bits: int = 0) -> np.ndarray:
        """== G::Group::msm_bigint(&bases[off..off+n], scalars) (mont=False) / ::msm (mont=True).  Returns Jacobian [12]."""
        sc = _np_u64(scalars, (4,))
        out = _out(12)
        check(lib().zk_msm(self._h, bases._h, off, sc.shape[0], _ptr(sc), int(mont), window_bits, out.ctypes.data_as(_u64p)))
        return out

    def msm_dev(self, bases: "Bases", d_scalars: int, n: int, off: int = 0, mont: bool = False, window_bits: int = 0) -> np.ndarray:
        out = _out(12)
        check(lib().zk_msm_dev(self._h, bases._h, off, n, ctypes.c_void_p(d_scalars), int(mont), window_bits, out.ctypes.data_as(_u64p)))
        return out

    def msm_partial(self, bases: "Bases", scalars_ptr: int, n: int, d_out: int, capacity_points: int, off: int = 0, mont: bool = False,
                    window_bits: int = 0) -> tuple:
        """This rank's slice of a sharded MSM, left on the device (zk_msm_partial): returns (c, groups); nothing is synchronised."""
        c, g = ctypes.c_uint(), ctypes.c_uint()
        check(lib().zk_msm_partial(self._h, bases._h, off, n, ctypes.c_void_p(scalars_ptr), int(mont), window_bits, ctypes.c_void_p(d_out),
                                   capacity_points, ctypes.byref(c), ctypes.byref(g)))
        return c.value, g.value

    def msm_finish_gathered(self, curve: int, d_all: int, world: int, c: int, groups: int) -> np.ndarray:
        out = _out(12)
        check(lib().zk_msm_finish_gathered(self._h, curve, ctypes.c_void_p(d_all), world, c, groups, out.ctypes.data_as(_u64p)))
        return out

    def msm_batch(self, bases: "Bases", scalars, off: int = 0, mont: bool = False, window_bits: int = 0) -> np.ndarray:
        """scalars [k, n, 4] -> Jacobian [k, 12]"""
        sc = np.ascontiguousarray(scalars, dtype=np.uint64)
        assert sc.ndim == 3 and sc.shape[2] == 4
        k, n = sc.shape[0], sc.shape[1]
        out = np.empty((k, 12), dtype=np.uint64)
        check(lib().zk_msm_batch(self._h, bases._h, off, n, _ptr(sc), k, int(mont), window_bits, out.ctypes.data_as(_u64p)))
        return out

    def msm_affine(self, bases: "Bases", scalars, **kw) -> np.ndarray:
        return jacobian_to_affine(bases.curve, self.msm(bases, scalars, **kw))

    # ------------------------------------------------------------------ NTT
    def ntt(self, field: int, data, inverse: bool = False, coset: bool = False, in_len: int = 0) -> np.ndarray:
        """Transforms a copy.  data [n,4] or [batch,n,4] (Montgomery); n a power of two."""
        a = np.array(data, dtype=np.uint64, order="C", copy=True)
        assert a.shape[-1] == 4
        n = a.shape[-2]
        batch = 1 if a.ndim == 2 else a.shape[0]
        log_n = n.bit_length() - 1
        assert 1 << log_n == n
        check(lib().zk_ntt_batch(self._h, field, _ptr(a), log_n, batch, in_len, int(inverse), int(coset)))
        return a

    def ntt_inplace(self, field: int, a: np.ndarray, inverse: bool = False, coset: bool = False, in_len: int = 0):
        """In-place transform of a C-contiguous uint64 array [n,4] or [batch,n,4] (e.g. a view of pinned memory): no copy
        on the Python side, exactly the zk_ntt_batch call a Rust caller makes on its own Vec."""
        assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"] and a.shape[-1] == 4
        n = a.shape[-2]
        batch = 1 if a.ndim == 2 else a.shape[0]
        log_n = n.bit_length() - 1
        assert 1 << log_n == n
        check(lib().zk_ntt_batch(self._h, field, _ptr(a), log_n, batch, in_len, int(inverse), int(coset)))

    def ntt_dev(self, field: int, d_data: int, log_n: int, batch: int = 1, in_len: int = 0, inverse: bool = False, coset: bool = False):
        check(lib().zk_ntt_dev(self._h, field, ctypes.c_void_p(d_data), log_n, batch, in_len, int(inverse), int(coset)))

    def ntt_dev_oop(self, field: int, d_in: int, in_stride: int, in_len: int, d_out: int, log_n: int, batch: int = 1, inverse: bool = False,
                    coset: bool = False):
        """out of place, device to device: polynomial b read from d_in + b * in_stride (first in_len elements), written to d_out + b * 2^log_n"""
        check(lib().zk_ntt_dev_oop(self._h, field, ctypes.c_void_p(d_in), in_stride, in_len, ctypes.c_void_p(d_out), log_n, batch, int(inverse), int(coset)))

    # ------------------------------------------------------------------ device memory (zk_dev_*)
    def dev_alloc(self, nbytes: int) -> int:
        p = ctypes.c_void_p()
        check(lib().zk_dev_alloc(self._h, nbytes, ctypes.byref(p)))
        return p.value

    def dev_free(self, d_ptr: int):
        check(lib().zk_dev_free(self._h, ctypes.c_void_p(d_ptr)))

    def dev_upload(self, d_dst: int, a: np.ndarray):
        a = np.ascontiguousarray(a)
        check(lib().zk_dev_upload(self._h, ctypes.c_void_p(d_dst), _ptr(a), a.nbytes))

    def dev_download(self, d_src: int, shape, dtype=np.uint64) -> np.ndarray:
        out = np.empty(shape, dtype=dtype)
        check(lib().zk_dev_download(self._h, _ptr(out), ctypes.c_void_p(d_src), out.nbytes))
        return out

    def perm_quotient_dev(self, field: int, log_m: int, d_w, d_z: int, d_sigma, d_zkpm: int, beta, gamma, alpha0, shifts, d_out: int, next_shift: int = 8):
        """zk_perm_quotient_dev: the permutation part of the quotient over d8, operands resident on the device; d_w, d_sigma: 7 device
        pointers each"""
        c = lambda a, k: np.ascontiguousarray(a, dtype=np.uint64).reshape(k)
        b, g, a0, sh = c(beta, 4), c(gamma, 4), c(alpha0, 4), c(shifts, 28)
        pw = (ctypes.c_void_p * 7)(*[int(p) for p in d_w])
        ps = (ctypes.c_void_p * 7)(*[int(p) for p in d_sigma])
        check(lib().zk_perm_quotient_dev(self._h, field, log_m, pw, ctypes.c_void_p(d_z), ps, ctypes.c_void_p(d_zkpm), _ptr(b), _ptr(g), _ptr(a0), _ptr(sh),
                                         next_shift, ctypes.c_void_p(d_out)))

    def expr_eval_dev(self, field: int, tokens, constants, cols, out_len: int, out_domain_mult: int, d_out: int, accumulate: bool = False):
        """zk_expr_eval_dev: tokens = [(op, arg)], constants [k, 4] Montgomery, cols = [(device pointer, len, domain_mult)]"""
        tk = (ExprToken * max(1, len(tokens)))(*[ExprToken(int(o), int(a)) for o, a in tokens])
        cn = np.ascontiguousarray(constants, dtype=np.uint64).reshape(-1, 4)
        cl = (ExprColumn * max(1, len(cols)))(*[ExprColumn(int(p), int(n), int(m), 0) for p, n, m in cols])
        check(lib().zk_expr_eval_dev(self._h, field, tk, len(tokens), _ptr(cn) if cn.size else None, cn.shape[0], cl, len(cols), out_len, out_domain_mult,
                                     int(accumulate), ctypes.c_void_p(d_out)))

    def poly_add_dev(self, field: int, d_dst: int, d_src: int, length: int):
        """zk_poly_add_dev: dst[i] += src[i] on device-resident coefficient vectors"""
        check(lib().zk_poly_add_dev(self._h, field, ctypes.c_void_p(d_dst), ctypes.c_void_p(d_src), length))

    def poly_divide_by_vanishing_dev(self, field: int, d_f: int, length: int, log_n: int, d_quot: int) -> bool:
        """zk_poly_divide_by_vanishing_dev: quotient of f by x^n - 1 into d_quot; returns whether the remainder is zero"""
        ok = ctypes.c_int()
        check(lib().zk_poly_divide_by_vanishing_dev(self._h, field, ctypes.c_void_p(d_f), length, log_n, ctypes.c_void_p(d_quot), ctypes.byref(ok)))
        return bool(ok.value)

    # ------------------------------------------------------------------ evaluations at zeta / zeta*omega (zk_lagrange_*, zk_poly_evaluate_chunks_dev)
    @staticmethod
    def lagrange_evals_chunks(domain_size: int, max_poly_size: int) -> int:
        """vectors of LagrangeBasisEvaluations::new(max_poly_size, D(domain_size), x); 0 when the reference would assert"""
        return int(lib().zk_lagrange_evals_chunks(domain_size, max_poly_size))

    def lagrange_basis_evals_dev(self, field: int, log_n: int, max_poly_size: int, x, d_out: int) -> int:
        """zk_lagrange_evals_dev: LagrangeBasisEvaluations::new(max_poly_size, D(2^log_n), x) into d_out (chunks x 2^log_n elements,
        chunk-major); returns the chunk count"""
        xv = np.ascontiguousarray(x, dtype=np.uint64).reshape(4)
        check(lib().zk_lagrange_evals_dev(self._h, field, log_n, max_poly_size, _ptr(xv), ctypes.c_void_p(d_out)))
        return self.lagrange_evals_chunks(1 << log_n, max_poly_size)

    def lagrange_evaluate_dev(self, field: int, d_bases, log_n: int, chunks: int, columns) -> np.ndarray:
        """zk_lagrange_evaluate_dev: columns = [(device pointer, len, boolean)] against the bases d_bases (one device pointer per point,
        built with the same log_n and chunks) -> uint64 [n_cols, n_points, chunks, 4] Montgomery"""
        bases = (ctypes.c_void_p * max(1, len(d_bases)))(*[int(p) for p in d_bases])
        cols = (EvalColumn * max(1, len(columns)))(*[EvalColumn(int(p), int(n), int(bool(b)), 0) for p, n, b in columns])
        out = np.zeros((len(columns), len(d_bases), chunks, 4), dtype=np.uint64)
        check(lib().zk_lagrange_evaluate_dev(self._h, field, bases, len(d_bases), log_n, chunks, cols, len(columns), _ptr(out)))
        return out

    def poly_evaluate_chunks_dev(self, field: int, polys, num_chunks: int, chunk_size: int, points) -> np.ndarray:
        """zk_poly_evaluate_chunks_dev: to_chunked_polynomial(num_chunks, chunk_size).evaluate_chunks(x) of polys = [(device pointer,
        len)] at every point of points [k, 4] (Montgomery) -> uint64 [n_polys, n_points, num_chunks, 4]"""
        pts = np.ascontiguousarray(points, dtype=np.uint64).reshape(-1, 4)
        arr = (DevPoly * max(1, len(polys)))(*[DevPoly(int(p), int(n)) for p, n in polys])
        out = np.zeros((len(polys), pts.shape[0], num_chunks, 4), dtype=np.uint64)
        check(lib().zk_poly_evaluate_chunks_dev(self._h, field, arr, len(polys), num_chunks, chunk_size, _ptr(pts) if pts.size else None,
                                                pts.shape[0], _ptr(out)))
        return out

    # ------------------------------------------------------------------ ft of Maller's optimisation (zk_prover_ft_dev)
    def prover_ft_dev(self, field: int, log_n: int, max_poly_size: int, terms, d_t: int, t_len: int, zeta_mont, d_ft: int):
        """zk_prover_ft_dev (kimchi/src/prover.rs:1147-1206): f = interpolate(sum coeff * evals[(len / n) i]) over D(2^log_n) from
        terms = [(device pointer, len, coeff_mont)], ft = f's chunks linearised at zeta^m minus (zeta^n - 1) times t's (d_t: t_len
        resident coefficients), written to d_ft (room for max_poly_size elements, zero past ft_len).  Returns (ft_len, ft(zeta omega)
        as uint64 [4] Montgomery)."""
        zv = np.ascontiguousarray(zeta_mont, dtype=np.uint64).reshape(4)
        arr = (LinTerm * max(1, len(terms)))()
        for k, (p, n, c) in enumerate(terms):
            arr[k].d_evals, arr[k].len = int(p), int(n)
            arr[k].coeff[:] = [int(v) for v in np.ascontiguousarray(c, dtype=np.uint64).reshape(4)]
        ft_len, ev1 = ctypes.c_size_t(), np.zeros(4, dtype=np.uint64)
        check(lib().zk_prover_ft_dev(self._h, field, log_n, max_poly_size, arr, len(terms), ctypes.c_void_p(d_t), t_len, _ptr(zv),
                                     ctypes.c_void_p(d_ft), ctypes.byref(ft_len), _ptr(ev1)))
        return int(ft_len.value), ev1

    # ------------------------------------------------------------------ permutation aggregation polynomial z (zk_perm_aggreg_dev)
    def perm_aggreg_dev(self, field: int, log_n: int, zk_rows: int, d_w, d_sigma, sigma_len: int, beta, gamma, shifts, rand, d_z: int) -> bool:
        """zk_perm_aggreg_dev (kimchi's ProverIndex::perm_aggreg): z's 2^log_n coefficients into d_z from the 7 resident witness columns
        d_w (2^log_n evaluations each) and the 7 resident sigma columns d_sigma (sigma_len evaluations each, read at stride
        sigma_len / 2^log_n); beta, gamma [4], shifts [7, 4] and rand [2, 4] (the two F::rand draws) Montgomery.  Returns whether
        z[n - zk_rows] == 1 (the reference's "final value" check); z is written either way."""
        c = lambda a, k: np.ascontiguousarray(a, dtype=np.uint64).reshape(k)
        b, g, sh, rn = c(beta, 4), c(gamma, 4), c(shifts, 28), c(rand, 8)
        pw = (ctypes.c_void_p * 7)(*[int(p) for p in d_w])
        ps = (ctypes.c_void_p * 7)(*[int(p) for p in d_sigma])
        ok = ctypes.c_int()
        check(lib().zk_perm_aggreg_dev(self._h, field, log_n, zk_rows, pw, ps, sigma_len, _ptr(b), _ptr(g), _ptr(sh), _ptr(rn),
                                       ctypes.c_void_p(d_z), ctypes.byref(ok)))
        return bool(ok.value)

    # ------------------------------------------------------------------ lookup argument (zk_lookup_*_dev)
    def lookup_joint_table_dev(self, field: int, log_n: int, d_cols, joint_combiner, table_id_combiner, d_out8: int, d_table_ids8: int | None = None,
                               d_runtime8: int | None = None, d_out1: int | None = None):
        """zk_lookup_joint_table_dev: T8[i] = sum_c jc^c col_c[i] + tic tid8[i] over d8 from the resident columns d_cols (8 * 2^log_n
        evaluations each; d_runtime8 is added to column 1), into d_out8 and, if given, its d1 values into d_out1.  Queued on the
        context's stream."""
        c = lambda a: np.ascontiguousarray(a, dtype=np.uint64).reshape(4)
        jc, tic = c(joint_combiner), c(table_id_combiner)
        cols = (ctypes.c_void_p * max(1, len(d_cols)))(*[int(p) for p in d_cols])
        check(lib().zk_lookup_joint_table_dev(self._h, field, log_n, cols, len(d_cols), ctypes.c_void_p(d_table_ids8), ctypes.c_void_p(d_runtime8),
                                              _ptr(jc), _ptr(tic), ctypes.c_void_p(d_out8), ctypes.c_void_p(d_out1)))

    def lookup_sorted_dev(self, field: int, log_n: int, zk_rows: int, d_w, d_table: int, table_stride: int, info, rand, d_sorted) -> int:
        """zk_lookup_sorted_dev (lookup::constraints::sorted + zk_patch): the max_per_row + 1 sorted columns (d1 evaluations) into
        d_sorted from the 15 resident witness columns d_w and the joint table T1[i] = d_table[table_stride i].  info: a LookupInfo
        structure (host.LookupSpec.info); rand: [(m + 1) * zk_rows, 4] Montgomery, column by column.  Returns -1, or the smallest row
        whose lookup value is not in the table (ValueNotInTable; d_sorted is then untouched)."""
        rn = np.ascontiguousarray(rand, dtype=np.uint64).reshape(-1)
        pw = (ctypes.c_void_p * 15)(*[int(p) for p in d_w])
        ps = (ctypes.c_void_p * max(1, len(d_sorted)))(*[int(p) for p in d_sorted])
        row = ctypes.c_int64(-2)
        check(lib().zk_lookup_sorted_dev(self._h, field, log_n, zk_rows, pw, ctypes.c_void_p(d_table), table_stride, ctypes.byref(info),
                                         _ptr(rn) if rn.size else None, ps, ctypes.byref(row)))
        return int(row.value)

    def lookup_aggreg_dev(self, field: int, log_n: int, zk_rows: int, d_w, d_table: int, table_stride: int, info, d_sorted, beta, gamma, rand,
                          d_aggreg: int) -> bool:
        """zk_lookup_aggreg_dev (lookup::constraints::aggregation): the lookup aggregation polynomial's 2^log_n d1 evaluations into
        d_aggreg; rand: [zk_rows, 4] Montgomery.  Returns whether agg[n - zk_rows - 1] == 1 (the reference's debug assertion)."""
        c = lambda a: np.ascontiguousarray(a, dtype=np.uint64).reshape(4)
        b, g = c(beta), c(gamma)
        rn = np.ascontiguousarray(rand, dtype=np.uint64).reshape(-1)
        pw = (ctypes.c_void_p * 15)(*[int(p) for p in d_w])
        ps = (ctypes.c_void_p * max(1, len(d_sorted)))(*[int(p) for p in d_sorted])
        ok = ctypes.c_int()
        check(lib().zk_lookup_aggreg_dev(self._h, field, log_n, zk_rows, pw, ctypes.c_void_p(d_table), table_stride, ctypes.byref(info), ps,
                                         _ptr(b), _ptr(g), _ptr(rn) if rn.size else None, ctypes.c_void_p(d_aggreg), ctypes.byref(ok)))
        return bool(ok.value)

    def points_fold_dev(self, curve: int, d_g: int, h: int, u_mont, d_out: int):
        """zk_points_fold_dev: out[i] = g[i] + [u] g[h + i] on device-resident affine points (the reference's per-round base fold)"""
        u = np.ascontiguousarray(u_mont, dtype=np.uint64).reshape(4)
        check(lib().zk_points_fold_dev(self._h, curve, ctypes.c_void_p(d_g), h, _ptr(u), ctypes.c_void_p(d_out)))

    # ------------------------------------------------------------------ diagnostics
    def field_op(self, field: int, op: str, a, b=None) -> np.ndarray:
        a = _np_u64(a, (4,))
        b = a if b is None else _np_u64(b, (4,))
        out = np.empty_like(a)
        code = {"mul": 0, "add": 1, "sub": 2, "inv": 3}[op]
        check(lib().zk_debug_field_op(self._h, field, code, _ptr(a), _ptr(b), _ptr(out), a.shape[0]))
        return out

    def op_throughput(self, kind: int, blocks: int, threads: int, iters: int = 500, field: int = FP) -> float:
        v = ctypes.c_double()
        check(lib().zk_debug_op_throughput(self._h, field, kind, blocks, threads, iters, ctypes.byref(v)))
        return v.value

    def mul_throughput(self, field: int = FP, iters: int = 2000) -> float:
        v = ctypes.c_double()
        check(lib().zk_debug_mul_throughput(self._h, field, iters, ctypes.byref(v)))
        return v.value


class Bases:
    """Resident MSM bases (SRS::g or one Lagrange basis) on the context's device."""

    def __init__(self, ctx: Context, curve: int, points, window_bits: int = -1, device_ptr: int | None = None, n: int | None = None):
        self.ctx, self.curve = ctx, curve
        self._h = ctypes.c_void_p()
        if device_ptr is not None:
            check(lib().zk_bases_upload(ctx._h, curve, ctypes.c_void_p(device_ptr), n, window_bits, 1, ctypes.byref(self._h)))
        else:
            pts = _np_u64(points, (8,))
            check(lib().zk_bases_upload(ctx._h, curve, _ptr(pts), pts.shape[0], window_bits, 0, ctypes.byref(self._h)))

    def __len__(self):
        return int(lib().zk_bases_len(self._h))

    @property
    def window_bits(self) -> int:
        return int(lib().zk_bases_window_bits(self._h))

    def free(self):
        if getattr(self, "_h", None):
            lib().zk_bases_free(self._h)
            self._h = None

    def __del__(self):
        try:
            if self.ctx._h:
                self.free()
        except Exception:
            pass
