"""proof_systems_b200 — H100-native MSM + NTT hot path of o1-labs/proof-systems (Kimchi).

The product is the C-ABI shared library `libzkb200.so` (include/zkb200.h; hand-written sm_90a CUDA kernels under
csrc/).  This package is the thin Python host layer used by the tests and bench.py: ctypes bindings plus mirrors of the
reference's interfaces on this path, with the reference's names:

    SRS.commit_non_hiding / commit_evaluations_non_hiding / mask_custom    poly-commitment/src/ipa.rs:605-728
    PolyComm                                                               poly-commitment/src/commitment.rs:47-50
    Radix2EvaluationDomain.fft_in_place / ifft_in_place                    ark_poly (kimchi/src/circuits/domains.rs:24-33)
    LagrangeBasisEvaluations.new / evaluate / evaluate_boolean             kimchi/src/lagrange_basis_evaluations.rs:72-258
    IndexCache.build / SRS.index_commitments                               kimchi/src/circuits/constraints.rs:510-760, verifier_index.rs:221-300

There is no CPU fallback anywhere in this package: importing it without the built library, or creating a Context
without a CUDA device, raises.
"""
from ._lib import (  # noqa: F401
    FP, FQ, PALLAS, VESTA, BASE_FIELD, SCALAR_FIELD, ZkError, Context, Bases, IndexHeader, lib, library_path,
    jacobian_to_affine, jacobian_sum,
)
from .host import (  # noqa: F401
    SRS, BatchEvaluationProof, ExprProgram, IndexCache, IpaRounds, LagrangeBasisEvaluations, LookupSpec, OpeningProof, PolyComm, Radix2EvaluationDomain, srs_open, srs_verify,
)
