//! H100 back end for Kimchi's two proving-time hot paths, behind the reference's own seams:
//!
//! * [`GpuSRS`] implements `poly_commitment::SRS<G>` (poly-commitment/src/lib.rs:61-241) — every MSM-bearing method runs on the
//!   device, the rest follows `ipa::SRS` (poly-commitment/src/ipa.rs:596-800);
//! * [`GpuOpeningProof`] implements `poly_commitment::OpenProof<G, FULL_ROUNDS>` (lib.rs:254-298) with the serde layout of
//!   `ipa::OpeningProof` (ipa.rs:1175-1191): `open` is one `zk_srs_open` call, `verify` is the reference's verifier;
//! * [`GpuRadix2Domain`] implements `ark_poly::EvaluationDomain<F>` by delegation to `Radix2EvaluationDomain`, with
//!   `fft_in_place` / `ifft_in_place` on field elements sent to `zk_ntt_batch`.
//!
//! * [`expr::DeviceColumns`] runs `Expr::evaluations` (kimchi/src/circuits/expr.rs:1938-2190) — the gate and lookup constraints of
//!   the quotient — as RPN programs over device-resident columns (`zk_expr_eval_dev`).
//! * [`evals::DeviceLagrangeEvals`] and [`evals::evaluate_chunks_dev`] compute the prover's evaluations at zeta and zeta*omega
//!   (kimchi/src/prover.rs:1009-1058) over the same resident columns (`zk_lagrange_evaluate_dev`, `zk_poly_evaluate_chunks_dev`).
//! * [`ft::ft_dev`] computes the ft polynomial of Maller's optimisation (kimchi/src/prover.rs:1147-1206) from the resident quotient
//!   and sigma_6 over d8, leaving ft resident for the opening proof (`zk_prover_ft_dev`).
//! * [`perm::perm_aggreg_dev`] builds the permutation aggregation polynomial z (kimchi/src/circuits/polynomials/permutation.rs:447-574)
//!   from the resident witness and `permutation_coefficients8`, leaving z resident (`zk_perm_aggreg_dev`).
//! * [`index::DeviceIndex`] builds the prover index's column evaluations (kimchi/src/circuits/constraints.rs:510-760) on the device
//!   from `cs.gates` and the commitments of its verifier index (kimchi/src/verifier_index.rs:221-300) (`zk_index_build`,
//!   `zk_index_commitments`); [`index::DeviceLookupIndex`] does the same for the lookup index (kimchi/src/circuits/lookup/index.rs:
//!   202-482) and the lookup commitments of the verifier index (`zk_lookup_index_build`, `zk_lookup_index_commitments`).
//! * [`accumulator::batch_dlog_accumulator_check`] and [`accumulator::batch_dlog_accumulator_generate`] are the recursion
//!   accumulators of poly-commitment/src/utils.rs:204-312 over the resident generators (`zk_srs_accumulator_*`).
//! * [`lookup::LookupLowering`] builds the lookup argument's joint table, sorted columns and aggregation polynomial
//!   (kimchi/src/prover.rs:383-673) from the resident witness and the index cache's lookup tables (`zk_lookup_*_dev`).
//!
//! Everything called is declared in include/zkb200.h and exported by libzkb200.so; there is no CPU fallback inside the library
//! (`Ctx::new` fails without a CUDA device) — code that must also run without a GPU keeps using `ipa::SRS`.
pub mod accumulator;
pub mod domain;
pub mod evals;
pub mod expr;
pub mod ffi;
pub mod ft;
pub mod index;
pub mod lookup;
pub mod marshal;
pub mod open;
pub mod perm;
pub mod srs;

pub use domain::GpuRadix2Domain;
pub use open::GpuOpeningProof;
pub use srs::{Ctx, GpuCurve, GpuSRS};
