//! The prover index built on the device (include/zkb200.h, "prover index built on the device").
//!
//! [`DeviceIndex::build`] serialises `cs.gates` and the header fields exactly as the cache writer does (kimchi/src/
//! cached_prover_index.rs:1384-1480: PrunedGate records, GateCoeffs records, ScalarHeader) and hands them to `zk_index_build`, which
//! computes `ColumnEvaluations` (constraints.rs:510-760) on the device.  The sections then stay resident for the prover's `*_dev`
//! calls (`zk_index_cache_section`), and [`DeviceIndex::section`] downloads one when host code still asks for it.  With the index
//! built here, `ProverIndex::create` can run with `lazy_mode = true` so the CPU never computes `ColumnEvaluations` (INTEGRATION.md,
//! "index").  [`DeviceIndex::verifier_commitments`] gives the `PolyComm` fields of `VerifierIndex` (verifier_index.rs:221-300).
use crate::{domain::GpuField, ffi::*, marshal::Limbs4, srs::{check, Ctx, GpuCurve, GpuSRS}};
use core::ffi::c_void;
use kimchi::circuits::{constraints::ConstraintSystem, gate::GateType};
use poly_commitment::PolyComm;
use std::sync::Arc;

/// gate_type_to_tag (cached_prover_index.rs:965-982)
fn gate_tag(t: GateType) -> u16 {
    match t {
        GateType::Zero => 0,
        GateType::Generic => 1,
        GateType::Poseidon => 2,
        GateType::CompleteAdd => 3,
        GateType::VarBaseMul => 4,
        GateType::EndoMul => 5,
        GateType::EndoMulScalar => 6,
        GateType::Lookup => 7,
        GateType::RangeCheck0 => 8,
        GateType::RangeCheck1 => 9,
        GateType::ForeignFieldAdd => 10,
        GateType::ForeignFieldMul => 11,
        GateType::Xor16 => 12,
        GateType::Rot64 => 13,
    }
}

/// The commitment fields of `VerifierIndex`, in the order `zk_index_commitments` writes them.
pub struct VerifierCommitments<G> {
    pub sigma_comm: Vec<PolyComm<G>>,
    pub coefficients_comm: Vec<PolyComm<G>>,
    pub generic_comm: PolyComm<G>,
    pub psm_comm: PolyComm<G>,
    pub complete_add_comm: PolyComm<G>,
    pub mul_comm: PolyComm<G>,
    pub emul_comm: PolyComm<G>,
    pub endomul_scalar_comm: PolyComm<G>,
    /// range_check0, range_check1, foreign_field_add, foreign_field_mul, xor, rot: present where the circuit uses the gate
    pub optional: [Option<PolyComm<G>>; 6],
}

/// A prover index resident on the device (a `zk_index_cache` handle).
pub struct DeviceIndex {
    pub(crate) h: *mut zk_index_cache,
    _ctx: Arc<Ctx>,
}
unsafe impl Send for DeviceIndex {}
unsafe impl Sync for DeviceIndex {}
impl Drop for DeviceIndex {
    fn drop(&mut self) {
        unsafe { zk_index_cache_free(self.h) }
    }
}

impl DeviceIndex {
    /// `zero_selectors`: the caller's `cfg!(debug_assertions) && cs.disable_gates_checks` (selector_polynomial, constraints.rs:334-362)
    pub fn build<F: GpuField>(ctx: &Arc<Ctx>, cs: &ConstraintSystem<F>, max_poly_size: usize, zero_selectors: bool) -> Result<Self, String> {
        let mut gates = Vec::with_capacity(cs.gates.len() * 60);
        let mut coeffs = Vec::new();
        for g in cs.gates.iter() {
            gates.extend_from_slice(&gate_tag(g.typ).to_le_bytes());
            gates.extend_from_slice(&[0u8; 2]);
            for w in g.wires.iter() {
                gates.extend_from_slice(&(w.row as u32).to_le_bytes());
                gates.extend_from_slice(&(w.col as u32).to_le_bytes());
            }
            coeffs.extend_from_slice(&(g.coeffs.len() as u32).to_le_bytes());
            for c in g.coeffs.iter() {
                for l in c.to_limbs() {
                    coeffs.extend_from_slice(&l.to_le_bytes());
                }
            }
        }
        let f = &cs.feature_flags;
        let optional = [f.range_check0, f.range_check1, f.foreign_field_add, f.foreign_field_mul, f.xor, f.rot]
            .iter()
            .enumerate()
            .fold(0u32, |b, (i, on)| if *on { b | 1 << i } else { b });
        let l = &f.lookup_features;
        let lookup_bits = [l.patterns.xor, l.patterns.lookup, l.patterns.range_check, l.patterns.foreign_field_mul, l.joint_lookup_used,
                           l.uses_runtime_tables]
            .iter()
            .enumerate()
            .fold(0u32, |b, (i, on)| if *on { b | 1 << (8 + i) } else { b });
        // ScalarHeader (cached_prover_index.rs:1434-1448); the lookup sections are not built here, so lookup_selectors_present is 0
        let hdr = zk_index_header {
            public_inputs: cs.public as u32,
            prev_challenges: cs.prev_challenges as u32,
            zk_rows: cs.zk_rows,
            max_poly_size: max_poly_size as u64,
            domain_d1_size: cs.domain.d1.size,
            feature_flags: optional | lookup_bits,          // pack_feature_flags (:808-847): the low six bits are the optional gates
            optional_selectors_present: optional,
            lookup_selectors_present: 0,
            num_sections: 0,
            disable_gates_checks: cs.disable_gates_checks as i32,
            has_verifier_index_digest: 0,
            endo: cs.endo.to_limbs(),
            shift: core::array::from_fn(|k| cs.shift[k].to_limbs()),
            verifier_index_digest: [0; 4],
            identifier: [0; 512],
        };
        let mut h = core::ptr::null_mut();
        check(unsafe {
            zk_index_build(ctx.0, F::FIELD_ID, &hdr, gates.as_ptr() as *const c_void, cs.gates.len(), coeffs.as_ptr() as *const c_void,
                           coeffs.len(), zero_selectors as i32, &mut h)
        })?;
        Ok(DeviceIndex { h, _ctx: ctx.clone() })
    }

    /// Device pointer and element count of a section (0x01 sid, 0x10 + i coefficients8, 0x20 .. 0x25 selectors, 0x30 + k
    /// permutation_coefficients8, 0x40 + b optional selectors), as the `*_dev` calls take them.
    pub fn section_ptr(&self, tag: u32) -> Result<(*const c_void, usize), String> {
        let (mut p, mut n, mut d) = (core::ptr::null(), 0usize, 0u32);
        check(unsafe { zk_index_cache_section(self.h, tag, &mut p, &mut n, &mut d) })?;
        Ok((p, n))
    }

    /// A section's evaluations on the host: what a `LazyCache` of `ColumnEvaluations` reads instead of recomputing them.
    pub fn section<F: GpuField>(&self, ctx: &Ctx, tag: u32) -> Result<Vec<F>, String> {
        let (p, n) = self.section_ptr(tag)?;
        let mut limbs = vec![0u64; 4 * n];
        check(unsafe { zk_dev_download(ctx.0, limbs.as_mut_ptr() as *mut c_void, p, 32 * n) })?;
        Ok(limbs.chunks(4).map(|l| F::from_limbs([l[0], l[1], l[2], l[3]])).collect())
    }

    /// `ProverIndex::verifier_index`'s commitments: 28 + k `commit_evaluations_non_hiding` over the resident sections, the six
    /// fixed selectors masked with blinder one.
    pub fn verifier_commitments<G: GpuCurve>(&self, srs: &GpuSRS<G>) -> Result<VerifierCommitments<G>, String> {
        let mut hdr = core::mem::MaybeUninit::<zk_index_header>::uninit();
        check(unsafe { zk_index_cache_header(self.h, hdr.as_mut_ptr()) })?;
        let hdr = unsafe { hdr.assume_init() };
        let chunks = unsafe { zk_srs_lagrange_basis_chunks(srs.dev.0, hdr.domain_d1_size as usize) };
        let count = 28 + hdr.optional_selectors_present.count_ones() as usize;
        let mut xy = vec![0u64; 8 * chunks * count];
        let mut got = 0usize;
        check(unsafe { zk_index_commitments(srs.dev.0, self.h, xy.as_mut_ptr(), chunks * count, &mut got) })?;
        let mut comms = xy[..8 * got].chunks(8 * chunks).map(|c| PolyComm::new(c.chunks(8).map(G::from_limbs).collect()));
        let mut next = || comms.next().expect("zk_index_commitments wrote every commitment");
        let sigma_comm = (0..7).map(|_| next()).collect();
        let coefficients_comm = (0..15).map(|_| next()).collect();
        let (generic_comm, psm_comm, complete_add_comm, mul_comm, emul_comm, endomul_scalar_comm) = (next(), next(), next(), next(), next(), next());
        let optional = core::array::from_fn(|b| if hdr.optional_selectors_present >> b & 1 == 1 { Some(next()) } else { None });
        Ok(VerifierCommitments { sigma_comm, coefficients_comm, generic_comm, psm_comm, complete_add_comm, mul_comm, emul_comm,
                                 endomul_scalar_comm, optional })
    }
}
