//! The prover index built on the device (include/zkb200.h, "prover index built on the device").
//!
//! [`DeviceIndex::build`] serialises `cs.gates` and the header fields exactly as the cache writer does (kimchi/src/
//! cached_prover_index.rs:1384-1480: PrunedGate records, GateCoeffs records, ScalarHeader) and hands them to `zk_index_build`, which
//! computes `ColumnEvaluations` (constraints.rs:510-760) on the device.  The sections then stay resident for the prover's `*_dev`
//! calls (`zk_index_cache_section`), and [`DeviceIndex::section`] downloads one when host code still asks for it.  With the index
//! built here, `ProverIndex::create` can run with `lazy_mode = true` so the CPU never computes `ColumnEvaluations` (INTEGRATION.md,
//! "index").  [`DeviceIndex::verifier_commitments`] gives the `PolyComm` fields of `VerifierIndex` (verifier_index.rs:221-300).
//!
//! [`DeviceLookupIndex::build`] does the same for `LookupConstraintSystem::create` (kimchi/src/circuits/lookup/index.rs:202-482):
//! `zk_lookup_index_build` computes `lookup_table8`, `table_ids8`, the pattern selectors and the runtime selector on the device, and
//! [`DeviceLookupIndex::verifier_commitments`] gives the commitment fields of `LookupVerifierIndex` (verifier_index.rs:196-215).
use crate::{domain::GpuField, ffi::*, marshal::Limbs4, srs::{check, last_error, Ctx, GpuCurve, GpuSRS}};
use ark_poly::Radix2EvaluationDomain as D;
use core::ffi::c_void;
use kimchi::circuits::{
    constraints::ConstraintSystem,
    gate::{CircuitGate, GateType},
    lookup::{index::{LookupError, LookupSelectors}, runtime_tables::RuntimeTableCfg, tables::LookupTable},
};
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

/// write_pruned_gate (cached_prover_index.rs:1007-1015): typ_tag u16 | pad[2] | 7 x (row u32, col u32)
fn pruned_gates<F>(gates: &[CircuitGate<F>]) -> Vec<u8> {
    let mut out = Vec::with_capacity(gates.len() * 60);
    for g in gates.iter() {
        out.extend_from_slice(&gate_tag(g.typ).to_le_bytes());
        out.extend_from_slice(&[0u8; 2]);
        for w in g.wires.iter() {
            out.extend_from_slice(&(w.row as u32).to_le_bytes());
            out.extend_from_slice(&(w.col as u32).to_le_bytes());
        }
    }
    out
}

impl DeviceIndex {
    /// `zero_selectors`: the caller's `cfg!(debug_assertions) && cs.disable_gates_checks` (selector_polynomial, constraints.rs:334-362)
    pub fn build<F: GpuField>(ctx: &Arc<Ctx>, cs: &ConstraintSystem<F>, max_poly_size: usize, zero_selectors: bool) -> Result<Self, String> {
        let gates = pruned_gates(&cs.gates);
        let mut coeffs = Vec::new();
        for g in cs.gates.iter() {
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

/// The commitment fields of `LookupVerifierIndex` (verifier_index.rs:196-215); the host adds `lookup_info` and `joint_lookup_used`.
pub struct LookupVerifierCommitments<G> {
    pub lookup_table: Vec<PolyComm<G>>,
    pub lookup_selectors: LookupSelectors<PolyComm<G>>,
    pub table_ids: Option<PolyComm<G>>,
    pub runtime_tables_selector: Option<PolyComm<G>>,
}

/// A lookup index resident on the device (a `zk_index_cache` handle with sections 0x50 .. 0x56).
pub struct DeviceLookupIndex {
    pub(crate) h: *mut zk_index_cache,
    /// `LookupConstraintSystem::runtime_table_offset`
    pub runtime_table_offset: Option<usize>,
    _ctx: Arc<Ctx>,
}
unsafe impl Send for DeviceLookupIndex {}
unsafe impl Sync for DeviceLookupIndex {}
impl Drop for DeviceLookupIndex {
    fn drop(&mut self) {
        unsafe { zk_index_cache_free(self.h) }
    }
}

impl DeviceLookupIndex {
    /// `LookupConstraintSystem::create(gates, fixed_tables, runtime_cfgs, domain, zk_rows)` on the device: `Ok(None)` when no gate
    /// uses a lookup.  `ConstraintSystem` does not keep the tables, so the caller passes the ones it gave `Builder::lookup` /
    /// `Builder::runtime`.  Panics where the library refuses the arguments (a null table, a width beyond 16, a Next pattern on the
    /// last row) or the device fails.
    pub fn build<F: GpuField>(ctx: &Arc<Ctx>, gates: &[CircuitGate<F>], fixed_tables: &[LookupTable<F>],
                              runtime_cfgs: Option<&[RuntimeTableCfg<F>]>, d1: D<F>, zk_rows: usize) -> Result<Option<Self>, LookupError> {
        // index.rs:394-399: the one LookupError the C ABI cannot express (it takes one length per table)
        if fixed_tables.iter().any(|t| t.data.iter().any(|c| c.len() != t.data[0].len())) {
            return Err(LookupError::InconsistentTableLength);
        }
        let limbs = |v: &[F]| v.iter().flat_map(|x| x.to_limbs()).collect::<Vec<u64>>();
        let data: Vec<Vec<u64>> = fixed_tables.iter().map(|t| t.data.iter().flat_map(|c| limbs(c.as_slice())).collect()).collect();
        let tables: Vec<zk_lookup_table> = fixed_tables
            .iter()
            .zip(data.iter())
            .map(|(t, d)| zk_lookup_table { id: t.id, width: t.data.len() as u32, len: t.data.first().map_or(0, |c| c.len()) as u64, data: d.as_ptr() })
            .collect();
        let rt = runtime_cfgs.unwrap_or(&[]);
        let first: Vec<Vec<u64>> = rt.iter().map(|r| limbs(r.first_column.as_slice())).collect();
        let runtime: Vec<zk_runtime_table_cfg> = rt
            .iter()
            .zip(first.iter())
            .map(|(r, c)| zk_runtime_table_cfg { id: r.id, len: r.first_column.len() as u64, first_column: c.as_ptr() })
            .collect();
        let g = pruned_gates(gates);
        let (mut kind, mut offset, mut h) = (ZK_LOOKUP_ERR_NONE, 0u64, core::ptr::null_mut());
        let rc = unsafe {
            zk_lookup_index_build(ctx.0, F::FIELD_ID, d1.size, zk_rows as u64, g.as_ptr() as *const c_void, gates.len(), tables.as_ptr(),
                                  tables.len(), runtime.as_ptr(), runtime.len(), runtime_cfgs.is_some() as i32, &mut kind, &mut offset, &mut h)
        };
        if rc != ZK_OK {
            let msg = last_error();
            // the library's message is the reference's Display text: recover the fields it carries
            let after = |p: &str| msg.split(p).nth(1).unwrap_or("").to_string();
            return match kind {
                ZK_LOOKUP_ERR_ID_COLLISION => Err(LookupError::LookupTableIdCollision { collision_type: after("The collision type is: ") }),
                ZK_LOOKUP_ERR_TABLE_ID_ZERO => Err(LookupError::TableIDZeroMustHaveZeroEntry),
                ZK_LOOKUP_ERR_TOO_LONG => {
                    let num = |p: &str| after(p).split(',').next().unwrap_or("").trim().parse().unwrap_or(0);
                    Err(LookupError::LookupTableTooLong { length: num("Observed: "), maximum_allowed: num("expected: ") })
                }
                _ => panic!("zkb200 error {rc}: {msg}"),
            };
        }
        if h.is_null() {
            return Ok(None);
        }
        Ok(Some(DeviceLookupIndex { h, runtime_table_offset: runtime_cfgs.map(|_| offset as usize), _ctx: ctx.clone() }))
    }

    /// Device pointer and element count of a section (0x50 the lookup_table8 columns back to back, 0x51 table_ids8, 0x52 .. 0x55
    /// the selectors xor, lookup, range_check, ffmul, 0x56 runtime_selector8), as the `*_dev` calls take them.
    pub fn section_ptr(&self, tag: u32) -> Result<(*const c_void, usize), String> {
        let (mut p, mut n, mut d) = (core::ptr::null(), 0usize, 0u32);
        check(unsafe { zk_index_cache_section(self.h, tag, &mut p, &mut n, &mut d) })?;
        Ok((p, n))
    }

    /// `ProverIndex::verifier_index`'s lookup commitments: the table columns and the table ids masked with blinder one, the
    /// selectors and the runtime selector not.
    pub fn verifier_commitments<G: GpuCurve>(&self, srs: &GpuSRS<G>) -> Result<LookupVerifierCommitments<G>, String> {
        let mut hdr = core::mem::MaybeUninit::<zk_index_header>::uninit();
        check(unsafe { zk_index_cache_header(self.h, hdr.as_mut_ptr()) })?;
        let hdr = unsafe { hdr.assume_init() };
        let (mut p, mut n, mut width) = (core::ptr::null(), 0usize, 0u32);
        check(unsafe { zk_index_cache_section(self.h, 0x50, &mut p, &mut n, &mut width) })?;
        let bits = hdr.lookup_selectors_present;
        let chunks = unsafe { zk_srs_lagrange_basis_chunks(srs.dev.0, hdr.domain_d1_size as usize) };
        let count = width as usize + (bits & 0x3F).count_ones() as usize;
        let mut xy = vec![0u64; 8 * chunks * count];
        let mut got = 0usize;
        check(unsafe { zk_lookup_index_commitments(srs.dev.0, self.h, xy.as_mut_ptr(), chunks * count, &mut got) })?;
        let mut comms = xy[..8 * got].chunks(8 * chunks).map(|c| PolyComm::new(c.chunks(8).map(G::from_limbs).collect()));
        let mut next = || comms.next().expect("zk_lookup_index_commitments wrote every commitment");
        let lookup_table = (0..width).map(|_| next()).collect();
        let mut opt = |b: u32| if bits >> b & 1 == 1 { Some(next()) } else { None };
        let table_ids = opt(0);
        let lookup_selectors = LookupSelectors { xor: opt(1), lookup: opt(2), range_check: opt(3), ffmul: opt(4) };
        let runtime_tables_selector = opt(5);
        Ok(LookupVerifierCommitments { lookup_table, lookup_selectors, table_ids, runtime_tables_selector })
    }
}
