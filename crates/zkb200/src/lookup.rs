//! The lookup argument on the device (kimchi/src/prover.rs:383-673; include/zkb200.h, "lookup argument"): the joint lookup table,
//! the sorted columns and the lookup aggregation polynomial, built from the resident witness and the index cache's
//! `lookup_table8` (section 0x50, the columns packed) and `table_ids8` (0x51), and left resident as d1 evaluations for
//! `commit_evaluations` (`zk_msm_dev` over the Lagrange basis), `zk_ntt_dev_oop` and the lookup constraints (`zk_expr_eval_dev`).
//!
//! [`LookupLowering::new`] lowers `LookupInfo::by_row(&index.cs.gates)` once per index: one pattern per distinct `LookupPattern`,
//! its `lookups()` as terms.  The prover's random values are drawn in the reference's order: the runtime table's zk rows (the
//! caller, before [`LookupLowering::joint_table_dev`]), (m + 1) x zk_rows for the sorted columns ([`LookupLowering::sorted_dev`]),
//! the sorted commitments' blinders (the caller's commit), zk_rows for the aggregation ([`LookupLowering::aggreg_dev`]), then its
//! blinders (INTEGRATION.md, "lookup").
use crate::{domain::GpuField, expr::DeviceEvals, ffi::*, srs::Ctx};
use ark_ff::{One, UniformRand};
use ark_poly::Radix2EvaluationDomain as D;
use core::ffi::c_void;
use core::marker::PhantomData;
use kimchi::circuits::gate::{CircuitGate, CurrOrNext};
use kimchi::circuits::lookup::lookups::{LookupInfo, LookupPattern, LookupTableID};
use kimchi::error::ProverError;
use rand_core::{CryptoRng, RngCore};

/// `LookupInfo` of one index in the form of `zk_lookup_info`
pub struct LookupLowering<F: GpuField> {
    terms: Vec<zk_lookup_term>,
    lookups: Vec<zk_lookup_joint>,
    pattern_first: Vec<u32>,
    pattern_count: Vec<u32>,
    row_pattern: Vec<u8>, // by_row over the gates: 0 none, p + 1 pattern p
    max_per_row: u32,
    _f: PhantomData<F>,
}

fn gpu(_: String) -> ProverError {
    ProverError::Prover("zkb200: lookup") // the library's message: zk_last_error()
}

fn alloc(ctx: &Ctx, n: usize, domain_mult: u32) -> Result<DeviceEvals, ProverError> {
    let mut p = core::ptr::null_mut();
    crate::srs::check(unsafe { zk_dev_alloc(ctx.0, 32 * n, &mut p) }).map_err(gpu)?;
    Ok(DeviceEvals { ptr: p, len: n as u64, domain_mult })
}

fn free_all(ctx: &Ctx, bufs: &[DeviceEvals]) {
    for b in bufs {
        unsafe { zk_dev_free(ctx.0, b.ptr) };
    }
}

impl<F: GpuField> LookupLowering<F> {
    /// `lookup_rows` = n - zk_rows - 1 rows of `LookupInfo::by_row(gates)` (lookups.rs:286-299), whose pattern assignment this
    /// repeats: a gate's `Curr` pattern on its row, its `Next` pattern on the row after.
    pub fn new(info: &LookupInfo, gates: &[CircuitGate<F>], lookup_rows: usize) -> Self {
        let mut kinds: Vec<Option<LookupPattern>> = vec![None; gates.len() + 1];
        for (i, g) in gates.iter().enumerate() {
            if let Some(p) = LookupPattern::from_gate(g.typ, CurrOrNext::Curr) {
                kinds[i] = Some(p);
            }
            if let Some(p) = LookupPattern::from_gate(g.typ, CurrOrNext::Next) {
                kinds[i + 1] = Some(p);
            }
        }
        let mut me = LookupLowering { terms: vec![], lookups: vec![], pattern_first: vec![], pattern_count: vec![], row_pattern: vec![],
                                      max_per_row: info.max_per_row as u32, _f: PhantomData };
        let mut index: Vec<(LookupPattern, u8)> = vec![];
        for i in 0..lookup_rows {
            let p = match kinds.get(i).copied().flatten() {
                None => 0,
                Some(kind) => match index.iter().find(|(k, _)| *k == kind) {
                    Some((_, p)) => *p,
                    None => {
                        me.lower_pattern(kind);
                        index.push((kind, me.pattern_first.len() as u8));
                        me.pattern_first.len() as u8
                    }
                },
            };
            me.row_pattern.push(p);
        }
        me
    }

    fn lower_pattern(&mut self, kind: LookupPattern) {
        let specs = kind.lookups::<F>();
        self.pattern_first.push(self.lookups.len() as u32);
        self.pattern_count.push(specs.len() as u32);
        for spec in specs {
            let first_term = self.terms.len() as u32;
            let mut entry_terms = [0u32; 4];
            for (e, single) in spec.entry.iter().enumerate() {
                for (coeff, pos) in &single.value {
                    let next = matches!(pos.row, CurrOrNext::Next) as u32;
                    self.terms.push(zk_lookup_term { coeff: coeff.to_limbs(), column: pos.column as u32, next });
                }
                if e < 4 {
                    entry_terms[e] = single.value.len() as u32;
                }
            }
            let (table_id, table_id_column) = match spec.table_id {
                LookupTableID::Constant(id) => (id, -1),
                LookupTableID::WitnessColumn(c) => (0, c as i32),
            };
            self.lookups.push(zk_lookup_joint { table_id, table_id_column, n_entries: spec.entry.len() as u32, entry_terms, first_term });
        }
    }

    fn info(&self, jc: F, tic: F, dummy: F) -> zk_lookup_info {
        zk_lookup_info {
            terms: self.terms.as_ptr(),
            n_terms: self.terms.len(),
            lookups: self.lookups.as_ptr(),
            n_lookups: self.lookups.len(),
            pattern_first: self.pattern_first.as_ptr(),
            pattern_count: self.pattern_count.as_ptr(),
            n_patterns: self.pattern_first.len(),
            row_pattern: self.row_pattern.as_ptr(),
            max_per_row: self.max_per_row,
            joint_combiner: jc.to_limbs(),
            table_id_combiner: tic.to_limbs(),
            dummy: dummy.to_limbs(),
        }
    }

    /// The joint lookup table over d8 and its d1 values (prover.rs:500-568): `lookup_table8` the table's columns over d8,
    /// `table_ids8` / `runtime8` (the runtime table contribution over d8, added to column 1) optional.
    #[allow(clippy::too_many_arguments)]
    pub fn joint_table_dev(ctx: &Ctx, domain: D<F>, lookup_table8: &[&DeviceEvals], table_ids8: Option<&DeviceEvals>,
                           runtime8: Option<&DeviceEvals>, jc: F, tic: F) -> Result<(DeviceEvals, DeviceEvals), ProverError> {
        let n = domain.size as usize;
        let cols: Vec<*const c_void> = lookup_table8.iter().map(|e| e.ptr as *const c_void).collect();
        let opt = |e: Option<&DeviceEvals>| e.map_or(core::ptr::null(), |e| e.ptr as *const c_void);
        let t8 = alloc(ctx, 8 * n, 8)?;
        let t1 = match alloc(ctx, n, 1) {
            Ok(b) => b,
            Err(e) => {
                free_all(ctx, &[t8]);
                return Err(e);
            }
        };
        let rc = crate::srs::check(unsafe {
            zk_lookup_joint_table_dev(ctx.0, F::FIELD_ID, domain.log_size_of_group, cols.as_ptr(), cols.len(), opt(table_ids8), opt(runtime8),
                                      jc.to_limbs().as_ptr(), tic.to_limbs().as_ptr(), t8.ptr, t1.ptr)
        });
        if let Err(e) = rc {
            free_all(ctx, &[t8, t1]);
            return Err(gpu(e));
        }
        Ok((t8, t1))
    }

    /// `lookup::constraints::sorted` and `zk_patch` per column: max_per_row + 1 resident d1 columns, or
    /// `ProverError::ValueNotInTable(row)`.  Draws the (m + 1) x zk_rows random values, column by column.
    #[allow(clippy::too_many_arguments)]
    pub fn sorted_dev<R: RngCore + CryptoRng>(&self, ctx: &Ctx, domain: D<F>, zk_rows: usize, witness: &[&DeviceEvals; 15], table8: &DeviceEvals,
                                              jc: F, tic: F, dummy: F, rng: &mut R) -> Result<Vec<DeviceEvals>, ProverError> {
        let n = domain.size as usize;
        let m = self.max_per_row as usize;
        let rand: Vec<u64> = (0..(m + 1) * zk_rows).flat_map(|_| F::rand(rng).to_limbs()).collect();
        let w: Vec<*const c_void> = witness.iter().map(|e| e.ptr as *const c_void).collect();
        let mut out = vec![];
        for _ in 0..=m {
            match alloc(ctx, n, 1) {
                Ok(b) => out.push(b),
                Err(e) => {
                    free_all(ctx, &out);
                    return Err(e);
                }
            }
        }
        let ptrs: Vec<*mut c_void> = out.iter().map(|b| b.ptr).collect();
        let info = self.info(jc, tic, dummy);
        let mut row = -1i64;
        let rc = crate::srs::check(unsafe {
            zk_lookup_sorted_dev(ctx.0, F::FIELD_ID, domain.log_size_of_group, zk_rows, w.as_ptr(), table8.ptr as *const c_void, 8, &info,
                                 rand.as_ptr(), ptrs.as_ptr(), &mut row)
        });
        if rc.is_err() || row >= 0 {
            free_all(ctx, &out);
            rc.map_err(gpu)?;
            return Err(ProverError::ValueNotInTable(row as usize));
        }
        Ok(out)
    }

    /// `lookup::constraints::aggregation` (and its zk_patch): the aggregation's resident d1 evaluations.  Draws the zk_rows random
    /// values.  Like the reference, panics on a final value other than one only with debug assertions.
    #[allow(clippy::too_many_arguments)]
    pub fn aggreg_dev<R: RngCore + CryptoRng>(&self, ctx: &Ctx, domain: D<F>, zk_rows: usize, witness: &[&DeviceEvals; 15], table8: &DeviceEvals,
                                              jc: F, tic: F, dummy: F, sorted: &[DeviceEvals], beta: F, gamma: F, rng: &mut R)
                                              -> Result<DeviceEvals, ProverError> {
        let n = domain.size as usize;
        let rand: Vec<u64> = (0..zk_rows).flat_map(|_| F::rand(rng).to_limbs()).collect();
        let w: Vec<*const c_void> = witness.iter().map(|e| e.ptr as *const c_void).collect();
        let s: Vec<*const c_void> = sorted.iter().map(|e| e.ptr as *const c_void).collect();
        let agg = alloc(ctx, n, 1)?;
        let info = self.info(jc, tic, dummy);
        let mut final_is_one = 0;
        let rc = crate::srs::check(unsafe {
            zk_lookup_aggreg_dev(ctx.0, F::FIELD_ID, domain.log_size_of_group, zk_rows, w.as_ptr(), table8.ptr as *const c_void, 8, &info,
                                 s.as_ptr(), beta.to_limbs().as_ptr(), gamma.to_limbs().as_ptr(), rand.as_ptr(), agg.ptr, &mut final_is_one)
        });
        if let Err(e) = rc {
            free_all(ctx, &[agg]);
            return Err(gpu(e));
        }
        if cfg!(debug_assertions) && final_is_one == 0 {
            panic!("aggregation incorrect: the final value is not {}", F::one());
        }
        Ok(agg)
    }
}
