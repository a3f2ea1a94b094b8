//! The prover's evaluations at zeta and zeta*omega on the device (kimchi/src/prover.rs:1009-1058; include/zkb200.h, "evaluations at
//! zeta and zeta*omega").
//!
//! [`DeviceLagrangeEvals`] mirrors `kimchi::lagrange_basis_evaluations::LagrangeBasisEvaluations` (lagrange_basis_evaluations.rs:24-258)
//! with its basis values resident, and evaluates resident [`DeviceEvals`] (the `permutation_coefficients8`, `coefficients8` and
//! selectors of the column evaluations, or of a cached prover index).  [`evaluate_chunks_dev`] is
//! `to_chunked_polynomial(num_chunks, max_poly_size).evaluate_chunks(x)` on resident coefficient vectors (witness, z, public).  The
//! prover's block then reads (INTEGRATION.md §3a)
//!
//! ```ignore
//! let zeta_evals = DeviceLagrangeEvals::new(&ctx, index.max_poly_size, index.cs.domain.d1, zeta)?;
//! let zeta_omega_evals = DeviceLagrangeEvals::new(&ctx, index.max_poly_size, index.cs.domain.d1, zeta_omega)?;
//! let cols: Vec<(&DeviceEvals, bool)> = s8.iter().chain(&coefficients8).map(|e| (e, false))
//!     .chain(selectors.iter().map(|e| (e, true))).collect();
//! let evals = DeviceLagrangeEvals::evaluate_all(&[&zeta_evals, &zeta_omega_evals], &cols)?;   // [column][point][chunk]
//! let chunks = evaluate_chunks_dev(&ctx, &polys, num_chunks, index.max_poly_size, &[zeta, zeta_omega])?;
//! ```
use crate::{
    domain::GpuField,
    expr::DeviceEvals,
    ffi::*,
    marshal::fields_of,
    srs::{check, Ctx},
};
use ark_poly::{EvaluationDomain, Radix2EvaluationDomain as D};
use core::ffi::c_void;
use core::marker::PhantomData;

/// `LagrangeBasisEvaluations<F>` with its `chunks x n` values in device memory (freed on drop).
pub struct DeviceLagrangeEvals<'c, F: GpuField> {
    ctx: &'c Ctx,
    ptr: *mut c_void,
    log_n: u32,
    chunks: usize,
    _f: PhantomData<F>,
}

impl<'c, F: GpuField> DeviceLagrangeEvals<'c, F> {
    /// `LagrangeBasisEvaluations::new(max_poly_size, domain, x)` (:242-258).  A domain larger than `max_poly_size` and not a multiple
    /// of it is the reference's assert and an error here.
    pub fn new(ctx: &'c Ctx, max_poly_size: usize, domain: D<F>, x: F) -> Result<Self, String> {
        let n = domain.size();
        let chunks = unsafe { zk_lagrange_evals_chunks(n, max_poly_size) };
        if chunks == 0 {
            return Err(format!("domain size {n} is not a multiple of max_poly_size {max_poly_size}"));
        }
        let mut ptr = core::ptr::null_mut();
        check(unsafe { zk_dev_alloc(ctx.0, 32 * chunks * n, &mut ptr) })?;
        let out = Self { ctx, ptr, log_n: domain.log_size_of_group, chunks, _f: PhantomData };
        let xl = x.to_limbs();
        check(unsafe { zk_lagrange_evals_dev(ctx.0, F::FIELD_ID, out.log_n, max_poly_size, xl.as_ptr(), ptr) })?;
        Ok(out)
    }

    /// `domain_size` (:45-47): the length of every chunk vector
    pub fn domain_size(&self) -> usize {
        1 << self.log_n
    }

    /// `evaluate(p)` (:72-109): one value per chunk
    pub fn evaluate(&self, p: &DeviceEvals) -> Result<Vec<F>, String> {
        Ok(Self::evaluate_all(&[self], &[(p, false)])?.remove(0).remove(0))
    }

    /// `evaluate_boolean(p)` (:116-131): one value per chunk; a nonzero entry of `p` counts as one
    pub fn evaluate_boolean(&self, p: &DeviceEvals) -> Result<Vec<F>, String> {
        Ok(Self::evaluate_all(&[self], &[(p, true)])?.remove(0).remove(0))
    }

    /// `evaluate` / `evaluate_boolean` (flag) of every column at every point in ONE call — zeta and zeta*omega together, each column
    /// read once.  Result `[column][point][chunk]`.
    pub fn evaluate_all(points: &[&Self], cols: &[(&DeviceEvals, bool)]) -> Result<Vec<Vec<Vec<F>>>, String> {
        let Some(p0) = points.first() else { return Ok(vec![Vec::new(); cols.len()]) };
        if points.iter().any(|p| p.log_n != p0.log_n || p.chunks != p0.chunks) {
            return Err(String::from("the bases must belong to the same domain and max_poly_size"));
        }
        let bases: Vec<*const c_void> = points.iter().map(|p| p.ptr as *const c_void).collect();
        let descs: Vec<zk_eval_column> = cols
            .iter()
            .map(|(e, b)| zk_eval_column { d_evals: e.ptr as *const c_void, len: e.len, boolean: *b as u32, reserved: 0 })
            .collect();
        let per_col = points.len() * p0.chunks;
        let mut out = vec![0u64; 4 * cols.len() * per_col];
        check(unsafe {
            zk_lagrange_evaluate_dev(p0.ctx.0, F::FIELD_ID, bases.as_ptr(), bases.len(), p0.log_n, p0.chunks, descs.as_ptr(), descs.len(),
                                     out.as_mut_ptr())
        })?;
        Ok(out
            .chunks_exact(4 * per_col)
            .map(|c| c.chunks_exact(4 * p0.chunks).map(fields_of::<F>).collect())
            .collect())
    }
}

impl<'c, F: GpuField> Drop for DeviceLagrangeEvals<'c, F> {
    fn drop(&mut self) {
        unsafe { zk_dev_free(self.ctx.0, self.ptr) };
    }
}

/// `to_chunked_polynomial(num_chunks, chunk_size).evaluate_chunks(x)` (utils/src/dense_polynomial.rs:50-69,
/// chunked_polynomial.rs:21-28) of resident coefficient vectors at every point, each vector read once.  Result
/// `[polynomial][point][chunk]`; a polynomial longer than `num_chunks * chunk_size` is the reference's assert and an error here.
pub fn evaluate_chunks_dev<F: GpuField>(
    ctx: &Ctx,
    polys: &[&DeviceEvals],
    num_chunks: usize,
    chunk_size: usize,
    points: &[F],
) -> Result<Vec<Vec<Vec<F>>>, String> {
    let descs: Vec<zk_dev_poly> = polys.iter().map(|p| zk_dev_poly { d_coeffs: p.ptr as *const c_void, len: p.len }).collect();
    let pts: Vec<u64> = points.iter().flat_map(|x| x.to_limbs()).collect();
    let per_poly = points.len() * num_chunks;
    let mut out = vec![0u64; 4 * polys.len() * per_poly];
    check(unsafe {
        zk_poly_evaluate_chunks_dev(ctx.0, F::FIELD_ID, descs.as_ptr(), descs.len(), num_chunks, chunk_size, pts.as_ptr(), points.len(),
                                    out.as_mut_ptr())
    })?;
    if per_poly == 0 {
        return Ok(vec![vec![Vec::new(); points.len()]; polys.len()]);
    }
    Ok(out
        .chunks_exact(4 * per_poly)
        .map(|c| c.chunks_exact(4 * num_chunks).map(fields_of::<F>).collect())
        .collect())
}
