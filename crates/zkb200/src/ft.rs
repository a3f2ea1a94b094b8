//! The ft polynomial of Maller's optimisation on the device (kimchi/src/prover.rs:1147-1206; include/zkb200.h, "ft of Maller's
//! optimisation").
//!
//! [`ft_dev`] turns the resident quotient t and the resident `permutation_coefficients8[6]` (sigma_6 over d8, a cached index's
//! section 0x36) into the resident ft, its length and ft(zeta omega); only those 40 bytes cross PCIe.  `blinding_ft` is computed
//! here with the reference's own `PolyComm::chunk_blinding`.  The prover's block then reads (INTEGRATION.md §4)
//!
//! ```ignore
//! let perm_scalar = ConstraintSystem::perm_scalars(&evals, beta, gamma, alphas, zkpm_zeta);
//! let ft = ft_dev(&ctx, index.max_poly_size, index.cs.domain.d1, &[(&sigma6_d8, perm_scalar)], &t, zeta, &t_comm.blinders)?;
//! // ft.coeffs (resident, ft.len coefficients) enters zk_srs_open with blinder ft.blinding_ft; ft.eval1 goes to the proof
//! ```
use crate::{domain::GpuField, expr::DeviceEvals, ffi::*, srs::{check, Ctx}};
use ark_ff::{Field, One, Zero};
use ark_poly::{EvaluationDomain, Radix2EvaluationDomain as D};
use core::ffi::c_void;
use poly_commitment::PolyComm;

/// ft resident on the device: `len` coefficients at `coeffs` (a buffer of max_poly_size elements, zero past `len`, freed on drop).
pub struct DeviceFt<'c, F: GpuField> {
    ctx: &'c Ctx,
    pub coeffs: *mut c_void,
    pub len: usize,
    /// ft(zeta * omega) (prover.rs:1208)
    pub eval1: F,
    /// blinding_f - (zeta^n - 1) t_comm.blinders.chunk_blinding(zeta^max_poly_size), blinding_f = 0 (prover.rs:1192-1203)
    pub blinding_ft: F,
}

impl<'c, F: GpuField> Drop for DeviceFt<'c, F> {
    fn drop(&mut self) {
        unsafe { zk_dev_free(self.ctx.0, self.coeffs) };
    }
}

/// `prover.rs:1147-1206` on resident data: f = interpolate(sum_k c_k * e_k[(len_k / n) i]) over `domain` (kimchi passes ONE term,
/// `(permutation_coefficients8[6], perm_scalar)`, with `perm_scalar` the output of `perm_scalars`), then
/// `ft = f.to_chunked_polynomial(num_chunks, m).linearize(zeta^m) - t.to_chunked_polynomial(7 num_chunks, m).linearize(zeta^m).scale(zeta^n - 1)`.
/// `t` is the quotient's coefficients (resident); `t_blinders` are `t_comm.blinders`.
pub fn ft_dev<'c, F: GpuField>(
    ctx: &'c Ctx,
    max_poly_size: usize,
    domain: D<F>,
    terms: &[(&DeviceEvals, F)],
    t: &DeviceEvals,
    zeta: F,
    t_blinders: &PolyComm<F>,
) -> Result<DeviceFt<'c, F>, String> {
    let descs: Vec<zk_lin_term> = terms
        .iter()
        .map(|(e, c)| zk_lin_term { d_evals: e.ptr as *const c_void, len: e.len, coeff: c.to_limbs() })
        .collect();
    let mut coeffs = core::ptr::null_mut();
    check(unsafe { zk_dev_alloc(ctx.0, 32 * max_poly_size, &mut coeffs) })?;
    let mut out = DeviceFt { ctx, coeffs, len: 0, eval1: F::zero(), blinding_ft: F::zero() };
    let (zl, mut e1) = (zeta.to_limbs(), [0u64; 4]);
    check(unsafe {
        zk_prover_ft_dev(ctx.0, F::FIELD_ID, domain.log_size_of_group, max_poly_size, descs.as_ptr(), descs.len(), t.ptr as *const c_void,
                         t.len as usize, zl.as_ptr(), coeffs, &mut out.len, e1.as_mut_ptr())
    })?;
    out.eval1 = F::from_limbs(e1);
    let zeta_to_srs_len = zeta.pow([max_poly_size as u64]);
    let zeta_to_domain_size = zeta.pow([domain.size]);
    out.blinding_ft = F::zero() - (zeta_to_domain_size - F::one()) * t_blinders.chunk_blinding(zeta_to_srs_len);
    Ok(out)
}
