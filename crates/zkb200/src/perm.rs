//! The permutation aggregation polynomial z on the device (kimchi/src/circuits/polynomials/permutation.rs:447-574,
//! `ProverIndex::perm_aggreg`; include/zkb200.h, "permutation aggregation polynomial z").
//!
//! [`perm_aggreg_dev`] builds z from the resident witness columns and the resident `permutation_coefficients8` (a cached index's
//! sections 0x30 .. 0x36) and leaves its coefficients resident for the commitment (`zk_msm_dev`), the FFT(8n)
//! (`zk_ntt_dev_oop`) and the quotient (`zk_perm_quotient_dev`).  Only the final-value flag crosses PCIe.  The prover's line
//! (prover.rs:679) then reads (INTEGRATION.md, "z")
//!
//! ```ignore
//! let z_poly = perm_aggreg_dev(&ctx, index.cs.domain.d1, index.cs.zk_rows as usize, &witness_d1, &sigma8, beta, gamma,
//!                              &index.cs.shift, rng)?;
//! ```
use crate::{domain::GpuField, expr::DeviceEvals, ffi::*, srs::Ctx};
use ark_ff::UniformRand;
use ark_poly::Radix2EvaluationDomain as D;
use core::ffi::c_void;
use kimchi::error::ProverError;
use rand_core::{CryptoRng, RngCore};

/// `perm_aggreg` on resident data: `witness` holds the first 7 columns as d1 evaluations, `sigma8` the 7
/// `permutation_coefficients8` over d8 (read at stride 8; any multiple 1 .. 8 of |d1| is accepted), `shifts` is `cs.shift`.
/// The two `F::rand(rng)` values are drawn here, in the reference's order.  Returns z's |d1| coefficients (untrimmed) in a new
/// device buffer, or `ProverError::Permutation("final value")` when z(omega^(n - zk_rows)) != 1, as the reference does.
#[allow(clippy::too_many_arguments)]
pub fn perm_aggreg_dev<F: GpuField, R: RngCore + CryptoRng>(
    ctx: &Ctx,
    domain: D<F>,
    zk_rows: usize,
    witness: &[&DeviceEvals; 7],
    sigma8: &[&DeviceEvals; 7],
    beta: F,
    gamma: F,
    shifts: &[F; 7],
    rng: &mut R,
) -> Result<DeviceEvals, ProverError> {
    let gpu = |_| ProverError::Prover("zkb200: perm_aggreg"); // the library's message: zk_last_error()
    let n = domain.size as usize;
    let rand = [F::rand(rng), F::rand(rng)]; // z[n - zk_rows + 1], z[n - zk_rows + 2] (permutation.rs:556-563)
    let w: Vec<*const c_void> = witness.iter().map(|e| e.ptr as *const c_void).collect();
    let s: Vec<*const c_void> = sigma8.iter().map(|e| e.ptr as *const c_void).collect();
    let sh: Vec<u64> = shifts.iter().flat_map(|x| x.to_limbs()).collect();
    let rl: Vec<u64> = rand.iter().flat_map(|x| x.to_limbs()).collect();
    let (bl, gl) = (beta.to_limbs(), gamma.to_limbs());
    let mut z = core::ptr::null_mut();
    crate::srs::check(unsafe { zk_dev_alloc(ctx.0, 32 * n, &mut z) }).map_err(gpu)?;
    let mut final_is_one = 0;
    let rc = crate::srs::check(unsafe {
        zk_perm_aggreg_dev(ctx.0, F::FIELD_ID, domain.log_size_of_group, zk_rows, w.as_ptr(), s.as_ptr(), sigma8[0].len, bl.as_ptr(),
                           gl.as_ptr(), sh.as_ptr(), rl.as_ptr(), z, &mut final_is_one)
    });
    if rc.is_err() || final_is_one == 0 {
        unsafe { zk_dev_free(ctx.0, z) };
        rc.map_err(gpu)?;
        return Err(ProverError::Permutation("final value"));
    }
    Ok(DeviceEvals { ptr: z, len: n as u64, domain_mult: 0 })
}
