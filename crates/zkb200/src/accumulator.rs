//! The recursion accumulators of poly-commitment/src/utils.rs:204-312 (the bindings' `batch_accumulator_check` and
//! `batch_accumulator_generate`, kimchi-stubs/src/urs_utils.rs:10-101) over the SRS resident on the device.
//!
//! Both functions keep the reference's signatures and panic where it panics (k = 0 with challenges, fewer challenges than
//! accumulators, a remainder, and for the check 2^rounds != |g|), with the library's message.  The challenge polynomials are
//! expanded on the device and the MSMs run over the resident generator table (csrc/accumulator.cu).
use crate::{ffi::*, srs::{check, GpuCurve, GpuSRS}};
use ark_ff::UniformRand;
use core::ffi::c_int;

/// `batch_dlog_accumulator_check(urs, comms, chals)`: true iff every `comms[i]` is `<b_poly_coefficients(chals_i), g>`, batched
/// with the powers of one scalar drawn from `OsRng`, as the reference draws it.
pub fn batch_dlog_accumulator_check<G: GpuCurve>(urs: &GpuSRS<G>, comms: &[G], chals: &[G::ScalarField]) -> bool {
    let r = G::ScalarField::rand(&mut rand::rngs::OsRng);
    let comm_l: Vec<u64> = comms.iter().flat_map(|p| p.limbs()).collect();
    let (chal_l, r_l) = (G::scalar_limbs(chals), G::scalar_limbs(&[r]));
    let mut ok: c_int = 0;
    check(unsafe {
        zk_srs_accumulator_check(urs.dev.0, comm_l.as_ptr(), comms.len(), chal_l.as_ptr(), chals.len(), r_l.as_ptr(), &mut ok,
                                 core::ptr::null_mut())
    })
    .expect("zkb200: batch_dlog_accumulator_check");
    ok != 0
}

/// `batch_dlog_accumulator_generate(urs, num_comms, chals)`: one accumulator per chunk of `chals.len() / num_comms` challenges.
pub fn batch_dlog_accumulator_generate<G: GpuCurve>(urs: &GpuSRS<G>, num_comms: usize, chals: &[G::ScalarField]) -> Vec<G> {
    let chal_l = G::scalar_limbs(chals);
    let cap = if num_comms > 0 && chals.len() >= num_comms { chals.len() / (chals.len() / num_comms) } else { 0 };
    let mut out = vec![0u64; 8 * cap.max(1)];
    let mut got = 0usize;
    check(unsafe { zk_srs_accumulator_generate(urs.dev.0, num_comms, chal_l.as_ptr(), chals.len(), out.as_mut_ptr(), cap, &mut got) })
        .expect("zkb200: batch_dlog_accumulator_generate");
    out[..8 * got].chunks(8).map(G::from_limbs).collect()
}
