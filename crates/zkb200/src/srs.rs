//! `GpuSRS<G>`: `poly_commitment::SRS<G>` with the MSMs on the device.  Template: `PairingSRS`, the reference's own delegating
//! implementation (poly-commitment/src/kzg.rs:253-330).  The chunking / padding / sub-sampling policies of `ipa::SRS`
//! (poly-commitment/src/ipa.rs:605-748) are carried out by the library's SRS mirror (csrc/srs.cu), which this type owns.
use crate::{ffi::*, marshal::*};
use ark_ec::{short_weierstrass::{Affine, SWCurveConfig}, AffineRepr};
use ark_ff::{UniformRand, Zero};
use ark_poly::{univariate::DensePolynomial, EvaluationDomain, Evaluations, Radix2EvaluationDomain as D};
use core::ops::Deref;
use poly_commitment::{
    commitment::{BlindedCommitment, CommitmentCurve},
    error::CommitmentError,
    ipa, PolyComm, SRS,
};
use rand_core::{CryptoRng, RngCore};
use std::{collections::HashMap, ffi::CStr, sync::{Arc, Mutex, OnceLock}};

/// One CUDA device + the library's lane pool.  `Send + Sync`: the library serialises per lane and runs independent
/// host-pointer calls concurrently (include/zkb200.h, zk_ctx), which is what the 15 rayon workers of
/// kimchi/src/prover.rs:329-351 need.
pub struct Ctx(pub(crate) *mut zk_ctx);
unsafe impl Send for Ctx {}
unsafe impl Sync for Ctx {}
impl Ctx {
    pub fn new(device: i32) -> Result<Self, String> {
        let mut p = core::ptr::null_mut();
        check(unsafe { zk_ctx_create(device, &mut p) })?;
        Ok(Ctx(p))
    }
    /// Process-wide context on device 0 (`ZKB200_DEVICE` overrides), created on first use.
    pub fn global() -> Arc<Ctx> {
        static G: OnceLock<Arc<Ctx>> = OnceLock::new();
        G.get_or_init(|| {
            let dev = std::env::var("ZKB200_DEVICE").ok().and_then(|s| s.parse().ok()).unwrap_or(0);
            Arc::new(Ctx::new(dev).expect("zkb200: no CUDA device (the library has no CPU fallback)"))
        })
        .clone()
    }
}
impl Drop for Ctx {
    fn drop(&mut self) {
        unsafe { zk_ctx_destroy(self.0) }
    }
}

pub(crate) fn last_error() -> String {
    unsafe { CStr::from_ptr(zk_last_error()) }.to_string_lossy().into_owned()
}
pub(crate) fn check(rc: i32) -> Result<(), String> {
    if rc == ZK_OK { Ok(()) } else { Err(format!("zkb200 error {rc}: {}", last_error())) }
}

/// The two curves the library knows (curves/src/pasta/curves/{pallas,vesta}.rs).
pub trait GpuCurve: CommitmentCurve {
    const CURVE_ID: i32;
    /// field_id of the SCALAR field (ZK_FQ for Pallas, ZK_FP for Vesta)
    const SCALAR_FIELD_ID: i32;
    fn limbs(&self) -> [u64; 8];
    fn from_limbs(l: &[u64]) -> Self;
    fn scalar_limbs(v: &[Self::ScalarField]) -> Vec<u64>;
    fn scalars_from_limbs(l: &[u64]) -> Vec<Self::ScalarField>;
}
macro_rules! impl_gpu_curve {
    ($params:ty, $cid:expr, $fid:expr) => {
        impl GpuCurve for Affine<$params> {
            const CURVE_ID: i32 = $cid;
            const SCALAR_FIELD_ID: i32 = $fid;
            fn limbs(&self) -> [u64; 8] { point_limbs(self) }
            fn from_limbs(l: &[u64]) -> Self { point_of::<$params>(l) }
            fn scalar_limbs(v: &[Self::ScalarField]) -> Vec<u64> { limbs_of(v) }
            fn scalars_from_limbs(l: &[u64]) -> Vec<Self::ScalarField> { fields_of(l) }
        }
    };
}
impl_gpu_curve!(mina_curves::pasta::PallasParameters, ZK_PALLAS, ZK_FQ);
impl_gpu_curve!(mina_curves::pasta::VestaParameters, ZK_VESTA, ZK_FP);

pub(crate) struct SrsHandle(pub(crate) *mut zk_srs);
unsafe impl Send for SrsHandle {}
unsafe impl Sync for SrsHandle {}
impl Drop for SrsHandle {
    fn drop(&mut self) {
        unsafe { zk_srs_destroy(self.0) }
    }
}

/// `ipa::SRS<G>` plus its resident copy on the device.
#[derive(Clone)]
pub struct GpuSRS<G: GpuCurve> {
    /// g, h and everything that never touches an MSM (serde, verification) stay with the reference type
    pub inner: Arc<ipa::SRS<G>>,
    pub(crate) ctx: Arc<Ctx>,
    pub(crate) dev: Arc<SrsHandle>,
    /// Lagrange bases read back from the device, per domain size (the reference's cache is private: ipa.rs:56-75)
    lagrange: Arc<Mutex<HashMap<usize, Arc<Vec<PolyComm<G>>>>>>,
}

impl<G: GpuCurve> core::fmt::Debug for GpuSRS<G> {
    fn fmt(&self, f: &mut core::fmt::Formatter<'_>) -> core::fmt::Result {
        write!(f, "GpuSRS {{ size: {} }}", self.inner.g.len())
    }
}

impl<G: GpuCurve> GpuSRS<G> {
    /// Upload `srs.g` (with its window table) and `srs.h`.
    pub fn from_srs(srs: ipa::SRS<G>, ctx: Arc<Ctx>) -> Result<Self, String> {
        let mut g = Vec::with_capacity(8 * srs.g.len());
        for p in &srs.g {
            g.extend_from_slice(&p.limbs());
        }
        let h = srs.h.limbs();
        let mut dev = core::ptr::null_mut();
        check(unsafe { zk_srs_create(ctx.0, G::CURVE_ID, g.as_ptr(), srs.g.len(), h.as_ptr(), -1, &mut dev) })?;
        Ok(Self { inner: Arc::new(srs), ctx, dev: Arc::new(SrsHandle(dev)), lagrange: Arc::new(Mutex::new(HashMap::new())) })
    }

    /// ipa.rs:780-795 + 1065-1172: the basis is computed ON THE DEVICE (group iFFT of the resident generators, chunked when the
    /// domain is larger than the SRS), registered there for `commit_evaluations_non_hiding`, and read back once for the callers
    /// that want the points (verifier index, `get_lagrange_basis`).
    fn basis(&self, n: usize) -> Arc<Vec<PolyComm<G>>> {
        let mut map = self.lagrange.lock().unwrap();
        if let Some(b) = map.get(&n) {
            return b.clone();
        }
        check(unsafe { zk_srs_lagrange_basis(self.dev.0, n, -1) }).expect("zkb200: lagrange_basis");
        let chunks = unsafe { zk_srs_lagrange_basis_chunks(self.dev.0, n) };
        let mut raw = vec![0u64; 8 * n * chunks];
        check(unsafe { zk_srs_get_lagrange_basis(self.dev.0, n, raw.as_mut_ptr(), n * chunks) }).expect("zkb200: get_lagrange_basis");
        // device layout: chunk-major (chunk c holds the n partial commitments of ipa.rs:1145-1164); PolyComm i = (chunk_c[i])_c
        let basis: Vec<PolyComm<G>> = (0..n)
            .map(|i| PolyComm::new((0..chunks).map(|c| G::from_limbs(&raw[8 * (c * n + i)..8 * (c * n + i) + 8])).collect()))
            .collect();
        let b = Arc::new(basis);
        map.insert(n, b.clone());
        b
    }
}

impl<G: GpuCurve> SRS<G> for GpuSRS<G> {
    fn max_poly_size(&self) -> usize {
        self.inner.g.len()
    }

    fn blinding_commitment(&self) -> G {
        self.inner.h
    }

    /// ipa.rs:605-622 — `zk_srs_mask_custom`; a length mismatch is `CommitmentError::BlindersDontMatch` (error.rs:3-9)
    fn mask_custom(&self, com: PolyComm<G>, blinders: &PolyComm<G::ScalarField>) -> Result<BlindedCommitment<G>, CommitmentError> {
        if com.len() != blinders.len() {
            return Err(CommitmentError::BlindersDontMatch(blinders.len(), com.len()));
        }
        let mut pts = Vec::with_capacity(8 * com.len());
        for p in &com.chunks {
            pts.extend_from_slice(&p.limbs());
        }
        let bl = G::scalar_limbs(&blinders.chunks);
        let mut out = vec![0u64; 8 * com.len()];
        let rc = unsafe { zk_srs_mask_custom(self.dev.0, pts.as_ptr(), com.len(), bl.as_ptr(), blinders.len(), out.as_mut_ptr()) };
        if rc == ZK_ERR_LENGTH {
            return Err(CommitmentError::BlindersDontMatch(blinders.len(), com.len()));
        }
        check(rc).expect("zkb200: mask_custom");
        Ok(BlindedCommitment {
            commitment: PolyComm::new(out.chunks_exact(8).map(G::from_limbs).collect()),
            blinders: blinders.clone(),
        })
    }

    fn mask(&self, comm: PolyComm<G>, rng: &mut (impl RngCore + CryptoRng)) -> BlindedCommitment<G> {
        let blinders = comm.map(|_| G::ScalarField::rand(rng));
        self.mask_custom(comm, &blinders).unwrap()
    }

    /// ipa.rs:638-683 — same chunk-count contract (pbt_srs.rs:21-85): `zk_srs_commit_non_hiding`
    fn commit_non_hiding(&self, plnm: &DensePolynomial<G::ScalarField>, num_chunks: usize) -> PolyComm<G> {
        let n = self.inner.g.len();
        let cap = core::cmp::max(core::cmp::max(plnm.coeffs.len().div_ceil(n), num_chunks), 1);
        let coeffs = G::scalar_limbs(&plnm.coeffs);
        let mut out = vec![0u64; 8 * cap];
        let mut produced = 0usize;
        check(unsafe { zk_srs_commit_non_hiding(self.dev.0, coeffs.as_ptr(), plnm.coeffs.len(), num_chunks, out.as_mut_ptr(), cap, &mut produced) })
            .expect("zkb200: commit_non_hiding");
        PolyComm::new(out[..8 * produced].chunks_exact(8).map(G::from_limbs).collect())
    }

    fn commit(&self, plnm: &DensePolynomial<G::ScalarField>, num_chunks: usize, rng: &mut (impl RngCore + CryptoRng)) -> BlindedCommitment<G> {
        self.mask(self.commit_non_hiding(plnm, num_chunks), rng)
    }

    fn commit_custom(&self, plnm: &DensePolynomial<G::ScalarField>, num_chunks: usize, blinders: &PolyComm<G::ScalarField>)
        -> Result<BlindedCommitment<G>, CommitmentError> {
        self.mask_custom(self.commit_non_hiding(plnm, num_chunks), blinders)
    }

    /// ipa.rs:706-728 + commitment.rs:350-394 — the sub-sampling and the per-chunk MSMs run in the library against the resident basis
    fn commit_evaluations_non_hiding(&self, domain: D<G::ScalarField>, plnm: &Evaluations<G::ScalarField, D<G::ScalarField>>) -> PolyComm<G> {
        let n = domain.size();
        if n > plnm.domain().size() {
            panic!("desired commitment domain size ({}) greater than evaluations' domain size ({}):", domain.size, plnm.domain().size);
        }
        check(unsafe { zk_srs_lagrange_basis(self.dev.0, n, -1) }).expect("zkb200: lagrange_basis");   // no-op once registered
        let chunks = unsafe { zk_srs_lagrange_basis_chunks(self.dev.0, n) };
        let evals = G::scalar_limbs(&plnm.evals);
        let mut out = vec![0u64; 8 * chunks];
        check(unsafe { zk_srs_commit_evaluations_non_hiding(self.dev.0, n, evals.as_ptr(), plnm.evals.len(), out.as_mut_ptr()) })
            .expect("zkb200: commit_evaluations_non_hiding");
        PolyComm::new(out.chunks_exact(8).map(G::from_limbs).collect())
    }

    fn commit_evaluations(&self, domain: D<G::ScalarField>, plnm: &Evaluations<G::ScalarField, D<G::ScalarField>>,
                          rng: &mut (impl RngCore + CryptoRng)) -> BlindedCommitment<G> {
        self.mask(self.commit_evaluations_non_hiding(domain, plnm), rng)
    }

    fn commit_evaluations_custom(&self, domain: D<G::ScalarField>, plnm: &Evaluations<G::ScalarField, D<G::ScalarField>>,
                                 blinders: &PolyComm<G::ScalarField>) -> Result<BlindedCommitment<G>, CommitmentError> {
        self.mask_custom(self.commit_evaluations_non_hiding(domain, plnm), blinders)
    }

    /// ipa.rs:751-778 — `zk_srs_generate`: g and h are hashed to the curve on the device and stay resident in the handle that call
    /// returns; `inner` is built from the host copies, so nothing is uploaded again
    fn create(depth: usize) -> Self {
        let ctx = Ctx::global();
        let mut g = vec![0u64; 8 * depth];
        let mut h = [0u64; 8];
        let mut dev = core::ptr::null_mut();
        check(unsafe { zk_srs_generate(ctx.0, G::CURVE_ID, depth, -1, g.as_mut_ptr(), h.as_mut_ptr(), &mut dev) }).expect("zkb200: SRS::create");
        let inner = ipa::SRS::new(g.chunks_exact(8).map(G::from_limbs).collect(), G::from_limbs(&h));
        Self { inner: Arc::new(inner), ctx, dev: Arc::new(SrsHandle(dev)), lagrange: Arc::new(Mutex::new(HashMap::new())) }
    }

    fn get_lagrange_basis(&self, domain: D<G::ScalarField>) -> impl Deref<Target = Vec<PolyComm<G>>> + '_ {
        self.basis(domain.size())
    }

    fn get_lagrange_basis_from_domain_size(&self, domain_size: usize) -> impl Deref<Target = Vec<PolyComm<G>>> + '_ {
        self.basis(domain_size)
    }

    fn size(&self) -> usize {
        self.inner.g.len()
    }
}

// keep the identity check of marshal.rs honest for both curves
#[allow(dead_code)]
fn _identity_is_all_zero<P: SWCurveConfig>()
where
    P::BaseField: Limbs4,
{
    debug_assert!(point_limbs(&Affine::<P>::zero()).iter().all(|w| *w == 0));
    let _ = <P::BaseField as Zero>::zero();
}
