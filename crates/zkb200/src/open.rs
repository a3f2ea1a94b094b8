//! `GpuOpeningProof<G, FULL_ROUNDS>`: `poly_commitment::OpenProof` (poly-commitment/src/lib.rs:254-298) with `open` on the device.
//! The struct IS `ipa::OpeningProof` (same fields, same serde: ipa.rs:1175-1191), so the unmodified verifier, the OCaml / wasm
//! bindings and every serialised proof keep working.
//!
//! `open` = one `zk_srs_open` call (csrc/open.cu): combine_polys, b_init, the folding rounds with h and U inside the MSMs, delta,
//! z1, z2 in the library; the sponge and the group map — generic parameters of the reference — stay here, behind three callbacks.
use crate::{ffi::*, srs::{check, GpuCurve, GpuSRS}};
use ark_ec::AffineRepr;
use ark_ff::{Field, One, PrimeField, UniformRand};
use ark_poly::EvaluationDomain;
use core::ffi::{c_int, c_uint, c_void};
use groupmap::GroupMap;
use mina_poseidon::{sponge::ScalarChallenge, FqSponge};
use poly_commitment::{
    commitment::{shift_scalar, squeeze_prechallenge, BatchEvaluationProof, CommitmentCurve, EndoCurve},
    ipa::{endos, OpeningProof},
    utils::DensePolynomialOrEvaluations,
    OpenProof, PolyComm,
};
use rand_core::{CryptoRng, RngCore};
use serde::{Deserialize, Serialize};

/// Newtype over the reference's proof: identical wire form.
#[derive(Clone, Debug, Serialize, Deserialize, PartialEq, Eq)]
#[repr(transparent)]
#[serde(transparent)]
#[serde(bound = "G: ark_serialize::CanonicalDeserialize + ark_serialize::CanonicalSerialize")]
pub struct GpuOpeningProof<G: AffineRepr, const FULL_ROUNDS: usize>(pub OpeningProof<G, FULL_ROUNDS>);

/// What the three callbacks share: the caller's sponge (the one of `open`, or one batch element's of `verify`), its group map and
/// the curve's endo coefficient.
struct Transcript<'a, G: GpuCurve, S, const FULL_ROUNDS: usize> {
    sponge: &'a mut S,
    group_map: &'a G::Map,
    endo_r: G::ScalarField,
}

unsafe extern "C" fn cb_u_base<G, S, const FULL_ROUNDS: usize>(user: *mut c_void, cip: *const u64, out_u_xy: *mut u64) -> c_int
where
    G: GpuCurve + EndoCurve,
    G::BaseField: PrimeField,
    S: FqSponge<G::BaseField, G, G::ScalarField, FULL_ROUNDS>,
{
    let t = &mut *(user as *mut Transcript<G, S, FULL_ROUNDS>);
    let cip = G::scalars_from_limbs(core::slice::from_raw_parts(cip, 4))[0];
    // ipa.rs:898-910
    t.sponge.absorb_fr(&[shift_scalar::<G>(cip)]);
    let (x, y) = t.group_map.to_group(t.sponge.challenge_fq());
    let u = G::of_coordinates(x, y);
    core::slice::from_raw_parts_mut(out_u_xy, 8).copy_from_slice(&u.limbs());
    0
}

unsafe extern "C" fn cb_round<G, S, const FULL_ROUNDS: usize>(user: *mut c_void, _round: c_uint, l_xy: *const u64, r_xy: *const u64, out_u: *mut u64) -> c_int
where
    G: GpuCurve + EndoCurve,
    G::BaseField: PrimeField,
    S: FqSponge<G::BaseField, G, G::ScalarField, FULL_ROUNDS>,
{
    let t = &mut *(user as *mut Transcript<G, S, FULL_ROUNDS>);
    let l = G::from_limbs(core::slice::from_raw_parts(l_xy, 8));
    let r = G::from_limbs(core::slice::from_raw_parts(r_xy, 8));
    // ipa.rs:962-970
    t.sponge.absorb_g(&[l]);
    t.sponge.absorb_g(&[r]);
    let u = squeeze_prechallenge(&mut *t.sponge).to_field(&t.endo_r);
    core::slice::from_raw_parts_mut(out_u, 4).copy_from_slice(&G::scalar_limbs(&[u]));
    0
}

unsafe extern "C" fn cb_final<G, S, const FULL_ROUNDS: usize>(user: *mut c_void, delta_xy: *const u64, out_c: *mut u64) -> c_int
where
    G: GpuCurve + EndoCurve,
    G::BaseField: PrimeField,
    S: FqSponge<G::BaseField, G, G::ScalarField, FULL_ROUNDS>,
{
    let t = &mut *(user as *mut Transcript<G, S, FULL_ROUNDS>);
    let delta = G::from_limbs(core::slice::from_raw_parts(delta_xy, 8));
    // ipa.rs:1040-1041
    t.sponge.absorb_g(&[delta]);
    let c = ScalarChallenge::new(t.sponge.challenge()).to_field(&t.endo_r);
    core::slice::from_raw_parts_mut(out_c, 4).copy_from_slice(&G::scalar_limbs(&[c]));
    0
}

impl<BaseField, G, const FULL_ROUNDS: usize> OpenProof<G, FULL_ROUNDS> for GpuOpeningProof<G, FULL_ROUNDS>
where
    BaseField: PrimeField,
    G: AffineRepr<BaseField = BaseField> + GpuCurve + EndoCurve,
{
    type SRS = GpuSRS<G>;

    fn open<EFqSponge, RNG, D: EvaluationDomain<<G as AffineRepr>::ScalarField>>(
        srs: &Self::SRS,
        group_map: &<G as CommitmentCurve>::Map,
        plnms: &[(DensePolynomialOrEvaluations<'_, G::ScalarField, D>, PolyComm<G::ScalarField>)],
        elm: &[<G as AffineRepr>::ScalarField],
        polyscale: <G as AffineRepr>::ScalarField,
        evalscale: <G as AffineRepr>::ScalarField,
        sponge: EFqSponge,
        rng: &mut RNG,
    ) -> Self
    where
        EFqSponge: Clone + FqSponge<<G as AffineRepr>::BaseField, G, <G as AffineRepr>::ScalarField, FULL_ROUNDS>,
        RNG: RngCore + CryptoRng,
    {
        let (_endo_q, endo_r) = endos::<G>();
        let n = srs.inner.g.len();
        let rounds = n.next_power_of_two().trailing_zeros() as usize;   // math::ceil_log2(self.g.len()), ipa.rs:844

        // plnms -> zk_open_poly[] (limb copies live until the call returns)
        let mut data: Vec<Vec<u64>> = Vec::with_capacity(plnms.len());
        let mut blinders: Vec<Vec<u64>> = Vec::with_capacity(plnms.len());
        let mut domains: Vec<usize> = Vec::with_capacity(plnms.len());
        for (p, comm) in plnms {
            match p {
                DensePolynomialOrEvaluations::DensePolynomial(d) => {
                    data.push(G::scalar_limbs(&d.coeffs));
                    domains.push(0);
                }
                DensePolynomialOrEvaluations::Evaluations(e, sub_domain) => {
                    data.push(G::scalar_limbs(&e.evals));
                    domains.push(sub_domain.size());
                }
            }
            blinders.push(G::scalar_limbs(&comm.chunks));
        }
        let polys: Vec<zk_open_poly> = (0..plnms.len())
            .map(|i| zk_open_poly {
                data: data[i].as_ptr(),
                len: data[i].len() / 4,
                domain_size: domains[i],
                blinders: blinders[i].as_ptr(),
                n_blinders: blinders[i].len() / 4,
            })
            .collect();

        // the random scalars in the order SRS::open draws them: rand_l, rand_r per round (ipa.rs:936-937), then d, r_delta (:1027-1028)
        let draws: Vec<G::ScalarField> = (0..2 * rounds + 2).map(|_| G::ScalarField::rand(rng)).collect();
        let draws = G::scalar_limbs(&draws);

        let mut sponge = sponge;
        let mut t = Transcript::<G, EFqSponge, FULL_ROUNDS> { sponge: &mut sponge, group_map, endo_r };
        let tr = zk_open_transcript {
            user: (&mut t as *mut Transcript<G, EFqSponge, FULL_ROUNDS>).cast(),
            u_base: cb_u_base::<G, EFqSponge, FULL_ROUNDS>,
            round: cb_round::<G, EFqSponge, FULL_ROUNDS>,
            final_challenge: cb_final::<G, EFqSponge, FULL_ROUNDS>,
        };
        let elm_l = G::scalar_limbs(elm);
        let (ps, es) = (G::scalar_limbs(&[polyscale]), G::scalar_limbs(&[evalscale]));
        let mut lr = vec![0u64; 16 * rounds.max(1)];
        let (mut delta, mut sg, mut z1, mut z2) = ([0u64; 8], [0u64; 8], [0u64; 4], [0u64; 4]);
        let mut got_rounds = 0usize;
        check(unsafe {
            zk_srs_open(srs.dev.0, polys.as_ptr(), polys.len(), elm_l.as_ptr(), elm.len(), ps.as_ptr(), es.as_ptr(), draws.as_ptr(),
                        2 * rounds + 2, &tr, lr.as_mut_ptr(), rounds, &mut got_rounds, delta.as_mut_ptr(), z1.as_mut_ptr(), z2.as_mut_ptr(),
                        sg.as_mut_ptr())
        })
        .expect("zkb200: open");
        assert_eq!(got_rounds, rounds, "IPA commitment folding must produce single elements after log rounds");
        let _ = G::ScalarField::one().inverse();
        GpuOpeningProof(OpeningProof {
            lr: lr[..16 * rounds].chunks_exact(16).map(|c| (G::from_limbs(&c[..8]), G::from_limbs(&c[8..]))).collect(),
            delta: G::from_limbs(&delta),
            z1: G::scalars_from_limbs(&z1)[0],
            z2: G::scalars_from_limbs(&z2)[0],
            sg: G::from_limbs(&sg),
        })
    }

    /// `verify` = one `zk_srs_verify` call (csrc/verify.cu): SRS::verify (ipa.rs:301-502) with the challenge polynomials of the
    /// whole batch expanded on the device and both MSMs there; each element's sponge stays here, behind the same three callbacks as
    /// `open`, called proof by proof in the reference's order.
    fn verify<EFqSponge, RNG>(
        srs: &Self::SRS,
        group_map: &G::Map,
        batch: &mut [BatchEvaluationProof<G, EFqSponge, Self, FULL_ROUNDS>],
        rng: &mut RNG,
    ) -> bool
    where
        EFqSponge: FqSponge<G::BaseField, G, G::ScalarField, FULL_ROUNDS>,
        RNG: RngCore + CryptoRng,
    {
        let (_endo_q, endo_r) = endos::<G>();
        // the reference's draws, in its order (ipa.rs:357-358)
        let rand_base = G::ScalarField::rand(rng);
        let sg_rand_base = G::ScalarField::rand(rng);
        let rng_l = G::scalar_limbs(&[rand_base, sg_rand_base]);

        // per element: limb copies of the proof and its evaluations (they live until the call returns) and a transcript over its sponge
        struct Limbs {
            lr: Vec<u64>,
            delta: [u64; 8],
            sg: [u64; 8],
            z: Vec<u64>,
            elm: Vec<u64>,
            scales: Vec<u64>,
            comm: Vec<u64>,
            chunks: Vec<usize>,
            cip: Vec<u64>,
        }
        let mut limbs: Vec<Limbs> = Vec::with_capacity(batch.len());
        let mut ts: Vec<Transcript<G, EFqSponge, FULL_ROUNDS>> = Vec::with_capacity(batch.len());
        for BatchEvaluationProof { sponge, evaluation_points, polyscale, evalscale, evaluations, opening, combined_inner_product } in batch.iter_mut() {
            let op = &opening.0;
            limbs.push(Limbs {
                lr: op.lr.iter().flat_map(|(l, r)| l.limbs().into_iter().chain(r.limbs())).collect(),
                delta: op.delta.limbs(),
                sg: op.sg.limbs(),
                z: G::scalar_limbs(&[op.z1, op.z2]),
                elm: G::scalar_limbs(evaluation_points),
                scales: G::scalar_limbs(&[*polyscale, *evalscale]),
                comm: evaluations.iter().flat_map(|e| e.commitment.chunks.iter().flat_map(|c| c.limbs())).collect(),
                chunks: evaluations.iter().map(|e| e.commitment.chunks.len()).collect(),
                cip: G::scalar_limbs(&[*combined_inner_product]),
            });
            ts.push(Transcript { sponge, group_map, endo_r });
        }
        let trs: Vec<zk_open_transcript> = ts
            .iter_mut()
            .map(|t| zk_open_transcript {
                user: (t as *mut Transcript<G, EFqSponge, FULL_ROUNDS>).cast(),
                u_base: cb_u_base::<G, EFqSponge, FULL_ROUNDS>,
                round: cb_round::<G, EFqSponge, FULL_ROUNDS>,
                final_challenge: cb_final::<G, EFqSponge, FULL_ROUNDS>,
            })
            .collect();
        let descs: Vec<zk_verify_proof> = limbs
            .iter()
            .zip(trs.iter())
            .map(|(l, tr)| zk_verify_proof {
                lr_xy: l.lr.as_ptr(),
                n_rounds: l.lr.len() / 16,
                delta_xy: l.delta.as_ptr(),
                z1: l.z.as_ptr(),
                z2: l.z[4..].as_ptr(),
                sg_xy: l.sg.as_ptr(),
                elm: l.elm.as_ptr(),
                n_elm: l.elm.len() / 4,
                polyscale: l.scales.as_ptr(),
                evalscale: l.scales[4..].as_ptr(),
                comm_xy: l.comm.as_ptr(),
                comm_chunks: l.chunks.as_ptr(),
                n_comms: l.chunks.len(),
                combined_inner_product: l.cip.as_ptr(),
                transcript: tr,
            })
            .collect();
        let mut ok: c_int = 0;
        check(unsafe { zk_srs_verify(srs.dev.0, descs.as_ptr(), descs.len(), rng_l.as_ptr(), &mut ok, core::ptr::null_mut()) })
            .expect("zkb200: verify");
        ok != 0
    }
}
