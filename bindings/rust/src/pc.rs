//! `impl PolynomialCommitment for B200MarlinKZG10 / B200SonicKZG10` -- SURVEY.md section 8 row f-4.
//!
//! `Marlin<F, PC, FS>` is generic over `PC: PolynomialCommitment<F, DensePolynomial<F>>` (reference src/lib.rs:64-71) and calls
//! exactly: `setup` (lib.rs:93), `trim` (:115), `commit` (:125,172,193,213), `open_combinations` (:292) and `check_combinations`
//! (:413).  The two types below plug into that parameter: every associated type is ark-poly-commit's own (so proofs, keys and
//! commitments are the stock ones and serialize identically), `setup` and the `check*` family delegate to the upstream CPU code
//! (pairings stay on the host), and `trim` / `commit` / `open*` go to libb2m over the C ABI of include/b2m.h:
//!
//!   trim                                      -> b2m_srs_create (window tables, once) + b2m_trim
//!   commit                                    -> b2m_ck_commit
//!   open_individual_opening_challenges        -> b2m_pc_open
//!   open_combinations_individual_opening_...  -> b2m_ck_open_combinations
//!
//! The trait's single-set `check*` methods stay upstream: on the GPU one set costs one pairing-product latency (17-56 ms,
//! DESIGN.md section 9).  Many sets at once go to the GPU through the inherent `check_combinations_many` (b2m_pc_check_combinations,
//! DESIGN.md section 16); `batch_check` / `check` are its case with one LC per commitment.
//!
//! NOT compiled in this repository (no Rust toolchain in the build image).  Signatures follow ark-poly-commit 0.3.0 as recalled
//! [U]; a maintainer should expect to touch lifetimes / bounds, not the marshalling, which is exercised through the ctypes twin of
//! these calls (tests/test_prover_gpu.py::test_trim_and_open_combinations_level1, ::test_generic_rng_callback).
use crate::{check, ffi, fr_mont_limbs, g1_from_limbs, g1_limbs, Context, Error as B2mError};
use ark_bls12_381::{Bls12_381, Fr, G1Affine};
use ark_ff::{BigInteger256, Field, One};
use ark_poly::univariate::DensePolynomial;
use ark_poly_commit::{
    kzg10, marlin_pc, sonic_pc, BatchLCProof, Evaluations, LabeledCommitment, LabeledPolynomial, LinearCombination, PCCommitterKey,
    PCRandomness, PolynomialCommitment, QuerySet,
};
use ark_std::collections::{BTreeMap, BTreeSet};
use rand_core::RngCore;
use std::os::raw::{c_int, c_void};
use std::sync::Arc;

type P = DensePolynomial<Fr>;
type UpMarlin = marlin_pc::MarlinKZG10<Bls12_381, P>;
type UpSonic = sonic_pc::SonicKZG10<Bls12_381, P>;

// ---- rng: any `RngCore` crosses the ABI as a callback ------------------------------------------------------------------------
unsafe extern "C" fn next_u64_trampoline(state: *mut c_void) -> u64 {
    // `state` points at a `&mut dyn RngCore` that outlives the FFI call
    let rng = &mut *(state as *mut &mut dyn RngCore);
    rng.next_u64()
}
/// `b2m_rng` over a `&mut dyn RngCore`: the library then issues exactly the draws of ark-ff's `F::rand`, in the reference's order.
pub fn callback_rng(rng: &mut &mut dyn RngCore) -> ffi::b2m_rng {
    ffi::b2m_rng { kind: ffi::B2M_RNG_CALLBACK, key: [0u8; 32], word_pos: 0, next_u64: Some(next_u64_trampoline),
                   state: rng as *mut &mut dyn RngCore as *mut c_void }
}

// ---- the device half of a committer key -------------------------------------------------------------------------------------
/// Owns the context, the uploaded SRS (window tables) and the trimmed key; shared by clones of the committer key.
pub struct DeviceKey {
    ctx: Context,
    srs: *mut ffi::b2m_srs,
    ck: *mut ffi::b2m_ck,
    max_bound: i64,
}
unsafe impl Send for DeviceKey {}
unsafe impl Sync for DeviceKey {}
impl Drop for DeviceKey {
    fn drop(&mut self) {
        unsafe {
            ffi::b2m_ck_destroy(self.ck);
            ffi::b2m_srs_destroy(self.srs);
        }
        let _ = &self.ctx; // destroyed last (any order is safe: the library reference-counts parents)
    }
}
impl DeviceKey {
    fn new(pp: &kzg10::UniversalParams<Bls12_381>, sonic: bool, supported_degree: usize, hiding_bound: usize, bounds: &[usize]) -> Result<Arc<Self>, B2mError> {
        let ctx = Context::new(0)?;
        let max_degree = pp.powers_of_g.len() - 1;
        let mut g = Vec::with_capacity(12 * pp.powers_of_g.len());
        pp.powers_of_g.iter().for_each(|p| g1_limbs(p, &mut g));
        // gamma powers the PC will ask for: 0..=hiding_bound+1, and for SonicKZG10 max_degree - bound + 0..=hiding_bound+1
        let mut wanted: BTreeSet<usize> = (0..=hiding_bound + 1).collect();
        if sonic {
            for b in bounds {
                wanted.extend((0..=hiding_bound + 1).map(|i| max_degree - b + i));
            }
        }
        let (mut gam, mut idx) = (Vec::new(), Vec::new());
        for i in wanted {
            if let Some(p) = pp.powers_of_gamma_g.get(&i) {
                idx.push(i as u64);
                g1_limbs(p, &mut gam);
            }
        }
        let mut srs = std::ptr::null_mut();
        check(unsafe {
            ffi::b2m_srs_create(ctx.raw, ffi::B2M_CURVE_BLS12_381, g.as_ptr(), pp.powers_of_g.len(), gam.as_ptr(), idx.as_ptr(), idx.len(), 0, &mut srs)
        })?;
        let b64: Vec<u64> = bounds.iter().map(|b| *b as u64).collect();
        let mut ck = std::ptr::null_mut();
        let pc = if sonic { ffi::B2M_PC_SONIC_KZG10 } else { ffi::B2M_PC_MARLIN_KZG10 };
        let rc = unsafe { ffi::b2m_trim(srs, pc, supported_degree, hiding_bound, b64.as_ptr(), b64.len(), &mut ck) };
        if rc != ffi::B2M_OK {
            unsafe { ffi::b2m_srs_destroy(srs) };
            check(rc)?;
        }
        Ok(Arc::new(DeviceKey { ctx, srs, ck, max_bound: bounds.iter().max().map(|b| *b as i64).unwrap_or(-1) }))
    }
}

/// `PC::CommitterKey`: the upstream key (so `Marlin::index` can keep it in the `IndexProverKey` and CPU code can still read it)
/// plus the shared device half.
#[derive(Clone)]
pub struct CommitterKey<K: Clone> {
    pub upstream: K,
    pub device: Arc<DeviceKey>,
}
impl<K: PCCommitterKey> PCCommitterKey for CommitterKey<K> {
    fn max_degree(&self) -> usize {
        self.upstream.max_degree()
    }
    fn supported_degree(&self) -> usize {
        self.upstream.supported_degree()
    }
}

fn pc_error<E: From<ark_poly_commit::Error>>(e: B2mError) -> E {
    // ark_poly_commit::Error has no "backend" variant; degree / rng errors map one to one, the rest surface as a panic message
    match e {
        B2mError::MissingRng => ark_poly_commit::Error::MissingRng.into(),
        B2mError::DegreeTooLarge => ark_poly_commit::Error::TrimmingDegreeTooLarge.into(),
        other => panic!("libb2m: {:?}", other),
    }
}

// ---- marshalling of labelled polynomials and randomness ------------------------------------------------------------------------
struct Marshalled {
    coeffs: Vec<Vec<u64>>,
    ptrs: Vec<*const u64>,
    lens: Vec<usize>,
    degree_bounds: Vec<i64>,
    hiding_bounds: Vec<i64>,
    labels: Vec<String>,
}
fn marshal_polys<'a>(polys: impl IntoIterator<Item = &'a LabeledPolynomial<Fr, P>>) -> Marshalled {
    let mut m = Marshalled { coeffs: vec![], ptrs: vec![], lens: vec![], degree_bounds: vec![], hiding_bounds: vec![], labels: vec![] };
    for p in polys {
        m.coeffs.push(fr_mont_limbs(&p.polynomial().coeffs));
        m.lens.push(p.polynomial().coeffs.len());
        m.degree_bounds.push(p.degree_bound().map(|d| d as i64).unwrap_or(-1));
        m.hiding_bounds.push(p.hiding_bound().map(|h| h as i64).unwrap_or(-1));
        m.labels.push(p.label().clone());
    }
    m.ptrs = m.coeffs.iter().map(|c| c.as_ptr()).collect();
    m
}
const RAND_STRIDE: usize = 4; // blinding polynomials of hiding bound h have h + 2 coefficients; Marlin uses h = 1
fn fr_from(l: &[u64]) -> Fr {
    let mut a = [0u64; 4];
    a.copy_from_slice(&l[..4]);
    Fr::new(BigInteger256(a))
}
fn rand_poly(limbs: &[u64], hiding: bool, hb: i64) -> kzg10::Randomness<Fr, P> {
    let mut r = kzg10::Randomness::<Fr, P>::empty();
    if hiding {
        let n = (hb + 2) as usize;
        r.blinding_polynomial = P { coeffs: (0..n).map(|k| fr_from(&limbs[4 * k..])).collect() };
    }
    r
}
fn rand_limbs(r: &kzg10::Randomness<Fr, P>, out: &mut Vec<u64>) {
    let c = &r.blinding_polynomial.coeffs;
    for k in 0..RAND_STRIDE {
        out.extend_from_slice(&c.get(k).map(|x| (x.0).0).unwrap_or([0u64; 4]));
    }
}

macro_rules! b200_pc {
    ($name:ident, $up:ty, $upmod:ident, $sonic:expr) => {
        /// Drop-in `PC` parameter for `Marlin<Fr, PC, FS>`; see the module documentation.
        pub struct $name;

        impl PolynomialCommitment<Fr, P> for $name {
            type UniversalParams = <$up as PolynomialCommitment<Fr, P>>::UniversalParams;
            type CommitterKey = CommitterKey<<$up as PolynomialCommitment<Fr, P>>::CommitterKey>;
            type VerifierKey = <$up as PolynomialCommitment<Fr, P>>::VerifierKey;
            type PreparedVerifierKey = <$up as PolynomialCommitment<Fr, P>>::PreparedVerifierKey;
            type Commitment = <$up as PolynomialCommitment<Fr, P>>::Commitment;
            type PreparedCommitment = <$up as PolynomialCommitment<Fr, P>>::PreparedCommitment;
            type Randomness = <$up as PolynomialCommitment<Fr, P>>::Randomness;
            type Proof = <$up as PolynomialCommitment<Fr, P>>::Proof;
            type BatchProof = <$up as PolynomialCommitment<Fr, P>>::BatchProof;
            type Error = <$up as PolynomialCommitment<Fr, P>>::Error;

            /// `KZG10::setup` stays upstream (a trusted setup is not a hot path; b2m_g1_powers / b2m_fixed_base_msm generate test
            /// keys on the GPU when the trapdoor is known).
            fn setup<R: RngCore>(max_degree: usize, num_vars: Option<usize>, rng: &mut R) -> Result<Self::UniversalParams, Self::Error> {
                <$up>::setup(max_degree, num_vars, rng)
            }

            fn trim(pp: &Self::UniversalParams, supported_degree: usize, supported_hiding_bound: usize, enforced_degree_bounds: Option<&[usize]>)
                    -> Result<(Self::CommitterKey, Self::VerifierKey), Self::Error> {
                let (ck, vk) = <$up>::trim(pp, supported_degree, supported_hiding_bound, enforced_degree_bounds)?;
                let device = DeviceKey::new(pp, $sonic, supported_degree, supported_hiding_bound, enforced_degree_bounds.unwrap_or(&[])).map_err(pc_error)?;
                Ok((CommitterKey { upstream: ck, device }, vk))
            }

            fn commit<'a>(ck: &Self::CommitterKey, polynomials: impl IntoIterator<Item = &'a LabeledPolynomial<Fr, P>>, rng: Option<&mut dyn RngCore>)
                          -> Result<(Vec<LabeledCommitment<Self::Commitment>>, Vec<Self::Randomness>), Self::Error>
            where
                P: 'a,
            {
                let m = marshal_polys(polynomials);
                let n = m.lens.len();
                let (mut comm, mut shifted) = (vec![0u64; 12 * n], vec![0u64; 12 * n]);
                let (mut rand, mut srand) = (vec![0u64; 4 * RAND_STRIDE * n], vec![0u64; 4 * RAND_STRIDE * n]);
                let mut dynrng = rng;
                let mut desc = dynrng.as_mut().map(|r| callback_rng(r));
                let rng_ptr = desc.as_mut().map(|d| d as *mut ffi::b2m_rng).unwrap_or(std::ptr::null_mut());
                check(unsafe {
                    ffi::b2m_ck_commit(ck.device.ck, n, m.ptrs.as_ptr(), m.lens.as_ptr(), m.degree_bounds.as_ptr(), m.hiding_bounds.as_ptr(), rng_ptr,
                                       comm.as_mut_ptr(), shifted.as_mut_ptr(), rand.as_mut_ptr(), srand.as_mut_ptr(), RAND_STRIDE)
                })
                .map_err(pc_error)?;
                let mut out_c = Vec::with_capacity(n);
                let mut out_r = Vec::with_capacity(n);
                for i in 0..n {
                    let c = kzg10::Commitment::<Bls12_381>(g1_from_limbs(&comm[12 * i..], false));
                    let hiding = m.hiding_bounds[i] >= 0;
                    let r = rand_poly(&rand[4 * RAND_STRIDE * i..], hiding, m.hiding_bounds[i]);
                    let bounded = m.degree_bounds[i] >= 0;
                    out_c.push(LabeledCommitment::new(m.labels[i].clone(), $upmod::wrap_commitment(c, bounded, &shifted[12 * i..]),
                                                      if bounded { Some(m.degree_bounds[i] as usize) } else { None }));
                    out_r.push($upmod::wrap_randomness(r, bounded, rand_poly(&srand[4 * RAND_STRIDE * i..], hiding && bounded, m.hiding_bounds[i])));
                }
                Ok((out_c, out_r))
            }

            fn open_individual_opening_challenges<'a>(ck: &Self::CommitterKey, labeled_polynomials: impl IntoIterator<Item = &'a LabeledPolynomial<Fr, P>>,
                                                      _commitments: impl IntoIterator<Item = &'a LabeledCommitment<Self::Commitment>>, point: &'a Fr,
                                                      opening_challenges: &dyn Fn(u64) -> Fr, rands: impl IntoIterator<Item = &'a Self::Randomness>,
                                                      _rng: Option<&mut dyn RngCore>)
                                                      -> Result<Self::Proof, Self::Error>
            where
                P: 'a,
                Self::Randomness: 'a,
                Self::Commitment: 'a,
            {
                let m = marshal_polys(labeled_polynomials);
                let xi = power_challenge(opening_challenges);
                let (mut rl, mut srl) = (Vec::new(), Vec::new());
                for r in rands {
                    let (r0, r1) = $upmod::unwrap_randomness(r);
                    rand_limbs(r0, &mut rl);
                    rand_limbs(r1, &mut srl);
                }
                let mut w = [0u64; 12];
                let mut has_rv: c_int = 0;
                let mut rv = [0u64; 4];
                check(unsafe {
                    ffi::b2m_pc_open(ck.device.srs, if $sonic { ffi::B2M_PC_SONIC_KZG10 } else { ffi::B2M_PC_MARLIN_KZG10 }, m.lens.len(), m.ptrs.as_ptr(),
                                     m.lens.as_ptr(), m.degree_bounds.as_ptr(), rl.as_ptr(), srl.as_ptr(), RAND_STRIDE, ck.device.max_bound,
                                     (point.0).0.as_ptr(), (xi.0).0.as_ptr(), w.as_mut_ptr(), &mut has_rv, rv.as_mut_ptr())
                })
                .map_err(pc_error)?;
                Ok(kzg10::Proof { w: g1_from_limbs(&w, false), random_v: if has_rv != 0 { Some(fr_from(&rv)) } else { None } })
            }

            /// All linear combinations are formed, divided and committed on the device (one call per proof).
            fn open_combinations_individual_opening_challenges<'a>(ck: &Self::CommitterKey, lc_s: impl IntoIterator<Item = &'a LinearCombination<Fr>>,
                                                                   polynomials: impl IntoIterator<Item = &'a LabeledPolynomial<Fr, P>>,
                                                                   _commitments: impl IntoIterator<Item = &'a LabeledCommitment<Self::Commitment>>,
                                                                   query_set: &QuerySet<Fr>, opening_challenges: &dyn Fn(u64) -> Fr,
                                                                   rands: impl IntoIterator<Item = &'a Self::Randomness>, _rng: Option<&mut dyn RngCore>)
                                                                   -> Result<BatchLCProof<Fr, P, Self>, Self::Error>
            where
                P: 'a,
                Self::Randomness: 'a,
                Self::Commitment: 'a,
            {
                let m = marshal_polys(polynomials);
                let index_of: BTreeMap<&str, usize> = m.labels.iter().enumerate().map(|(i, l)| (l.as_str(), i)).collect();
                let hiding: Vec<c_int> = m.hiding_bounds.iter().map(|h| (*h >= 0) as c_int).collect();
                let (mut rl, mut srl) = (Vec::new(), Vec::new());
                for r in rands {
                    let (r0, r1) = $upmod::unwrap_randomness(r);
                    rand_limbs(r0, &mut rl);
                    rand_limbs(r1, &mut srl);
                }
                // linear combinations in label order (upstream sorts them: reference src/ahp/mod.rs:219)
                let mut lcs: Vec<&LinearCombination<Fr>> = lc_s.into_iter().collect();
                lcs.sort_by(|a, b| a.label().cmp(b.label()));
                let (mut off, mut lc_poly, mut lc_coeff) = (vec![0usize], Vec::new(), Vec::new());
                for lc in &lcs {
                    for (coeff, term) in lc.iter() {
                        lc_poly.push(if term.is_one() { -1i64 } else { index_of[term.try_into().expect("polynomial label")] as i64 });
                        lc_coeff.extend_from_slice(&(coeff.0).0);
                    }
                    off.push(lc_poly.len());
                }
                let lc_index: BTreeMap<&str, usize> = lcs.iter().enumerate().map(|(i, lc)| (lc.label().as_str(), i)).collect();
                // points in the order of their labels (the QuerySet is a BTreeSet<(String, (String, F))>; upstream groups by point label)
                let mut point_of: BTreeMap<&str, Fr> = BTreeMap::new();
                for (_, (pl, p)) in query_set.iter() {
                    point_of.insert(pl.as_str(), *p);
                }
                let point_index: BTreeMap<&str, usize> = point_of.keys().enumerate().map(|(i, l)| (*l, i)).collect();
                let points: Vec<u64> = point_of.values().flat_map(|p| (p.0).0.to_vec()).collect();
                let (mut q_lc, mut q_pt) = (Vec::new(), Vec::new());
                for (l, (pl, _)) in query_set.iter() {
                    q_lc.push(lc_index[l.as_str()]);
                    q_pt.push(point_index[pl.as_str()]);
                }
                let xi = power_challenge(opening_challenges);
                let np = point_of.len();
                let (mut w, mut has_rv, mut rv) = (vec![0u64; 12 * np], vec![0 as c_int; np], vec![0u64; 4 * np]);
                check(unsafe {
                    ffi::b2m_ck_open_combinations(ck.device.ck, m.lens.len(), m.ptrs.as_ptr(), m.lens.as_ptr(), m.degree_bounds.as_ptr(), hiding.as_ptr(),
                                                  rl.as_ptr(), srl.as_ptr(), RAND_STRIDE, lcs.len(), off.as_ptr(), lc_poly.as_ptr(), lc_coeff.as_ptr(),
                                                  q_lc.len(), q_lc.as_ptr(), q_pt.as_ptr(), np, points.as_ptr(), (xi.0).0.as_ptr(), w.as_mut_ptr(),
                                                  has_rv.as_mut_ptr(), rv.as_mut_ptr())
                })
                .map_err(pc_error)?;
                let proofs: Vec<kzg10::Proof<Bls12_381>> = (0..np)
                    .map(|i| kzg10::Proof { w: g1_from_limbs(&w[12 * i..], false), random_v: if has_rv[i] != 0 { Some(fr_from(&rv[4 * i..])) } else { None } })
                    .collect();
                Ok(BatchLCProof { proof: proofs.into(), evals: None })
            }

            // ---- verification: upstream, on the CPU (pairings) -----------------------------------------------------------------
            fn check_individual_opening_challenges<'a>(vk: &Self::VerifierKey, commitments: impl IntoIterator<Item = &'a LabeledCommitment<Self::Commitment>>,
                                                       point: &'a Fr, values: impl IntoIterator<Item = Fr>, proof: &Self::Proof,
                                                       opening_challenges: &dyn Fn(u64) -> Fr, rng: Option<&mut dyn RngCore>)
                                                       -> Result<bool, Self::Error>
            where
                Self::Commitment: 'a,
            {
                <$up>::check_individual_opening_challenges(vk, commitments, point, values, proof, opening_challenges, rng)
            }
            fn batch_check_individual_opening_challenges<'a, R: RngCore>(vk: &Self::VerifierKey,
                                                                          commitments: impl IntoIterator<Item = &'a LabeledCommitment<Self::Commitment>>,
                                                                          query_set: &QuerySet<Fr>, evaluations: &Evaluations<Fr, Fr>, proof: &Self::BatchProof,
                                                                          opening_challenges: &dyn Fn(u64) -> Fr, rng: &mut R)
                                                                          -> Result<bool, Self::Error>
            where
                Self::Commitment: 'a,
            {
                <$up>::batch_check_individual_opening_challenges(vk, commitments, query_set, evaluations, proof, opening_challenges, rng)
            }
            fn check_combinations_individual_opening_challenges<'a, R: RngCore>(vk: &Self::VerifierKey, lc_s: impl IntoIterator<Item = &'a LinearCombination<Fr>>,
                                                                                 commitments: impl IntoIterator<Item = &'a LabeledCommitment<Self::Commitment>>,
                                                                                 query_set: &QuerySet<Fr>, evaluations: &Evaluations<Fr, Fr>,
                                                                                 proof: &BatchLCProof<Fr, P, Self>, opening_challenges: &dyn Fn(u64) -> Fr, rng: &mut R)
                                                                                 -> Result<bool, Self::Error>
            where
                Self::Commitment: 'a,
            {
                // same Proof / BatchProof types as upstream: re-tag the batch proof and let the stock verifier run
                let up = BatchLCProof::<Fr, P, $up> { proof: proof.proof.clone(), evals: proof.evals.clone() };
                <$up>::check_combinations_individual_opening_challenges(vk, lc_s, commitments, query_set, evaluations, &up, opening_challenges, rng)
            }
        }
    };
}

/// Marlin only ever passes `|pow| opening_challenge.pow(&[pow])` (reference src/lib.rs:290-302): the ABI takes xi itself.
fn power_challenge(opening_challenges: &dyn Fn(u64) -> Fr) -> Fr {
    let xi = opening_challenges(1);
    debug_assert!(opening_challenges(0).is_one() && opening_challenges(2) == xi.square(), "libb2m takes power-structured opening challenges only");
    xi
}

/// MarlinKZG10's commitment / randomness carry an optional shifted half; SonicKZG10 uses the bare KZG10 types.
mod marlin_glue {
    use super::*;
    pub fn wrap_commitment(c: kzg10::Commitment<Bls12_381>, bounded: bool, shifted: &[u64]) -> marlin_pc::Commitment<Bls12_381> {
        marlin_pc::Commitment { comm: c, shifted_comm: if bounded { Some(kzg10::Commitment(g1_from_limbs(shifted, false))) } else { None } }
    }
    pub fn wrap_randomness(r: kzg10::Randomness<Fr, P>, bounded: bool, s: kzg10::Randomness<Fr, P>) -> marlin_pc::Randomness<Fr, P> {
        marlin_pc::Randomness { rand: r, shifted_rand: if bounded { Some(s) } else { None } }
    }
    pub fn unwrap_randomness(r: &marlin_pc::Randomness<Fr, P>) -> (&kzg10::Randomness<Fr, P>, &kzg10::Randomness<Fr, P>) {
        (&r.rand, r.shifted_rand.as_ref().unwrap_or(&EMPTY))
    }
    lazy_static::lazy_static! { pub static ref EMPTY: kzg10::Randomness<Fr, P> = kzg10::Randomness::empty(); }
}
mod sonic_glue {
    use super::*;
    pub fn wrap_commitment(c: kzg10::Commitment<Bls12_381>, _bounded: bool, _shifted: &[u64]) -> kzg10::Commitment<Bls12_381> {
        c
    }
    pub fn wrap_randomness(r: kzg10::Randomness<Fr, P>, _bounded: bool, _s: kzg10::Randomness<Fr, P>) -> kzg10::Randomness<Fr, P> {
        r
    }
    pub fn unwrap_randomness(r: &kzg10::Randomness<Fr, P>) -> (&kzg10::Randomness<Fr, P>, &kzg10::Randomness<Fr, P>) {
        (r, r) // (the shifted slot is ignored for SonicKZG10)
    }
}

b200_pc!(B200MarlinKZG10, UpMarlin, marlin_glue, false);
b200_pc!(B200SonicKZG10, UpSonic, sonic_glue, true);

// ---- batched check_combinations on the GPU ---------------------------------------------------------------------------------
/// One `check_combinations` call's inputs, as the trait method takes them.
pub struct OpeningSet<'a, C> {
    pub lc_s: Vec<&'a LinearCombination<Fr>>,
    pub commitments: Vec<&'a LabeledCommitment<C>>,
    pub query_set: &'a QuerySet<Fr>,
    pub evaluations: &'a Evaluations<Fr, Fr>,
    pub proof: &'a [kzg10::Proof<Bls12_381>],
    pub opening_challenge: Fr,
}

/// A device-side `PC::VerifierKey` (b2m_pc_vk): G2 points prepared once, reused by every batch.
pub struct DeviceVerifierKey {
    _ctx: Context,
    vk: *mut ffi::b2m_pc_vk,
}
impl Drop for DeviceVerifierKey {
    fn drop(&mut self) {
        unsafe { ffi::b2m_pc_vk_destroy(self.vk) }
    }
}

fn g2_uncompressed(p: &<Bls12_381 as ark_ec::PairingEngine>::G2Affine, out: &mut Vec<u8>) {
    use ark_serialize::CanonicalSerialize;
    p.serialize_uncompressed(&mut *out).expect("G2 serialization");
}
fn g1_compressed(p: &G1Affine, out: &mut Vec<u8>) {
    use ark_serialize::CanonicalSerialize;
    p.serialize(&mut *out).expect("G1 serialization");
}
fn fr_canonical(v: &Fr, out: &mut Vec<u8>) {
    use ark_serialize::CanonicalSerialize;
    v.serialize(&mut *out).expect("Fr serialization");
}

/// The arrays of b2m_pc_check_combinations for many sets: commitments, LCs and points in label order (upstream sorts all three).
#[derive(Default)]
struct SetArrays {
    comm_off: Vec<usize>, comms: Vec<u8>, comm_bounds: Vec<i64>, has_shifted: Vec<c_int>, shifted: Vec<u8>,
    lc_off: Vec<usize>, lc_term_off: Vec<usize>, lc_comm: Vec<i64>, lc_coeff: Vec<u64>,
    point_off: Vec<usize>, points: Vec<u64>, w: Vec<u8>, has_rv: Vec<c_int>, rv: Vec<u8>,
    query_off: Vec<usize>, q_lc: Vec<usize>, q_pt: Vec<usize>, evals: Vec<u8>, xi: Vec<u64>,
}

macro_rules! check_many {
    ($name:ident, $comm:ty, $pc:expr, $split:expr) => {
        impl $name {
            /// `PC::VerifierKey` on the device: g, gamma g, h, beta h and the per-bound material of the upstream key.
            pub fn device_verifier_key(ctx: Context, vk: &<Self as PolynomialCommitment<Fr, P>>::VerifierKey) -> Result<DeviceVerifierKey, B2mError> {
                let (g, gamma_g, h, beta_h, max_degree, bounds, bound_points) = $split(vk);
                let (mut gl, mut gg) = (Vec::new(), Vec::new());
                g1_limbs(&g, &mut gl);
                g1_limbs(&gamma_g, &mut gg);
                let (mut hb, mut bhb) = (Vec::new(), Vec::new());
                g2_uncompressed(&h, &mut hb);
                g2_uncompressed(&beta_h, &mut bhb);
                let mut out = std::ptr::null_mut();
                check(unsafe {
                    ffi::b2m_pc_vk_create(ctx.raw, ffi::B2M_CURVE_BLS12_381, $pc, max_degree, gl.as_ptr(), gg.as_ptr(), hb.as_ptr(), bhb.as_ptr(),
                                          bounds.len(), bounds.as_ptr(), bound_points.as_ptr() as *const c_void, &mut out)
                })?;
                Ok(DeviceVerifierKey { _ctx: ctx, vk: out })
            }

            /// `check_combinations` of many independent sets in one GPU batch: Some(true) accepted, Some(false) rejected,
            /// None malformed (an evaluation or random_v not below r cannot occur for ark types; a bounded MarlinKZG10
            /// commitment without its shifted commitment can).  The randomisers come from `rng`.
            pub fn check_combinations_many<R: RngCore>(vk: &DeviceVerifierKey, sets: &[OpeningSet<$comm>], rng: &mut R)
                                                       -> Result<Vec<Option<bool>>, B2mError> {
                let mut a = SetArrays { comm_off: vec![0], lc_off: vec![0], lc_term_off: vec![0], point_off: vec![0], query_off: vec![0], ..Default::default() };
                for s in sets {
                    let mut comms: Vec<&LabeledCommitment<$comm>> = s.commitments.clone();
                    comms.sort_by(|x, y| x.label().cmp(y.label()));
                    let ci: BTreeMap<&str, usize> = comms.iter().enumerate().map(|(i, c)| (c.label().as_str(), i)).collect();
                    for c in &comms {
                        let (comm, shifted) = $name::split_commitment(c.commitment());
                        g1_compressed(&comm, &mut a.comms);
                        a.comm_bounds.push(c.degree_bound().map(|d| d as i64).unwrap_or(-1));
                        a.has_shifted.push(shifted.is_some() as c_int);
                        g1_compressed(&shifted.unwrap_or_default(), &mut a.shifted);
                    }
                    a.comm_off.push(a.comm_bounds.len());
                    let mut lcs = s.lc_s.clone();
                    lcs.sort_by(|x, y| x.label().cmp(y.label()));
                    for lc in &lcs {
                        for (coeff, term) in lc.iter() {
                            a.lc_comm.push(if term.is_one() { -1 } else { ci[term.try_into().expect("polynomial label")] as i64 });
                            a.lc_coeff.extend_from_slice(&(coeff.0).0);
                        }
                        a.lc_term_off.push(a.lc_comm.len());
                    }
                    a.lc_off.push(a.lc_term_off.len() - 1);
                    let li: BTreeMap<&str, usize> = lcs.iter().enumerate().map(|(i, lc)| (lc.label().as_str(), i)).collect();
                    let mut point_of: BTreeMap<&str, Fr> = BTreeMap::new();
                    for (_, (pl, p)) in s.query_set.iter() {
                        point_of.insert(pl.as_str(), *p);
                    }
                    let pi: BTreeMap<&str, usize> = point_of.keys().enumerate().map(|(i, l)| (*l, i)).collect();
                    for (p, proof) in point_of.values().zip(s.proof.iter()) {
                        a.points.extend_from_slice(&(p.0).0);
                        g1_compressed(&proof.w, &mut a.w);
                        a.has_rv.push(proof.random_v.is_some() as c_int);
                        fr_canonical(&proof.random_v.unwrap_or_default(), &mut a.rv);
                    }
                    a.point_off.push(a.has_rv.len());
                    for (l, (pl, p)) in s.query_set.iter() {
                        a.q_lc.push(li[l.as_str()]);
                        a.q_pt.push(pi[pl.as_str()]);
                        fr_canonical(&s.evaluations[&(l.clone(), *p)], &mut a.evals);
                    }
                    a.query_off.push(a.q_lc.len());
                    a.xi.extend_from_slice(&(s.opening_challenge.0).0);
                }
                let mut verdicts = vec![0 as c_int; sets.len()];
                let mut dynrng: &mut dyn RngCore = rng;
                let mut desc = callback_rng(&mut dynrng);
                check(unsafe {
                    ffi::b2m_pc_check_combinations(vk.vk, sets.len(), a.comm_off.as_ptr(), a.comms.as_ptr(), a.comm_bounds.as_ptr(), a.has_shifted.as_ptr(),
                                                   a.shifted.as_ptr(), a.lc_off.as_ptr(), a.lc_term_off.as_ptr(), a.lc_comm.as_ptr(), a.lc_coeff.as_ptr(),
                                                   a.point_off.as_ptr(), a.points.as_ptr(), a.w.as_ptr(), a.has_rv.as_ptr(), a.rv.as_ptr(),
                                                   a.query_off.as_ptr(), a.q_lc.as_ptr(), a.q_pt.as_ptr(), a.evals.as_ptr(), a.xi.as_ptr(), &mut desc,
                                                   verdicts.as_mut_ptr())
                })?;
                Ok(verdicts.into_iter().map(|v| match v { 1 => Some(true), 0 => Some(false), _ => None }).collect())
            }
        }
    };
}

impl B200MarlinKZG10 {
    fn split_commitment(c: &marlin_pc::Commitment<Bls12_381>) -> (G1Affine, Option<G1Affine>) {
        (c.comm.0, c.shifted_comm.map(|s| s.0))
    }
}
impl B200SonicKZG10 {
    fn split_commitment(c: &kzg10::Commitment<Bls12_381>) -> (G1Affine, Option<G1Affine>) {
        (c.0, None)
    }
}
type G2 = <Bls12_381 as ark_ec::PairingEngine>::G2Affine;
fn marlin_vk_parts(vk: &marlin_pc::VerifierKey<Bls12_381>) -> (G1Affine, G1Affine, G2, G2, usize, Vec<u64>, Vec<u64>) {
    let mut bounds = Vec::new();
    let mut points = Vec::new();
    for (d, p) in vk.degree_bounds_and_shift_powers.iter().flatten() {
        bounds.push(*d as u64);
        g1_limbs(p, &mut points);
    }
    (vk.vk.g, vk.vk.gamma_g, vk.vk.h, vk.vk.beta_h, vk.max_degree, bounds, points)
}
fn sonic_vk_parts(vk: &sonic_pc::VerifierKey<Bls12_381>) -> (G1Affine, G1Affine, G2, G2, usize, Vec<u64>, Vec<u8>) {
    let mut bounds = Vec::new();
    let mut points = Vec::new();
    for (d, p) in vk.degree_bounds_and_neg_powers_of_h.iter().flatten() {
        bounds.push(*d as u64);
        g2_uncompressed(p, &mut points);
    }
    (vk.g, vk.gamma_g, vk.h, vk.beta_h, vk.max_degree, bounds, points)
}
check_many!(B200MarlinKZG10, marlin_pc::Commitment<Bls12_381>, ffi::B2M_PC_MARLIN_KZG10, marlin_vk_parts);
check_many!(B200SonicKZG10, kzg10::Commitment<Bls12_381>, ffi::B2M_PC_SONIC_KZG10, sonic_vk_parts);

/// `Marlin::<Fr, B200MarlinKZG10, FS>` -- the reference's own `index` / `prove` / `verify` with the GPU behind `PC`.
pub type GpuMarlin<FS> = ark_marlin::Marlin<Fr, B200MarlinKZG10, FS>;
