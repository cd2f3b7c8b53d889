//! Replays a kit made by tools/make_replay_kit.py through the real arkworks Marlin and diffs bytes.  See Cargo.toml.
//! The kit's meta.json names its curve: BLS12-381 or BLS12-377 (ark-bn254 is not a dependency of the reference).

// One module per curve, identical but for the curve crate, its pairing engine and the curve id of the SRS file.
macro_rules! curve_replay {
    ($module:ident, $krate:ident, $engine:ident, $curve_id:expr) => {
        mod $module {
            use $krate::{$engine as E, Fr, G1Affine, G2Affine};
            use ark_ff::{to_bytes, Field, PrimeField};
            use ark_marlin::{Marlin, SimpleHashFiatShamirRng};
            use ark_poly::univariate::DensePolynomial;
            use ark_poly_commit::{kzg10::UniversalParams, marlin_pc::MarlinKZG10, sonic_pc::SonicKZG10, PolynomialCommitment};
            use ark_relations::{lc, r1cs::{ConstraintSynthesizer, ConstraintSystemRef, SynthesisError}};
            use ark_serialize::{CanonicalDeserialize, CanonicalSerialize};
            use blake2::Blake2s;
            use rand::SeedableRng;
            use rand_chacha::{ChaCha12Rng, ChaChaRng};
            use std::collections::BTreeMap;
            use std::io::Read;

            type FS = SimpleHashFiatShamirRng<Blake2s, ChaChaRng>;

            /// The reference bench's circuit (benches/bench.rs:25-67), with the witness values of the kit.
            #[derive(Copy, Clone)]
            struct DummyCircuit { a: Option<Fr>, b: Option<Fr>, num_variables: usize, num_constraints: usize }
            impl ConstraintSynthesizer<Fr> for DummyCircuit {
                fn generate_constraints(self, cs: ConstraintSystemRef<Fr>) -> Result<(), SynthesisError> {
                    let a = cs.new_witness_variable(|| self.a.ok_or(SynthesisError::AssignmentMissing))?;
                    let b = cs.new_witness_variable(|| self.b.ok_or(SynthesisError::AssignmentMissing))?;
                    let c = cs.new_input_variable(|| Ok(self.a.ok_or(SynthesisError::AssignmentMissing)? * self.b.ok_or(SynthesisError::AssignmentMissing)?))?;
                    for _ in 0..(self.num_variables - 3) {
                        let _ = cs.new_witness_variable(|| self.a.ok_or(SynthesisError::AssignmentMissing))?;
                    }
                    for _ in 0..self.num_constraints - 1 {
                        cs.enforce_constraint(lc!() + a, lc!() + b, lc!() + c)?;
                    }
                    cs.enforce_constraint(lc!(), lc!(), lc!())?;
                    Ok(())
                }
            }

            fn read_u64(r: &mut impl Read) -> u64 { let mut b = [0u8; 8]; r.read_exact(&mut b).unwrap(); u64::from_le_bytes(b) }

            /// marlin_b200/srsfile.py layout: tag, curve id, then the public fields of kzg10::UniversalParams, each `serialize_uncompressed`.
            fn load_srs(path: &str) -> UniversalParams<E> {
                let mut f = std::io::BufReader::new(std::fs::File::open(path).expect("srs file"));
                let mut tag = [0u8; 8];
                f.read_exact(&mut tag).unwrap();
                assert_eq!(&tag, b"B2MSRS01");
                assert_eq!(read_u64(&mut f), $curve_id, "the kit's curve id");
                let n = read_u64(&mut f) as usize;
                let powers_of_g: Vec<G1Affine> = (0..n).map(|_| G1Affine::deserialize_unchecked(&mut f).unwrap()).collect();
                let mut powers_of_gamma_g = BTreeMap::new();
                for _ in 0..read_u64(&mut f) { let k = read_u64(&mut f) as usize; powers_of_gamma_g.insert(k, G1Affine::deserialize_unchecked(&mut f).unwrap()); }
                let h = G2Affine::deserialize_unchecked(&mut f).unwrap();
                let beta_h = G2Affine::deserialize_unchecked(&mut f).unwrap();
                let mut neg_powers_of_h = BTreeMap::new();
                for _ in 0..read_u64(&mut f) { let k = read_u64(&mut f) as usize; neg_powers_of_h.insert(k, G2Affine::deserialize_unchecked(&mut f).unwrap()); }
                UniversalParams { powers_of_g, powers_of_gamma_g, h, beta_h, neg_powers_of_h, prepared_h: h.into(), prepared_beta_h: beta_h.into() }
            }

            fn fr_from_dec(s: &str) -> Fr { Fr::from_str(s).ok().expect("decimal field element") }

            fn replay<PC>(dir: &str, meta: &serde_json::Value, srs: &PC::UniversalParams) -> bool
            where PC: PolynomialCommitment<Fr, DensePolynomial<Fr>> {
                let scheme = meta["pc"].as_str().unwrap();
                let circ = DummyCircuit { a: Some(fr_from_dec(meta["a"].as_str().unwrap())), b: Some(fr_from_dec(meta["b"].as_str().unwrap())),
                                          num_variables: meta["num_variables"].as_u64().unwrap() as usize, num_constraints: meta["num_constraints"].as_u64().unwrap() as usize };
                let (pk, vk) = Marlin::<Fr, PC, FS>::index(srs, circ).expect("index");
                let want_vk = std::fs::read(format!("{}/{}_index_vk_tobytes.bin", dir, scheme)).unwrap();
                let got_vk = to_bytes![vk].unwrap();
                let mut seed = [0u8; 32];
                seed.copy_from_slice(&hex::decode(meta["zk_seed_hex"].as_str().unwrap()).unwrap());
                let mut zk = ChaCha12Rng::from_seed(seed);
                let proof = Marlin::<Fr, PC, FS>::prove(&pk, circ, &mut zk).expect("prove");
                let mut got_proof = Vec::new();
                proof.serialize(&mut got_proof).unwrap();
                let want_proof = std::fs::read(format!("{}/{}_proof.bin", dir, scheme)).unwrap();
                let c = circ.a.unwrap() * circ.b.unwrap();
                let ok_verify = Marlin::<Fr, PC, FS>::verify(&vk, &[c], &proof, &mut ChaCha12Rng::from_seed([7u8; 32])).expect("verify");
                let want_pos = meta["zk_word_pos_after"][scheme].as_u64().unwrap() as u128;
                println!("{}: index_vk {} | proof {} | rng position {} | verify {}", scheme,
                         if got_vk == want_vk { "MATCH" } else { "DIFFER" }, if got_proof == want_proof { "MATCH" } else { "DIFFER" },
                         if zk.get_word_pos() == want_pos { "MATCH" } else { "DIFFER" }, ok_verify);
                // the GPU-made proof must also be accepted by the real verifier
                let gpu_proof = ark_marlin::Proof::<Fr, PC>::deserialize(&want_proof[..]).expect("deserialize the kit's proof");
                let ok_gpu = Marlin::<Fr, PC, FS>::verify(&vk, &[c], &gpu_proof, &mut ChaCha12Rng::from_seed([7u8; 32])).unwrap_or(false);
                println!("{}: the kit's proof is accepted by ark-marlin: {}", scheme, ok_gpu);
                let ok_keys = replay_key_files::<PC>(dir, scheme, &pk, &vk, circ, &c);
                got_vk == want_vk && got_proof == want_proof && zk.get_word_pos() == want_pos && ok_verify && ok_gpu && ok_keys
            }

            // Index key files (IndexProverKey::save / save_verifier_key, compressed form; marlin_b200/keyfile.py): each file must
            // `deserialize` into the real arkworks type, serialize back to the same bytes, and equal this run's own `Marlin::index`
            // output byte for byte -- the check that pins the recalled layouts.  A kit without the files skips the check.
            fn replay_key_files<PC>(dir: &str, scheme: &str, pk: &ark_marlin::IndexProverKey<Fr, PC>, vk: &ark_marlin::IndexVerifierKey<Fr, PC>,
                                    circ: DummyCircuit, c: &Fr) -> bool
            where PC: PolynomialCommitment<Fr, DensePolynomial<Fr>> {
                let pk_path = format!("{}/{}_index_pk.bin", dir, scheme);
                let vk_path = format!("{}/{}_index_vk.bin", dir, scheme);
                let (file_pk, file_vk) = match (std::fs::read(&pk_path), std::fs::read(&vk_path)) {
                    (Ok(p), Ok(v)) => (p, v),
                    _ => {
                        println!("{}: no index key files in the kit, skipped", scheme);
                        return true;
                    }
                };
                let mut own_pk = Vec::new();
                pk.serialize(&mut own_pk).unwrap();
                let mut own_vk = Vec::new();
                vk.serialize(&mut own_vk).unwrap();
                let read_pk = ark_marlin::IndexProverKey::<Fr, PC>::deserialize(&file_pk[..]);
                let read_vk = ark_marlin::IndexVerifierKey::<Fr, PC>::deserialize(&file_vk[..]);
                let round_pk = read_pk.as_ref().map(|k| { let mut b = Vec::new(); k.serialize(&mut b).unwrap(); b == file_pk }).unwrap_or(false);
                let round_vk = read_vk.as_ref().map(|k| { let mut b = Vec::new(); k.serialize(&mut b).unwrap(); b == file_vk }).unwrap_or(false);
                let first_diff = |a: &[u8], b: &[u8]| a.iter().zip(b).position(|(x, y)| x != y).unwrap_or(a.len().min(b.len()));
                println!("{}: index_pk file deserializes {} | round trip {} | equals Marlin::index {} (first difference at byte {} of {} / {})",
                         scheme, read_pk.is_ok(), round_pk, own_pk == file_pk, first_diff(&own_pk, &file_pk), own_pk.len(), file_pk.len());
                println!("{}: index_vk file deserializes {} | round trip {} | equals Marlin::index {} (first difference at byte {} of {} / {})",
                         scheme, read_vk.is_ok(), round_vk, own_vk == file_vk, first_diff(&own_vk, &file_vk), own_vk.len(), file_vk.len());
                // the deserialized verifier key verifies a proof made with the deserialized prover key
                let ok_use = match (read_pk, read_vk) {
                    (Ok(rpk), Ok(rvk)) => {
                        let mut zk = ChaCha12Rng::from_seed([9u8; 32]);
                        let proof = Marlin::<Fr, PC, FS>::prove(&rpk, circ, &mut zk).expect("prove with the file's key");
                        Marlin::<Fr, PC, FS>::verify(&rvk, &[*c], &proof, &mut ChaCha12Rng::from_seed([7u8; 32])).unwrap_or(false)
                    }
                    _ => false,
                };
                println!("{}: a proof made with the file's prover key verifies under the file's verifier key: {}", scheme, ok_use);
                round_pk && round_vk && own_pk == file_pk && own_vk == file_vk && ok_use
            }

            pub fn run(dir: &str, meta: &serde_json::Value) -> bool {
                let srs = load_srs(&format!("{}/srs.bin", dir));
                let a = replay::<MarlinKZG10<E, DensePolynomial<Fr>>>(dir, meta, &srs);
                let b = replay::<SonicKZG10<E, DensePolynomial<Fr>>>(dir, meta, &srs);
                a && b
            }
        }
    };
}

curve_replay!(bls12_381, ark_bls12_381, Bls12_381, 0);
curve_replay!(bls12_377, ark_bls12_377, Bls12_377, 2);

fn main() {
    let dir = std::env::args().nth(1).expect("usage: replay_rs <kit directory>");
    let meta: serde_json::Value = serde_json::from_slice(&std::fs::read(format!("{}/meta.json", dir)).unwrap()).unwrap();
    let ok = match meta["curve"].as_str().unwrap_or("bls12_381") {
        "bls12_381" => bls12_381::run(&dir, &meta),
        "bls12_377" => bls12_377::run(&dir, &meta),
        other => panic!("kit for an unsupported curve {}", other),
    };
    std::process::exit(if ok { 0 } else { 1 });
}
