#!/usr/bin/env python3
"""Writes the replay kit tools/replay_rs consumes (needs a GPU): an SRS file in ark-serialize layout, and -- for MarlinKZG10 and
SonicKZG10 -- the `ToBytes` image of index_vk, the `CanonicalSerialize` bytes of a proof of the reference bench's DummyCircuit and
the index key files (`IndexProverKey` / `IndexVerifierKey` `serialize`, marlin_b200/keyfile.py), all produced by libb2m.so, plus the inputs in meta.json.   python tools/make_replay_kit.py tests/golden/replay_kit [log_n [curve]]
(curve: bls12_381, the default, or bls12_377; tools/replay_rs reads it from meta.json)"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from marlin_b200 import api, fields, r1cs  # noqa: E402


def main():
    out = sys.argv[1]
    log_n = int(sys.argv[2]) if len(sys.argv) > 2 else 6
    curve = sys.argv[3] if len(sys.argv) > 3 else "bls12_381"
    assert curve in ("bls12_381", "bls12_377"), "the replay crate depends on ark-bls12-381 and ark-bls12-377 only"
    os.makedirs(out, exist_ok=True)
    n = 1 << log_n
    a, b = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
    beta, gamma = 0x5eed5eed5eed5eed5eed5eed, 7
    seed = bytes(range(32))
    meta = {"curve": curve, "log_n": log_n, "num_constraints": n, "num_variables": 10, "a": str(a), "b": str(b),
            "beta": str(beta), "gamma": str(gamma), "zk_seed_hex": seed.hex(), "zk_rng": "rand_chacha::ChaCha12Rng::from_seed (= StdRng of rand 0.8)",
            "note": "gamma_g = gamma * g, g = the standard G1 generator, h = the standard G2 generator", "zk_word_pos_after": {}}
    bounds = (n - 2, 4 * n - 2)
    ctx = api.Context(0)
    srs = None
    for pc in ("marlin_kzg10", "sonic_kzg10"):
        m = api.Marlin(curve, pc, ctx=ctx)
        if srs is None:
            srs = m.universal_setup(n, n, 3 * n, beta=beta, gamma=gamma, degree_bounds=bounds)
            srs.save(os.path.join(out, "srs.bin"), degree_bounds=bounds)
        circ = r1cs.dummy_circuit(m.curve_id, a, b, 10, n)
        pk = m.index(srs, circ)
        rng = api.ZkRng(seed, 12)
        proof = m.prove(pk, circ, rng)
        open(os.path.join(out, f"{pc}_index_vk_tobytes.bin"), "wb").write(pk.vk_bytes)
        open(os.path.join(out, f"{pc}_proof.bin"), "wb").write(proof)
        pk.save(os.path.join(out, f"{pc}_index_pk.bin"), compressed=True)  # IndexProverKey / IndexVerifierKey `serialize`
        pk.save_verifier_key(os.path.join(out, f"{pc}_index_vk.bin"), compressed=True)
        meta["zk_word_pos_after"][pc] = rng.word_pos
        pk.close()
    srs.close()
    meta["public_input"] = [str(a * b % fields.FR_MODULUS[fields.CURVE_IDS[curve]])]
    json.dump(meta, open(os.path.join(out, "meta.json"), "w"), indent=1)
    print("replay kit written to", out, {k: os.path.getsize(os.path.join(out, k)) for k in sorted(os.listdir(out))})


if __name__ == "__main__":
    main()
