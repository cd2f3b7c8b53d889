"""CPU: the committed replay kit (tests/golden/replay_kit, written on a GPU by tools/make_replay_kit.py and consumed by
tools/replay_rs on a machine with Rust) against the oracle: the GPU-made index_vk bytes and proof bytes are the oracle's for the same
SRS, circuit and rng seed; the SRS file holds the oracle's G1 powers in `serialize_uncompressed` form and a consistent G2 half; and the
bench.py reference arm keeps its JSON contract."""
import json
import os
import subprocess
import sys

import pytest

from marlin_b200 import srsfile
from oracle import ec, kzg, marlin as omarlin, r1cs as or1cs
from oracle import rng as orng
from oracle.params import BLS12_381 as curve

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KIT = os.path.join(ROOT, "tests", "golden", "replay_kit")


@pytest.fixture(scope="module")
def meta():
    return json.load(open(os.path.join(KIT, "meta.json")))


def test_kit_srs_file_is_the_oracles_srs(meta):
    d = srsfile.read_srs(os.path.join(KIT, "srs.bin"))
    assert d["curve_id"] == 0
    nb = curve.fq.nbytes
    n = 1 << meta["log_n"]
    beta, gamma = int(meta["beta"]), int(meta["gamma"])
    D = len(d["powers"]) // (2 * nb) - 1
    assert D == 4 * n - 1
    want = ec.fixed_base_powers(curve, curve.g, beta, D + 1)

    def g1(raw):
        x, y = int.from_bytes(raw[:nb], "little"), int.from_bytes(raw[nb:2 * nb], "little")
        assert y >> (8 * nb - 2) == 0  # no flag bits set on a finite point
        return (x, y)

    for i in range(D + 1):
        assert g1(d["powers"][i * 2 * nb:(i + 1) * 2 * nb]) == want[i]
    gamma_g = ec.scalar_mul(curve, gamma, curve.g)
    r = curve.fr.p
    for k, raw in d["gamma"].items():
        assert g1(raw) == ec.scalar_mul(curve, pow(beta, k, r), gamma_g)
    assert set(d["gamma"]) >= {0, 1, 2}
    # G2 half: beta_h = beta * h and neg_powers[k] = beta^-k * h, checked with the pairing-free identity in the oracle's own
    # G2 arithmetic is not available byte-wise (it works in E(Fq12)); tests/test_srs_files.py checks b2m_g2_scalar_muls against
    # definitional Fq2 arithmetic, here the keys and sizes
    assert sorted(d["neg_powers"]) == sorted(D - b for b in (n - 2, 4 * n - 2))
    assert len(d["h"]) == len(d["beta_h"]) == 4 * nb


@pytest.mark.parametrize("pc,scheme", [("marlin_kzg10", kzg.MARLIN), ("sonic_kzg10", kzg.SONIC)])
def test_kit_bytes_are_the_oracles(meta, pc, scheme):
    f = curve.fr
    n = 1 << meta["log_n"]
    a, b = int(meta["a"]), int(meta["b"])
    circ = or1cs.dummy_circuit(f, a % f.p, b % f.p, meta["num_variables"], n)
    srs = omarlin.universal_setup(curve, n, n, 3 * n, beta=int(meta["beta"]), g_scalar=1, gamma=int(meta["gamma"]))
    eng = kzg.Engine(use_trapdoor=True)
    pk = omarlin.index(srs, circ, scheme, eng)
    assert pk.vk_bytes == open(os.path.join(KIT, f"{pc}_index_vk_tobytes.bin"), "rb").read()
    zk = orng.ChaChaRng(bytes.fromhex(meta["zk_seed_hex"]), 12)
    proof = omarlin.prove(pk, circ, zk, eng)
    assert omarlin.serialize_proof(curve, scheme, proof) == open(os.path.join(KIT, f"{pc}_proof.bin"), "rb").read()
    assert zk.word_pos == meta["zk_word_pos_after"][pc]
    assert omarlin.verify(pk, [int(v) for v in meta["public_input"]], proof)


def test_reference_arm_json_contract():
    """`bench.py --impl reference`: same metric / unit / config keys as the GPU arm, the steps actually timed, explicit thread count
    (not the launcher's OMP_NUM_THREADS), on a tiny instance."""
    env = dict(os.environ, OMP_NUM_THREADS="1", RANK="0")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--log-n", "10", "--steps", "3", "--warmup", "2",
                          "--ref-budget-s", "60"], capture_output=True, text=True, env=env, timeout=300)
    assert out.returncode == 0, out.stderr
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["metric"] == "prover_constraints_per_sec" and line["unit"] == "constraints/s"
    assert line["steps"] == 3 and line["steps_requested"] == 3 and line["higher_is_better"] is True
    assert line["config"]["same_config_as_gpu_arm"] is True and "2^10" in line["config"]["workload"]
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
    from oracle import cport
    assert line["cpu_baseline"]["cores"] == min(cport.usable_cpus(), cport.lib().cport_max_threads())  # not 1 because of OMP_NUM_THREADS
    assert line["e2e"] == {"value": line["value"], "unit": "constraints/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    # other ranks of a torchrun launch print nothing and exit 0
    out2 = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--log-n", "10"], capture_output=True, text=True,
                          env=dict(env, RANK="1"), timeout=60)
    assert out2.returncode == 0 and out2.stdout.strip() == ""
