#!/usr/bin/env python3
"""Batched verification throughput on one GPU (Marlin.verify_batch, DESIGN.md section 9): proofs verified per second, the
library's phase split and the card's name and power limit read in the same run, printed as one JSON line.  Writes nothing.

Verification cost barely depends on the circuit, so the proofs are of a small DummyCircuit (2^log_n constraints): 64 distinct
proofs (distinct zk streams) repeated to fill the batch.  Every proof is valid, so a batch is one randomised check and no
bisection.  The phase split is the library's own (host wall clock around synchronised work), averaged over the timed steps.

    python tools/bench_verify.py --batch 4096 [--curve bn254] [--pc sonic_kzg10] [--log-n 10] [--steps 3] [--warmup 1]
"""
import argparse
import json
import random
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from marlin_b200 import api, fields, r1cs  # noqa: E402


def gpu_card():
    """name and power limit of device 0"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, limit = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as e:
        return {"name": None, "power_limit": None, "error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096, help="proofs per verify_batch call")
    ap.add_argument("--log-n", type=int, default=10, help="log2 of the constraints of the verified circuit")
    ap.add_argument("--curve", default="bls12_381", choices=["bls12_381", "bn254", "bls12_377"])
    ap.add_argument("--pc", default="marlin_kzg10", choices=["marlin_kzg10", "sonic_kzg10"])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--bad", type=int, default=0, help="proofs checked against a wrong public input, at seeded positions")
    ap.add_argument("--seed", type=int, default=1, help="seed of the bad positions")
    args = ap.parse_args()
    if args.steps < 1 or args.batch < 1:
        ap.error("--steps and --batch must be at least 1")
    if not 0 <= args.bad <= args.batch:
        ap.error("--bad must be between 0 and --batch")

    m = api.Marlin(args.curve, args.pc, device=0)
    n = 1 << args.log_n
    a, b = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
    circ = r1cs.dummy_circuit(m.curve_id, a, b, 10, n)
    md = api.max_degree(n, n, 3 * n)
    # SonicKZG10 needs the gamma powers of the bounds |H| - 2 and |K| - 2: keep those of every power of two up to md
    bounds = [(1 << k) - 2 for k in range(2, md.bit_length() + 1) if (1 << k) - 2 <= md]
    srs = m.srs_from_trapdoor(md, beta=0x5eed5eed5eed5eed5eed5eed, gamma=7, degree_bounds=bounds)
    pk = m.index(srs, circ)
    vk = m.verifier_key(pk, srs)
    distinct = [m.prove(pk, circ, api.ZkRng(bytes([i]) * 32, 12)) for i in range(64)]
    proofs = [distinct[i % 64] for i in range(args.batch)]
    inputs = [circ.public_input()] * len(proofs)
    bad = set(random.Random(args.seed).sample(range(args.batch), args.bad))
    wrong = [(x + 1) % fields.FR_MODULUS[m.curve_id] for x in circ.public_input()]
    inputs = [wrong if i in bad else x for i, x in enumerate(inputs)]
    want = [i not in bad for i in range(args.batch)]
    rng = api.ZkRng()
    for _ in range(max(args.warmup, 1)):
        assert m.verify_batch(vk, inputs, proofs, rng) == want
    secs, phases, ok = [], [], True
    for _ in range(args.steps):
        t0 = time.perf_counter()
        ok = m.verify_batch(vk, inputs, proofs, rng) == want and ok  # synchronous at return
        secs.append(time.perf_counter() - t0)
        phases.append(vk.timings())
    keys = [k for k in phases[0] if k.endswith("_ms")]
    mean_s = sum(secs) / len(secs)
    print(json.dumps({
        "metric": "verified_proofs_per_sec", "value": args.batch / mean_s, "unit": "proofs/s", "n_gpus": 1, "steps": args.steps,
        "warmup": max(args.warmup, 1), "ms_per_batch": 1e3 * mean_s, "higher_is_better": True,
        "config": {"workload": f"Marlin.verify_batch of {args.batch} proofs (64 distinct, repeated) of DummyCircuit 2^{args.log_n}, "
                               f"{args.curve}, {args.pc}, {args.bad} checked against a wrong public input (seed {args.seed})",
                   "timing": "host wall clock around each verify_batch call (synchronous at return)"},
        "all_accepted": ok, "phases_ms": {k: sum(p[k] for p in phases) / len(phases) for k in keys}, "checks_per_batch": phases[-1]["checks"],
        "gpu": gpu_card(),
    }))
    vk.close()
    pk.close()
    srs.close()


if __name__ == "__main__":
    main()
