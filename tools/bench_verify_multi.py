#!/usr/bin/env python3
"""Cross-key batched verification on one GPU (api.verify_many, DESIGN.md section 9): M verifier keys on one SRS, P proofs
each, timed (a) as M Marlin.verify_batch calls, one per key, and (b) as one verify_many call over all M * P proofs, the two
alternated in one process.  Prints one JSON line: proofs/s and the library's phase split of each (for (a) summed over the M
calls), and the card's name and power limit read in the same run.  Writes nothing.

Key k is DummyCircuit with 2^log_n - k constraints (so all keys share |H| and their indexes differ; DummyCircuit's
num_variables would not tell them apart, since squaring the matrices pads the witness to the constraint count).  With
--sonic, the odd keys are SonicKZG10 keys of the same circuits.  8 distinct proofs per key are repeated to fill P; --bad m of
the M * P proofs, at seeded positions, are checked against a wrong public input.

    python tools/bench_verify_multi.py --keys 64 --per-key 64 [--curve bls12_381] [--sonic] [--bad 7] [--log-n 8]
"""
import argparse
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_verify import gpu_card  # noqa: E402
from marlin_b200 import api, fields, r1cs  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curve", default="bls12_381", choices=["bls12_381", "bn254", "bls12_377"])
    ap.add_argument("--keys", type=int, default=8, help="verifier keys M")
    ap.add_argument("--per-key", type=int, default=64, help="proofs per key P")
    ap.add_argument("--bad", type=int, default=0, help="proofs checked against a wrong public input, at seeded positions")
    ap.add_argument("--log-n", type=int, default=8, help="log2 of the constraints of key 0's circuit")
    ap.add_argument("--sonic", action="store_true", help="make every odd key a SonicKZG10 key")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=1, help="seed of the bad positions")
    args = ap.parse_args()
    n_all = args.keys * args.per_key
    if args.steps < 1 or args.keys < 1 or args.per_key < 1:
        ap.error("--steps, --keys and --per-key must be at least 1")
    if not 0 <= args.bad <= n_all:
        ap.error("--bad must be between 0 and keys * per-key")
    if 2 * args.keys > 1 << args.log_n:
        ap.error("--keys must be at most 2^(log_n - 1)")

    ctx = api.Context(0)
    pcs = ["sonic_kzg10" if args.sonic and k % 2 else "marlin_kzg10" for k in range(args.keys)]
    ms = {pc: api.Marlin(args.curve, pc, ctx=ctx) for pc in set(pcs)}
    m0 = next(iter(ms.values()))
    n = 1 << args.log_n
    a, b = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
    md = api.max_degree(n, n, 3 * n)
    bounds = [(1 << k) - 2 for k in range(2, md.bit_length() + 1) if (1 << k) - 2 <= md]
    # one SRS (one trapdoor) per PC object: the same h and beta h, so all keys form one G2 group
    srss = {pc: m.srs_from_trapdoor(md, beta=0x5eed5eed5eed5eed5eed5eed, gamma=7, degree_bounds=bounds) for pc, m in ms.items()}
    keys, entries = [], []
    wrong_of = {}
    bad = set(random.Random(args.seed).sample(range(n_all), args.bad))
    for k, pc in enumerate(pcs):
        m = ms[pc]
        circ = r1cs.dummy_circuit(m.curve_id, a, b, 10, n - k)
        pk = m.index(srss[pc], circ)
        vk = m.verifier_key(pk, srss[pc])
        pub = circ.public_input()
        wrong_of[k] = [(x + 1) % fields.FR_MODULUS[m.curve_id] for x in pub]
        distinct = [m.prove(pk, circ, api.ZkRng(bytes([i]) * 32, 12)) for i in range(8)]
        pk.close()
        keys.append((m, vk))
        for j in range(args.per_key):
            i = len(entries)
            entries.append((vk, wrong_of[k] if i in bad else pub, distinct[j % 8]))
    want = [i not in bad for i in range(n_all)]
    rng = api.ZkRng()

    def run_calls():
        got, phases = [], []
        for k, (m, vk) in enumerate(keys):
            part = entries[k * args.per_key:(k + 1) * args.per_key]
            got += m.verify_batch(vk, [e[1] for e in part], [e[2] for e in part], rng)
            phases.append(vk.timings())
        return got, {key: sum(p[key] for p in phases) for key in phases[0] if key.endswith("_ms") or key in ("checks", "products")}

    def run_many():
        got = api.verify_many(entries, rng)
        return got, keys[0][1].timings()

    for _ in range(max(args.warmup, 1)):
        assert run_calls()[0] == want and run_many()[0] == want
    out = {"calls": {"secs": [], "phases": []}, "many": {"secs": [], "phases": []}}
    ok = True
    for _ in range(args.steps):  # alternated, so both see the same machine state
        for name, fn in (("calls", run_calls), ("many", run_many)):
            t0 = time.perf_counter()
            got, ph = fn()  # synchronous at return
            out[name]["secs"].append(time.perf_counter() - t0)
            out[name]["phases"].append(ph)
            ok = ok and got == want
    res = {}
    for name, o in out.items():
        mean_s = sum(o["secs"]) / len(o["secs"])
        res[name] = {"proofs_per_sec": n_all / mean_s, "ms_per_batch": 1e3 * mean_s, "ms_per_step": [1e3 * s for s in o["secs"]],
                     "phases": {k: sum(p[k] for p in o["phases"]) / len(o["phases"]) for k in o["phases"][0] if isinstance(o["phases"][0][k], (int, float))}}
    print(json.dumps({
        "metric": "verified_proofs_per_sec", "value": res["many"]["proofs_per_sec"], "unit": "proofs/s", "higher_is_better": True,
        "n_gpus": 1, "steps": args.steps, "warmup": max(args.warmup, 1), "speedup": res["many"]["proofs_per_sec"] / res["calls"]["proofs_per_sec"],
        "config": {"workload": f"{args.keys} keys x {args.per_key} proofs (8 distinct per key) of DummyCircuit 2^{args.log_n} - k, {args.curve}, "
                               f"{'MarlinKZG10 / SonicKZG10 alternating' if args.sonic else 'MarlinKZG10'}, {args.bad} checked against a wrong "
                               f"public input (seed {args.seed})",
                   "timing": "host wall clock around the M verify_batch calls (calls) and the verify_many call (many), alternated"},
        "all_accepted_as_expected": ok, "per_key_calls": res["calls"], "verify_many": res["many"], "gpu": gpu_card(),
    }))
    for _, vk in keys:
        vk.close()
    for s in srss.values():
        s.close()
    ctx.close()


if __name__ == "__main__":
    main()
