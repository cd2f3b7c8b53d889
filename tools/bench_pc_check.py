#!/usr/bin/env python3
"""Level-1 `PC::check_combinations` throughput on one GPU (b2m_pc_check_combinations, DESIGN.md section 16): opening sets checked
per second, the library's phase split, and the card's name and power limit read in the same run, one JSON line per
configuration.  Writes nothing.

Each set has 8 commitments (6 plain, every other one hiding, and 2 degree-bounded ones, bounds 12 and 20 -- two bounds, so
SonicKZG10 has two bound slots in the pairing product) in arbitrary linear combinations opened at 2 points, the shape of
tests/pc_check_oracle.py.  64 distinct sets (made by the oracle) are repeated to fill the batch; --bad m gives m of them, at
seeded positions, a wrong opening challenge, so the batch is bisected.  The timed call is the library call alone (the arrays
are marshalled once); the Python marshalling time is reported beside it.

    python tools/bench_pc_check.py [--sets 4096] [--curve bls12_381 bn254] [--pc marlin_kzg10 sonic_kzg10] [--bad 0] [--steps 3]
"""
import argparse
import ctypes
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_verify import gpu_card  # noqa: E402
from marlin_b200 import _lib, api  # noqa: E402
import pc_check_oracle as P  # noqa: E402
from oracle import kzg  # noqa: E402
from oracle.params import BLS12_381, BN254  # noqa: E402

CURVES = {"bls12_381": BLS12_381, "bn254": BN254}


def run(ctx, cname, pc, args):
    m = api.Marlin(cname, pc, ctx=ctx)
    srs = m.srs_from_trapdoor(P.D, beta=0x5eed5eed5eed, gamma=7, degree_bounds=list(P.BOUNDS))
    vk = m.pc_verifier_key(srs, P.BOUNDS)
    ock = P.ck_for(P.pp_for(CURVES[cname], 0x5eed5eed5eed), kzg.MARLIN if pc == "marlin_kzg10" else kzg.SONIC)
    distinct = [P.random_set(ock, 1000 + i, n_plain=6, bounded=P.BOUNDS).api_set() for i in range(64)]
    bad = set(random.Random(args.seed).sample(range(args.sets), args.bad))
    sets = []
    for i in range(args.sets):
        s = distinct[i % 64]
        if i in bad:
            s = api.OpeningSet(s.commitments, s.query_set, s.evaluations, s.proofs, s.challenge + 1, lcs=s.lcs, degree_bounds=s.degree_bounds,
                               shifted=s.shifted)
        sets.append(s)
    want = [i not in bad for i in range(args.sets)]
    t0 = time.perf_counter()
    arrays = api.pc_check_arrays(m.curve_id, sets, False, None)
    marshal_s = time.perf_counter() - t0
    ptrs = [_lib.ptr(a) for a in arrays]
    verdicts = np.zeros(args.sets, dtype=np.int32)
    rng = api.ZkRng()

    def call():
        _lib.check(_lib.lib().b2m_pc_check_combinations(vk.handle, args.sets, *ptrs, ctypes.byref(rng.c), _lib.ptr(verdicts)))
        return [bool(v == 1) for v in verdicts] == want
    for _ in range(max(args.warmup, 1)):
        assert call()
    secs, phases, ok = [], [], True
    for _ in range(args.steps):
        t0 = time.perf_counter()
        ok = call() and ok  # synchronous at return
        secs.append(time.perf_counter() - t0)
        phases.append(vk.timings())
    keys = [k for k in phases[0] if k.endswith("_ms")]
    mean_s = sum(secs) / len(secs)
    print(json.dumps({
        "metric": "checked_sets_per_sec", "value": args.sets / mean_s, "unit": "sets/s", "n_gpus": 1, "steps": args.steps,
        "warmup": max(args.warmup, 1), "ms_per_call": 1e3 * mean_s, "higher_is_better": True,
        "config": {"workload": f"b2m_pc_check_combinations of {args.sets} sets (64 distinct, repeated) of 8 commitments (bounds 12, 20) "
                               f"at 2 points, {cname}, {pc}, {args.bad} with a wrong challenge (seed {args.seed})",
                   "timing": "host wall clock around each library call (synchronous at return)"},
        "verdicts_as_expected": ok, "marshal_s": marshal_s, "phases_ms": {k: sum(p[k] for p in phases) / len(phases) for k in keys},
        "checks_per_call": phases[-1]["checks"], "gpu": gpu_card(),
    }), flush=True)
    vk.close()
    srs.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sets", type=int, default=4096)
    ap.add_argument("--curve", nargs="+", default=["bls12_381", "bn254"], choices=list(CURVES))
    ap.add_argument("--pc", nargs="+", default=["marlin_kzg10", "sonic_kzg10"], choices=["marlin_kzg10", "sonic_kzg10"])
    ap.add_argument("--bad", type=int, default=0, help="sets with a wrong opening challenge, at seeded positions")
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if args.steps < 1 or args.sets < 1 or not 0 <= args.bad <= args.sets:
        ap.error("need --steps >= 1, --sets >= 1 and 0 <= --bad <= --sets")
    ctx = api.Context(0)
    for cname in args.curve:
        for pc in args.pc:
            run(ctx, cname, pc, args)
    ctx.close()


if __name__ == "__main__":
    main()
