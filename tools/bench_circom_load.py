"""Time the circom loaders by phase on seeded files (tests/circom_writer.py): bench.py's DummyCircuit (one term per LC) and
the same circuit with several shuffled terms per LC, so every row is normalised.  Phases: framing (marlin_b200.circom), the
host walk over the term counts (b2m_circom_constraint_rows), the section's H2D copies, decode and normalise, the D2H copies
(spans of b2m_circom_decode_constraints), the witness decode (load_wtns with check=False), the satisfiability check
(which_is_unsatisfied) and, for scale, `Marlin.index` of the loaded matrices.  Prints one JSON line per (curve, size,
terms) with the GPU name and power limit read in the same run.

    python tools/bench_circom_load.py --log-n 20 22 --curves bls12_381 bn254 --terms 1 4
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from marlin_b200 import api, circom, fields  # noqa: E402

import circom_writer as cw  # noqa: E402


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def span_ms(report, *names):
    return round(sum(report.get(n, {}).get("ms", 0.0) for n in names), 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, nargs="+", default=[20, 22], help="2^k constraints")
    ap.add_argument("--curves", nargs="+", default=["bls12_381", "bn254"])
    ap.add_argument("--terms", type=int, nargs="+", default=[1, 4], help="terms per linear combination")
    ap.add_argument("--repeat", type=int, default=2, help="loads per file; the first warms the module")
    ap.add_argument("--index-max-log", type=int, default=22, help="index the one-term circuit up to 2^k constraints")
    args = ap.parse_args()
    gpu = gpu_info()
    ctx = api.Context(0)
    a, b = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
    for curve in args.curves:
        cid = fields.CURVE_IDS[curve]
        m = api.Marlin(curve, "marlin_kzg10", ctx=ctx)
        for k in args.log_n:
            n = 1 << k
            for terms in args.terms:
                with tempfile.TemporaryDirectory() as tmp:
                    rp, wp = os.path.join(tmp, "c.r1cs"), os.path.join(tmp, "c.wtns")
                    cw.dummy_files(rp, wp, cid, a, b, 10, n, terms=terms, seed=k)
                    size = os.path.getsize(rp)
                    for rep in range(args.repeat):
                        t = time.perf_counter()
                        f = circom.read_r1cs(rp)
                        framing = (time.perf_counter() - t) * 1e3
                        t = time.perf_counter()
                        circom.constraint_rows(f)
                        walk = (time.perf_counter() - t) * 1e3
                        ctx.profile(True)
                        t = time.perf_counter()
                        r = m.load_r1cs(rp)
                        load = (time.perf_counter() - t) * 1e3
                        t = time.perf_counter()
                        rw = m.load_wtns(r, wp, check=False)
                        wtns = (time.perf_counter() - t) * 1e3
                        t = time.perf_counter()
                        bad = m.which_is_unsatisfied(rw)
                        check = (time.perf_counter() - t) * 1e3
                        rep_ = ctx.profile_report()
                        ctx.profile(False)
                        assert bad is None, f"constraint {bad} is not satisfied"
                        row = {"gpu": gpu, "curve": curve, "log_n": k, "terms_per_lc": terms, "r1cs_bytes": size, "rep": rep,
                               "framing_ms": round(framing, 2), "host_walk_ms": round(walk, 2),
                               "h2d_ms": span_ms(rep_, "circom_h2d"), "decode_normalise_ms": span_ms(rep_, "circom_decode"),
                               "d2h_ms": span_ms(rep_, "circom_d2h"), "load_r1cs_ms": round(load, 2), "load_wtns_ms": round(wtns, 2),
                               "witness_decode_ms": span_ms(rep_, "ark_h2d", "ark_fr_decode"),
                               "check_ms": round(check, 2), "check_h2d_ms": span_ms(rep_, "r1cs_check_h2d")}
                        if terms == 1 and k <= args.index_max_log and rep == args.repeat - 1:
                            srs = m.universal_setup(n, n, 3 * n, beta=0x5eed5eed5eed5eed5eed5eed, gamma=7)
                            t = time.perf_counter()
                            pk = m.index(srs, r)
                            row["index_ms"] = round((time.perf_counter() - t) * 1e3, 2)
                            pk.close()
                            srs.close()
                        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
