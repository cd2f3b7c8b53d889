"""Time Marlin.load_ptau by phase: a power-(log D + 1) Powers-of-Tau file is written with its tauG1 prefix computed on the GPU
(tests/ptau_writer.py: the rest of the file is holes), then loaded with check=True.  Phases: framing (marlin_b200.ptau), the G1
and G2 LEM decode kernels, the window tables (the rest of a check=False load), and the power check's MSM, pairing and
bisection spans.  Prints one JSON line per (curve, D) with the GPU name and power limit read in the same run.

    python tools/bench_ptau_load.py --log-degree 20 22 --curves bls12_381 bn254
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

from marlin_b200 import api, fields, ptau  # noqa: E402

import ptau_writer as pw  # noqa: E402


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
    ap.add_argument("--log-degree", type=int, nargs="+", default=[20, 22], help="D = 2^k - 1 for each k")
    ap.add_argument("--curves", nargs="+", default=["bls12_381", "bn254"])
    ap.add_argument("--repeat", type=int, default=2, help="loads per size; the first warms the module and the pairing stack")
    args = ap.parse_args()
    gpu = gpu_info()
    ctx = api.Context(0)
    for curve in args.curves:
        cid = fields.CURVE_IDS[curve]
        m = api.Marlin(curve, "marlin_kzg10", ctx=ctx)
        for k in args.log_degree:
            D = (1 << k) - 1
            power = ptau.power_for_degree(D)
            with tempfile.TemporaryDirectory() as tmp:
                path = os.path.join(tmp, "bench.ptau")
                pw.write_gpu_prefix(ctx, cid, path, power, D, 0x5eed5eed5eed5eed5eed5eed, 7)
                for rep in range(args.repeat):
                    t = time.perf_counter()
                    ptau.read_ptau(path)
                    framing = (time.perf_counter() - t) * 1e3
                    ctx.profile(True)
                    t = time.perf_counter()
                    srs = m.load_ptau(path, max_degree=D, check=False)
                    unchecked = (time.perf_counter() - t) * 1e3
                    dec = ctx.profile_report()
                    srs.close()
                    ctx.profile(True)
                    t = time.perf_counter()
                    srs = m.load_ptau(path, max_degree=D, check=True, rng=api.ZkRng(bytes([rep + 1]) * 32, 20))
                    total = (time.perf_counter() - t) * 1e3
                    chk = ctx.profile_report()
                    ctx.profile(False)
                    srs.close()
                    g1 = span_ms(dec, "lem_g1_decode")
                    g2 = span_ms(dec, "lem_g2_decode")
                    copies = span_ms(dec, "ark_h2d", "ark_d2h")
                    print(json.dumps({
                        "gpu": gpu, "curve": curve, "D": D, "power": power, "rep": rep,
                        "framing_ms": round(framing, 2), "g1_decode_ms": g1, "g2_decode_ms": g2, "decode_copies_ms": copies,
                        "tables_and_host_ms": round(unchecked - framing - g1 - g2 - copies, 2),
                        "check_msm_ms": span_ms(chk, "srs_check_msm"), "check_pairing_ms": span_ms(chk, "srs_check_pairing"),
                        "bisection_ms": span_ms(chk, "srs_check_bisection"), "check_ms": round(total - unchecked, 2),
                        "total_ms": round(total, 2)}), flush=True)


if __name__ == "__main__":
    main()
