#!/usr/bin/env python3
"""Loading arkworks SRS files on one GPU (Marlin.load_ark_srs, DESIGN.md section 10): per curve and form, a `universal_setup`
key of 2^k powers is written with save_ark into a temporary directory and loaded back, timed by phase -- read and parse,
H2D, G1 decode, G2 decode, D2H (the library's CUDA-event spans) and the window-table build -- plus the card's name and power
limit, one JSON line per file.  SonicKZG10's G2 half is stood in for by 2^k neg_powers_of_h repeating a few valid points
(decode cost does not depend on the value).

    python tools/bench_srs_load.py [--log-powers 20 22] [--curves bls12_381 bn254 bls12_377]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_verify import gpu_card  # noqa: E402
from marlin_b200 import api, srsfile  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-powers", type=int, nargs="+", default=[20, 22])
    ap.add_argument("--curves", nargs="+", default=["bls12_381", "bn254"], choices=["bls12_381", "bn254", "bls12_377"])
    args = ap.parse_args()
    card = gpu_card()
    with tempfile.TemporaryDirectory() as tmp:
        for curve in args.curves:
            m = api.Marlin(curve, "sonic_kzg10", device=0)
            for lg in args.log_powers:
                n = 1 << lg
                srs = m.srs_from_trapdoor(n - 1, beta=0x5eed5eed5eed5eed, gamma=7, degree_bounds=[n // 2])
                h, beta_h, neg = srsfile.g2_setup(m.curve_id, api.fields.FR_MODULUS[m.curve_id], srs.trapdoor[0], n - 1, [1, 2, 3, 4])
                few = np.frombuffer(b"".join(neg[k] for k in sorted(neg)), dtype=np.uint8).reshape(len(neg), -1)
                srs.trapdoor, srs.g2 = None, (h, beta_h, srsfile.G2Points(np.arange(n, dtype=np.uint64), few[np.arange(n) % len(few)]))
                for compressed in (True, False):
                    path = os.path.join(tmp, "srs.bin")
                    srs.save_ark(path, compressed=compressed)
                    size = os.path.getsize(path)
                    t0 = time.perf_counter()
                    srsfile.read_ark(path, m.curve_id, compressed)
                    parse_ms = 1e3 * (time.perf_counter() - t0)
                    tables = []
                    real = api.Marlin.srs_from_points

                    def timed(self, *a, **k):
                        t = time.perf_counter()
                        s = real(self, *a, **k)
                        tables.append(1e3 * (time.perf_counter() - t))
                        return s
                    api.Marlin.srs_from_points = timed
                    m.ctx.profile(True)
                    t0 = time.perf_counter()
                    loaded = m.load_ark_srs(path, compressed=compressed, degree_bounds=[n // 2])
                    total_ms = 1e3 * (time.perf_counter() - t0)
                    spans = m.ctx.profile_report()
                    m.ctx.profile(False)
                    api.Marlin.srs_from_points = real
                    ms = {k: spans.get(k, {}).get("ms", 0.0) for k in ("ark_h2d", "ark_g1_decode", "ark_g2_decode", "ark_d2h")}
                    g1_pts = spans.get("ark_g1_decode", {}).get("units", 0)
                    g2_pts = spans.get("ark_g2_decode", {}).get("units", 0)
                    print(json.dumps({
                        "metric": "srs_load_ms", "value": total_ms, "unit": "ms", "curve": curve, "compressed": compressed,
                        "powers": n, "g1_points": g1_pts, "g2_points": g2_pts, "file_bytes": size,
                        "phases_ms": {"read_parse": parse_ms, "h2d": ms["ark_h2d"], "g1_decode": ms["ark_g1_decode"],
                                      "g2_decode": ms["ark_g2_decode"], "d2h": ms["ark_d2h"], "window_tables": sum(tables)},
                        "g1_points_per_sec": g1_pts / (ms["ark_g1_decode"] / 1e3) if ms["ark_g1_decode"] else None,
                        "g2_points_per_sec": g2_pts / (ms["ark_g2_decode"] / 1e3) if ms["ark_g2_decode"] else None,
                        "gpu": card}), flush=True)
                    loaded.close()
                    os.remove(path)
                srs.close()


if __name__ == "__main__":
    main()
