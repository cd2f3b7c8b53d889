"""Throughput of b2m_pairing_check: for each curve, products per second with 2, 3 and 4 pairs per product at 1 to 2^16
products per call, one JSON line per (curve, pairs, products), with the card's name and power limit read in the same run.

The products are packed into their C arrays once, outside the timed region, and the C entry point is called directly.  A
call is timed by the host clock (it returns after its device work has finished).  It includes the host preparation of the
four G2 points' line coefficients; that preparation is also timed alone (a call with no products) and reported as `g2_prep_s`,
and `products_per_s` is computed from the call time minus it.  Every product is one (P against -P; with an odd pair count
one more pair has G1 at infinity), so every verdict is checked as well.

The first line reports device free memory (torch.cuda.mem_get_info) before and after the first pairing launch of the process:
the kernel's per-thread stack makes the driver grow the context's local-memory reservation.

    python tools/bench_pairing.py [--curves bls12_381,bn254,bls12_377] [--max-log 16] [--reps 3]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from marlin_b200 import _lib, api  # noqa: E402

CURVES = {"bls12_381": _lib.CURVE_BLS12_381, "bn254": _lib.CURVE_BN254, "bls12_377": _lib.CURVE_BLS12_377}


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", default=",".join(CURVES))
    ap.add_argument("--max-log", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    import pairing_ate_oracle as A
    from oracle import ec
    name, power = card()
    ctx = api.Context(0)
    L = _lib.lib()
    first = True
    for cname in a.curves.split(","):
        ci = CURVES[cname]
        curve, tw = A.CURVES[ci], A.Twist(A.CURVES[ci])
        nq = curve.fq.nbytes // 8
        g2 = np.frombuffer(b"".join(tw.uncompressed(tw.smul(k, tw.gen)) for k in (1, 2, 3, 5)), dtype=np.uint8)
        P = ec.scalar_mul(curve, 7, curve.g)
        mont = lambda Q: np.array([(curve.fq.to_mont(c) >> (64 * i)) & (2 ** 64 - 1) for c in Q for i in range(nq)], dtype=np.uint64)  # noqa: E731
        pp, pn, inf = mont(P), mont(ec.affine_neg(curve, P)), np.zeros(2 * nq, dtype=np.uint64)

        def call(n, off, g1, idx, out):
            _lib.check(L.b2m_pairing_check(ctx.handle, ci, 4, _lib.ptr(g2), n, _lib.ptr(off), _lib.ptr(g1), _lib.ptr(idx), _lib.ptr(out)))

        for n_pairs in (2, 3, 4):
            unit_g1, unit_q = [], []
            for j in range(n_pairs // 2):
                unit_g1 += [pp, pn]
                unit_q += [j, j]
            if n_pairs % 2:
                unit_g1.append(inf)
                unit_q.append(3)
            for lg in range(0, a.max_log + 1, 2):
                n = 1 << lg
                g1 = np.tile(np.concatenate(unit_g1), n)
                idx = np.tile(np.array(unit_q, dtype=np.uint32), n)
                off = (np.arange(n + 1, dtype=np.uint64) * n_pairs).astype(np.uint64)
                out = np.zeros(n, dtype=np.int32)
                if first:
                    free0 = torch.cuda.mem_get_info(0)[0]
                call(1, off, g1, idx, out)  # warm-up
                if first:
                    free1 = torch.cuda.mem_get_info(0)[0]
                    print(json.dumps({"first_pairing_launch_free_bytes_before": free0, "after": free1, "drop_bytes": free0 - free1, "curve": cname,
                                      "card": name, "power_limit": power}), flush=True)
                    first = False
                prep = min(_timed(lambda: call(0, off, g1, idx, out)) for _ in range(a.reps))
                best = None
                for _ in range(a.reps):
                    out[:] = 0
                    dt = _timed(lambda: call(n, off, g1, idx, out))
                    assert out.all()
                    best = dt if best is None else min(best, dt)
                print(json.dumps({"curve": cname, "pairs": n_pairs, "products": n, "call_s": round(best, 6), "g2_prep_s": round(prep, 6),
                                  "products_per_s": round(n / max(best - prep, 1e-9), 1), "card": name, "power_limit": power}), flush=True)


def _timed(f):
    t0 = time.perf_counter()
    f()
    return time.perf_counter() - t0


if __name__ == "__main__":
    main()
