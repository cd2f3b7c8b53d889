"""Loading an index key file against re-indexing, on one GPU: DummyCircuit 2^log_n (bench.py's instance), BLS12-381 /
MarlinKZG10 by default.  Prints one JSON line: the file size, `Marlin.index` from the matrices, `IndexProverKey.save`, and
`Marlin.load_index` split into host framing (keyfile.read_prover_key) and the rest, with the device spans of the loader's
kernels (ark_h2d, ark_fr_decode, ark_g1_decode, ark_g2_decode, ntt) from the context profiler, and the card's name and power
limit.  Wall-clock seconds of one run after one warm-up load; the file goes to a temporary directory.

    python tools/bench_index_load.py [--log-n 20] [--curve bls12_381] [--pc marlin_kzg10] [--uncompressed]
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_verify import gpu_card  # noqa: E402
from marlin_b200 import api, keyfile, r1cs as gr1cs  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--curve", default="bls12_381")
    ap.add_argument("--pc", default="marlin_kzg10")
    ap.add_argument("--uncompressed", action="store_true")
    args = ap.parse_args()
    compressed = not args.uncompressed
    n = 1 << args.log_n
    m = api.Marlin(args.curve, args.pc)
    a, b = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
    srs = m.universal_setup(n, n, 3 * n, beta=0x5eed5eed5eed5eed5eed5eed, gamma=7, degree_bounds=(n - 2, 4 * n - 2))
    circ = gr1cs.dummy_circuit(m.curve_id, a, b, 10, n)
    out = {"log_n": args.log_n, "curve": args.curve, "pc": args.pc, "compressed": compressed, "gpu": gpu_card()}
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "pk.bin")
        t = time.perf_counter()
        pk = m.index(srs, circ)
        out["index_s"] = time.perf_counter() - t
        t = time.perf_counter()
        pk.save(path, compressed=compressed)
        out["save_s"] = time.perf_counter() - t
        want = m.prove(pk, circ, api.ZkRng.test_rng())
        pk.close()
        out["file_bytes"] = os.path.getsize(path)
        m.load_index(srs, path, compressed=compressed).close()  # warm-up (page cache, NTT tables)
        t = time.perf_counter()
        keyfile.read_prover_key(path, m.curve_id, m.pc, compressed)
        out["parse_s"] = time.perf_counter() - t
        m.ctx.profile(True)
        t = time.perf_counter()
        pk2 = m.load_index(srs, path, compressed=compressed)
        out["load_index_s"] = time.perf_counter() - t
        spans = m.ctx.profile_report()
        m.ctx.profile(False)
        out["device_spans_ms"] = {k: round(v["ms"], 3) for k, v in spans.items()} if isinstance(spans, dict) else spans
        out["proof_identical"] = m.prove(pk2, circ, api.ZkRng.test_rng()) == want
        pk2.close()
    srs.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
