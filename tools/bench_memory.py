"""How large a circuit proves on one GPU, and what fewer window tables and bounded MSM passes cost.

For each configuration -- log2 of the constraints, curve, PC, and either a device-memory limit (auto layout) or a forced layout
(window tables, pass cap) -- runs universal_setup -> index -> prove (warm-up, then timed proves) on a DummyCircuit with
|K| = 4|H|, and prints one JSON line: ms per proof, the layout (c, T, pass cap), the byte model's figures and budget, the device
pool's high-water mark over setup + index + prove, and GPU verification of the proof (true) and of a wrong public input (false).
It also records where the index keeps its twelve |K|-vectors ("device", or "host": pinned, streamed to every proof), the pinned
bytes, and per proof the bytes streamed, the copy engine's time on them and the host-to-device rate this gives.  A key the
model refuses is reported with the refusal's message.  The card's name and power limit are read in the same run.

    python tools/bench_memory.py --log-n 20 --tables 0 4 2 1          # one line per forced table count (0: the planned layout)
    python tools/bench_memory.py --log-n 22 --pc sonic_kzg10
    python tools/bench_memory.py --log-n 23 --limit-gb 70
    python tools/bench_memory.py --log-n 20 --index-host                 # host-resident index at a size that fits the device
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,memory.total", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run(args, tables, cap):
    from marlin_b200 import _lib, api, fields, r1cs
    n = 1 << args.log_n
    ctx = api.Context(0, memory_limit=int(args.limit_gb * 1e9) if args.limit_gb else None)
    rec = {"log_n": args.log_n, "curve": args.curve, "pc": args.pc, "limit_gb": args.limit_gb, "forced_tables": tables, "forced_max_pairs": cap,
           "card": card()}
    if cap:
        os.environ["B2M_MSM_MAX_PAIRS"] = str(cap)
    if args.index_host:
        os.environ["B2M_INDEX_HOST"] = "1"
        rec["forced_index_host"] = True
    try:
        m = api.Marlin(args.curve, args.pc, ctx=ctx)
        a, b = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
        circ = r1cs.dummy_circuit(m.curve_id, a, b, 10, n)
        ctx.memory()
        rec["pool_before"] = ctx.memory()["used"]
        t0 = time.time()
        try:
            srs = m.universal_setup(n, n, 3 * n, beta=0x5eed5eed5eed5eed5eed5eed, gamma=7, degree_bounds=(n - 2, 4 * n - 2),
                                    window_tables=tables)
        except _lib.B2MError as e:
            rec["refused"] = str(e)
            return rec
        finally:
            os.environ.pop("B2M_MSM_MAX_PAIRS", None)
        rec["layout"] = srs.layout()
        try:
            pk = m.index(srs, circ)
            rec["setup_index_s"] = round(time.time() - t0, 2)
            rec["residency"], rec["pinned_bytes"] = pk.residency, pk.host_bytes
            try:
                m.stage(pk, circ)
                zk = api.ZkRng.test_rng()
                for _ in range(args.warmup):
                    m.prove(pk, None, zk)
                ms, h2d = [], []
                for _ in range(args.steps):
                    m.prove(pk, None, zk)
                    t = pk.timings()
                    ms.append(t["Marlin::Prover"])
                    if "IndexStream::H2D" in t:
                        h2d.append(t["IndexStream::H2D"])
                        rec["streamed_bytes_per_proof"] = int(t["IndexStream::bytes"])
                rec["ms_per_proof"] = round(sum(ms) / len(ms), 2)
                if h2d:
                    rec["h2d_ms_per_proof"] = round(sum(h2d) / len(h2d), 2)
                    rec["h2d_gb_per_s"] = round(rec["streamed_bytes_per_proof"] / (rec["h2d_ms_per_proof"] * 1e6), 2)
                rec["ms_min_max"] = [round(min(ms), 2), round(max(ms), 2)]
                rec["pool_peak"] = ctx.memory()["peak"]
                proof = m.prove(pk, circ, api.ZkRng.test_rng())
                import hashlib
                rec["proof_sha256"] = hashlib.sha256(proof).hexdigest()
                vk = m.verifier_key(pk, srs)
                try:
                    c_pub = a * b % fields.FR_MODULUS[m.curve_id]
                    rec["verify_ok"] = m.verify(vk, [c_pub], proof, api.ZkRng())
                    rec["verify_wrong_input"] = m.verify(vk, [(c_pub + 1) % fields.FR_MODULUS[m.curve_id]], proof, api.ZkRng())
                finally:
                    vk.close()
            finally:
                pk.close()
        finally:
            srs.close()
    except _lib.B2MError as e:
        rec["error"] = str(e)
    finally:
        os.environ.pop("B2M_INDEX_HOST", None)
        ctx.close()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--curve", default="bls12_381", choices=["bls12_381", "bn254", "bls12_377"])
    ap.add_argument("--pc", default="marlin_kzg10", choices=["marlin_kzg10", "sonic_kzg10"])
    ap.add_argument("--limit-gb", type=float, default=0.0, help="device-memory limit of the context (0: free device memory)")
    ap.add_argument("--tables", type=int, nargs="*", default=[0], help="forced window tables, one run each (0: the planned layout)")
    ap.add_argument("--max-pairs", type=int, default=0, help="forced MSM pass cap (0: the planned one)")
    ap.add_argument("--index-host", action="store_true", help="force a host-resident index (B2M_INDEX_HOST=1)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    for t in args.tables:
        rec = run(args, t, args.max_pairs)
        line = json.dumps(rec)
        print(line, flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(line + "\n")


if __name__ == "__main__":
    main()
