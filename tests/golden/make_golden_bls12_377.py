#!/usr/bin/env python3
"""Generates tests/golden/marlin_proofs_bls12_377.json from the oracle, the BLS12-377 counterpart of make_golden.py: the same
trapdoor, seeds and record format (tests_golden.regenerate_case), on the curve bls12_377_oracle.py registers with the
oracle.   Usage: python tests/golden/make_golden_bls12_377.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import bls12_377_oracle  # noqa: E402,F401  (registers the curve)
from oracle import kzg  # noqa: E402
from tests_golden import regenerate_case  # noqa: E402

CASES = [
    {"name": "bls377_marlin_test_circuit_26x25", "curve": "bls12_377", "scheme": kzg.MARLIN, "circuit": "test", "nc": 26, "nv": 25},
    {"name": "bls377_sonic_test_circuit_25x100", "curve": "bls12_377", "scheme": kzg.SONIC, "circuit": "test", "nc": 25, "nv": 100},
    {"name": "bls377_marlin_dummy_2p6", "curve": "bls12_377", "scheme": kzg.MARLIN, "circuit": "dummy", "nc": 64, "nv": 10},
    {"name": "bls377_sonic_dummy_2p6", "curve": "bls12_377", "scheme": kzg.SONIC, "circuit": "dummy", "nc": 64, "nv": 10},
    {"name": "bls377_marlin_dummy_2p10", "curve": "bls12_377", "scheme": kzg.MARLIN, "circuit": "dummy", "nc": 1024, "nv": 10},
]

if __name__ == "__main__":
    out = {"generator": "tests/golden/make_golden_bls12_377.py (oracle/ with tests/bls12_377_oracle.py)", "cases": [regenerate_case(c) for c in CASES]}
    with open(os.path.join(HERE, "marlin_proofs_bls12_377.json"), "w") as fh:
        json.dump(out, fh, indent=1)
    print("wrote", len(out["cases"]), "cases")
