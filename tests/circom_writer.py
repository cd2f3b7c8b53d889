"""Test helper: circom `.r1cs` and `.wtns` files from rows and assignments (not product code: the product only reads them,
marlin_b200/circom.py).

`r1cs_sections(...)` / `wtns_sections(...)` return a file as a list of [id, bytearray] and `write(...)` frames them, so a
test can reorder sections, add unknown or custom-gate ones, or corrupt a field before writing.  Rows are given as circom
writes them: per constraint three lists of (wire, canonical coefficient), in any order, with duplicate wires or zero
coefficients allowed.  `dummy_files(...)` writes bench.py's DummyCircuit vectorised, for 2^20 constraints and more.
[U circom r1csfile / snarkjs wtns_utils] as in marlin_b200/circom.py."""
import struct

import numpy as np

from marlin_b200 import fields


def write(path, magic, version, sections):
    with open(path, "wb") as fh:
        fh.write(magic + struct.pack("<II", version, len(sections)))
        for sid, data in sections:
            fh.write(struct.pack("<IQ", sid, len(data)))
            fh.write(bytes(data))
    return path


def r1cs_header(prime, n_wires, n_pub_out, n_pub_in, n_prv_in, m, n_labels=None, n8=32):
    return (struct.pack("<I", n8) + prime.to_bytes(n8, "little") + struct.pack("<IIII", n_wires, n_pub_out, n_pub_in, n_prv_in)
            + struct.pack("<QI", n_wires if n_labels is None else n_labels, m))


def lc_bytes(terms):
    return struct.pack("<I", len(terms)) + b"".join(struct.pack("<I", w) + (c % (1 << 256)).to_bytes(32, "little") for w, c in terms)


def constraints_bytes(constraints):
    """constraints: [(A, B, C)], each a list of (wire, coefficient); coefficients are written as given (mod 2^256)"""
    return b"".join(lc_bytes(a) + lc_bytes(b) + lc_bytes(c) for a, b, c in constraints)


def r1cs_sections(prime, n_wires, n_pub_out, n_pub_in, constraints, n_prv_in=0, labels=True):
    secs = [[1, bytearray(r1cs_header(prime, n_wires, n_pub_out, n_pub_in, n_prv_in, len(constraints)))],
            [2, bytearray(constraints_bytes(constraints))]]
    if labels:
        secs.append([3, bytearray(struct.pack(f"<{n_wires}Q", *range(n_wires)))])
    return secs


def wtns_sections(prime, values, n8=32):
    return [[1, bytearray(struct.pack("<I", n8) + prime.to_bytes(n8, "little") + struct.pack("<I", len(values)))],
            [2, bytearray(b"".join((v % (1 << 256)).to_bytes(32, "little") for v in values))]]


def write_r1cs(path, *args, order=None, extra=(), **kw):
    """order: section ids in file order (default as made); extra: [id, bytes] sections appended (unknown or custom gates)"""
    secs = r1cs_sections(*args, **kw)
    if order is not None:
        by = {s: d for s, d in secs}
        secs = [[s, by[s]] for s in order]
    return write(path, b"r1cs", 1, secs + [list(e) for e in extra])


def write_wtns(path, prime, values):
    return write(path, b"wtns", 2, wtns_sections(prime, values))


def from_generated(g):
    """(n_wires, n_pub_out, n_pub_in, constraints, wtns values) of a tests/r1cs_random.py system (keep_rows=True):
    wire = the unpadded column, public inputs as outputs"""
    a_rows, b_rows, c_rows = g.rows
    cons = [([(i, c) for c, i in ra], [(i, c) for c, i in rb], [(i, c) for c, i in rc]) for ra, rb, rc in zip(a_rows, b_rows, c_rows)]
    values = list(g.instance) + list(g.witness)
    return len(values), len(g.instance) - 1, 0, cons, values


def normal_form(rows, p):
    """rows as from_rows takes them ([(coeff, col)]) -> columns ascending, equal columns summed mod p, zero sums dropped"""
    out = []
    for row in rows:
        acc = {}
        for c, i in row:
            acc[i] = (acc.get(i, 0) + c) % p
        out.append([(acc[i], i) for i in sorted(acc) if acc[i]])
    return out


# ---- vectorised files at full size ---------------------------------------------------------------------------------------
def _u32(v):
    return np.frombuffer(struct.pack("<I", v), dtype=np.uint8)


def _fe(v):
    return np.frombuffer(v.to_bytes(32, "little"), dtype=np.uint8)


def _records(patterns, idx):
    """section bytes of rows idx[k] drawn from equal-length byte patterns"""
    pat = np.stack([np.frombuffer(p, dtype=np.uint8) for p in patterns])
    return pat[idx].reshape(-1)


def dummy_files(r1cs_path, wtns_path, curve_id, a, b, num_variables, n, terms=1, seed=0):
    """bench.py's `dummy_circuit(cid, a, b, num_variables, n)` as circom files: wire 1 = c = a b (the public output), wire 2 =
    a, wire 3 = b, the rest copies of a; n - 1 constraints a * b = c and one empty constraint.  terms > 1 gives every LC
    `terms` terms in shuffled wire order: A = sum k_t a-copies with sum k_t = 1, B = b + zero-sum a-copy terms, C = c +
    zero-sum a-copy terms (64 seeded patterns), so the instance stays satisfied and loads to rows that need normalising."""
    p = fields.FR_MODULUS[curve_id]
    c = a * b % p
    n_wires = num_variables + 1  # One, c, a, b, num_variables - 3 copies of a
    copies = [2] + list(range(4, n_wires))
    rnd = np.random.default_rng(seed)

    def rand_fe():
        return int.from_bytes(rnd.bytes(32), "little") % p

    def spread(base_terms, total):
        """base_terms plus (terms - len(base)) a-copy terms whose coefficients add up to `total`, shuffled"""
        k = terms - len(base_terms)
        ks = [rand_fe() for _ in range(k - 1)]
        ks.append((total - sum(ks)) % p)
        ws = list(rnd.choice(copies, size=k, replace=len(copies) < k))
        lc = base_terms + list(zip(ws, ks))
        return [lc[i] for i in rnd.permutation(len(lc))]

    if terms == 1:
        patterns = [constraints_bytes([([(2, 1)], [(3, 1)], [(1, 1)])])]
    else:
        patterns = [constraints_bytes([(spread([], 1), spread([(3, 1)], 0), spread([(1, 1)], 0))]) for _ in range(64)]
    idx = rnd.integers(0, len(patterns), size=n - 1)
    body = np.concatenate([_records(patterns, idx), np.zeros(12, dtype=np.uint8)])
    with open(r1cs_path, "wb") as fh:
        hdr = r1cs_header(p, n_wires, 1, 0, 2, n)
        fh.write(b"r1cs" + struct.pack("<II", 1, 2))
        fh.write(struct.pack("<IQ", 1, len(hdr)) + hdr)
        fh.write(struct.pack("<IQ", 2, len(body)))
        body.tofile(fh)
    vals = [1, c, a, b] + [a] * (n_wires - 4)
    write_wtns(wtns_path, p, vals)
    return n_wires
