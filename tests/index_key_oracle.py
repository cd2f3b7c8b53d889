"""Independent writer of arkworks index key files for the key-file tests: the `IndexProverKey` and `IndexVerifierKey` bytes of
the Python oracle's `Marlin::index` (oracle/marlin.py, oracle/ahp.py) on an oracle SRS with a known trapdoor, in the layout
marlin_b200/keyfile.py documents [U ark-serialize / ark-poly / ark-poly-commit 0.3].  Plain integers over oracle/ and the
point encodings of oracle/transcript.py and tests/ark_srs_oracle.py; the product is never imported."""
import struct

from oracle import kzg
from oracle import marlin as omarlin
from oracle.poly import Domain

import ark_srs_oracle as ao

LABELS = ("row", "col", "a_val", "b_val", "c_val", "row_col")
EVAL_FIELDS = ("row", "col", "row_col", "val_a", "val_b", "val_c")


def u64(v):
    return struct.pack("<Q", v)


def fe(f, v):
    return (v % f.p).to_bytes(32, "little")


def vec(items):
    return u64(len(items)) + b"".join(items)


def strip(coeffs):
    coeffs = list(coeffs)
    while coeffs and coeffs[-1] == 0:
        coeffs.pop()
    return coeffs


def domain(f, size):
    d = Domain(f, size)
    return (b"\x00" + u64(d.size) + struct.pack("<I", d.log_size) + fe(f, d.size_as_field_element) + fe(f, d.size_inv)
            + fe(f, d.group_gen) + fe(f, d.group_gen_inv) + fe(f, pow(f.generator, -1, f.p)))


def zero_c_circuit(f, a, num_constraints):
    """A circuit whose C matrix is empty: (a) * (z) = 0 with the witness z = 0, repeated, and (x - a) * 1 = 0 binding the
    public input x = a.  Its c_val is the zero polynomial, which `DensePolynomial` stores with no coefficients at all, so a
    key file holds an empty coefficient vector that the loader must zero-pad back to |K|."""
    def gen(cs):
        va = cs.new_witness_variable(a)
        vz = cs.new_witness_variable(0)
        vx = cs.new_input_variable(a)
        for _ in range(num_constraints - 1):
            cs.enforce_constraint([(1, va)], [(1, vz)], [])
        cs.enforce_constraint([(1, vx), (f.p - 1, va)], [(1, ("i", 0))], [])
    return gen


class KeyWriter:
    """Both files of one oracle index.  `osrs`: oracle kzg.UniversalParams with generator g = curve.g (its trapdoor gives the
    G2 half); `opk`: omarlin.index(osrs, circuit, scheme)."""

    def __init__(self, osrs, opk, compressed):
        self.osrs, self.opk, self.compressed = osrs, opk, compressed
        self.curve = osrs.curve
        self.f = self.curve.fr
        self.marlin = opk.scheme == kzg.MARLIN
        self.g2 = ao.G2(self.curve)
        ck = opk.ck
        self.D = ck.max_degree
        self.bounds = ck.enforced_degree_bounds

    def g1(self, P):
        return ao.g1_bytes(self.curve, P, self.compressed)

    def g2b(self, P):
        return self.g2.compressed(P) if self.compressed else self.g2.uncompressed(P)

    def g2_power(self, e):
        return self.g2.smul(e % self.f.p, self.g2.gen)

    def info(self):
        i = self.opk.index.info
        return u64(i.num_variables) + u64(i.num_constraints) + u64(i.num_non_zero) + u64(i.num_instance_variables)

    def verifier_key(self):
        osrs, r = self.osrs, self.f.p
        out = self.info() + u64(6)
        for c in self.opk.index_comms:
            out += self.g1(c.comm) + (b"\x00" if self.marlin else b"")
        out += self.g1(osrs.g) + self.g1(osrs.gamma_g) + self.g2b(self.g2.gen) + self.g2b(self.g2_power(osrs.beta))
        md = self.opk.ck.supported_degree
        if self.marlin:
            out += b"\x01" + vec([u64(d) + self.g1(osrs.powers_of_g[self.D - d]) for d in self.bounds])
            out += u64(self.D) + u64(md)
        else:
            binv = pow(osrs.beta, -1, r)
            out += b"\x01" + vec([u64(d) + self.g2b(self.g2_power(pow(binv, self.D - d, r))) for d in self.bounds])
            out += u64(md) + u64(self.D)
        return out

    def prover_key(self):
        f, idx, ck, osrs = self.f, self.opk.index, self.opk.ck, self.osrs
        out = self.verifier_key()
        out += u64(6) + (u64(0) + (b"\x00" if self.marlin else b"")) * 6
        out += self.info()
        for m in (idx.a, idx.b, idx.c):
            out += vec([vec([fe(f, c) + u64(i) for c, i in row]) for row in m])
        by_label = {p.label: p for p in idx.polys}
        for label in LABELS:
            out += u64(len(label)) + label.encode() + vec([fe(f, c) for c in strip(by_label[label].coeffs)]) + b"\x00\x00"
        dom = domain(f, len(idx.evals["row"]))
        for name in EVAL_FIELDS:
            out += vec([fe(f, v) for v in idx.evals[name]]) + dom
        D = self.D
        powers = vec([self.g1(P) for P in osrs.powers_of_g[:ck.supported_degree + 1]])
        shifted = b"\x01" + vec([self.g1(P) for P in osrs.powers_of_g[D - self.bounds[-1]:D + 1]])
        gamma = vec([self.g1(P) for P in ck.powers_of_gamma_g])
        bounds = b"\x01" + vec([u64(d) for d in self.bounds])
        if self.marlin:
            out += powers + shifted + gamma + bounds + u64(D)
        else:
            sg = b"\x01" + u64(len(self.bounds))
            for d in self.bounds:
                sg += u64(d) + vec([self.g1(osrs.power_of_gamma_g(D - d + i)) for i in range(3) if D - d + i < D + 2])
            out += powers + gamma + shifted + sg + bounds + u64(D)
        return out
