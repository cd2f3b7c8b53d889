"""circom `.r1cs` and `.wtns` files: the iden3 binary container, read through a memory map.

Layout [U circom r1csfile / snarkjs wtns_utils, recalled, not pinned]: all integers little-endian; a 4-byte magic, u32
version, u32 section count, then the sections in any order, each a u32 type, a u64 byte size and the data.  Unknown
section types are skipped.
- `.r1cs` (magic `r1cs`, version 1).  Section 1 (header): u32 n8, the prime (n8 bytes), u32 nWires, u32 nPubOut, u32 nPubIn,
  u32 nPrvIn, u64 nLabels, u32 mConstraints; 32 + n8 bytes.  Section 2 (constraints): mConstraints records of three linear
  combinations A, B, C, each a u32 term count and that many (u32 wire, n8-byte canonical coefficient) terms, decoded on the
  GPU (b2m_circom_decode_constraints).  Section 3 (wire -> label map) is not read.  Sections 4 and 5 (PLONK custom gates,
  circom >= 2.0.6) are refused: they are not R1CS constraints.
- `.wtns` (magic `wtns`, version 2).  Section 1: u32 n8, the prime, u32 nWitness.  Section 2: nWitness canonical values,
  one per wire, wire 0 the constant one (decoded on the GPU by b2m_fr_decode_ark).
Only n8 = 32 is accepted; the prime must be the Fr modulus of the prover's curve (Marlin.load_r1cs / load_wtns check it).
Nothing beyond the section table, the headers and the slices a caller reads is loaded.
"""
import ctypes
import os
from collections import namedtuple

import numpy as np

from . import _lib, fields

R1CS_SECTIONS = {1: "header", 2: "constraints", 3: "wire2LabelId", 4: "customGatesList", 5: "customGatesApplication"}
WTNS_SECTIONS = {1: "header", 2: "witness"}
MATRICES = "ABC"
TERM_BYTES = 36  # u32 wire + 32-byte coefficient

# the circom header fields an instance keeps (R1CS.circom)
CircomInfo = namedtuple("CircomInfo", "n_wires n_pub_out n_pub_in n_prv_in m_constraints")


def curve_of_prime(prime):
    """the curve id whose Fr modulus is `prime`, or None"""
    return next((cid for cid, r in fields.FR_MODULUS.items() if r == prime), None)


def _section(names, sid):
    return f"section {sid} ({names[sid]})" if sid in names else f"section {sid}"


def _container(path, magic, version, names, required):
    """memory map, section table {id: (offset, size)} of an iden3 binary file; every framing error names its section"""
    size = os.path.getsize(path)
    if size < 12:
        raise ValueError(f"{path}: not a .{magic} file (shorter than its 12-byte preamble)")
    mm = np.memmap(path, dtype=np.uint8, mode="r")
    u32 = lambda off: int.from_bytes(bytes(mm[off:off + 4]), "little")  # noqa: E731
    u64 = lambda off: int.from_bytes(bytes(mm[off:off + 8]), "little")  # noqa: E731
    if bytes(mm[:4]) != magic.encode():
        raise ValueError(f"{path}: not a .{magic} file (the magic is not '{magic}')")
    if u32(4) != version:
        raise ValueError(f"{path}: .{magic} version {u32(4)}, only version {version} is known")
    sections = {}
    off = 12
    for s in range(u32(8)):
        if size - off < 12:
            raise ValueError(f"{path}: the header of section entry {s} runs past the end of the file")
        sid, ssize = u32(off), u64(off + 4)
        off += 12
        if ssize > size - off:
            raise ValueError(f"{path}: {_section(names, sid)} of {ssize} bytes runs past the end of the file")
        if sid in required and sid in sections:
            raise ValueError(f"{path}: {_section(names, sid)} appears more than once")
        sections.setdefault(sid, (off, ssize))
        off += ssize
    for sid in required:
        if sid not in sections:
            raise ValueError(f"{path}: {_section(names, sid)} is missing")
    return mm, sections, u32, u64


class R1csFile:
    """The framing of one .r1cs file: n8, prime, n_wires, n_pub_out, n_pub_in, n_prv_in, n_labels, m (mConstraints) and
    `constraints`, a uint8 view of section 2 (memory-mapped)."""

    def __init__(self, path):
        self.path = path
        mm, secs, u32, u64 = _container(path, "r1cs", 1, R1CS_SECTIONS, (1, 2))
        for sid in (4, 5):
            if sid in secs:
                raise ValueError(f"{path}: {_section(R1CS_SECTIONS, sid)}: PLONK custom gates are not R1CS constraints")
        hoff, hsize = secs[1]
        h = _section(R1CS_SECTIONS, 1)
        if hsize < 4:
            raise ValueError(f"{path}: {h} is too short")
        n8 = u32(hoff)
        if hsize != 32 + n8:
            raise ValueError(f"{path}: {h} has {hsize} bytes, n8 = {n8} needs {32 + n8}")
        if n8 != 32:
            raise ValueError(f"{path}: {h}: n8 = {n8}, only 32-byte fields are supported")
        self.n8 = n8
        self.prime = int.from_bytes(bytes(mm[hoff + 4:hoff + 4 + n8]), "little")
        o = hoff + 4 + n8
        self.n_wires, self.n_pub_out, self.n_pub_in, self.n_prv_in = (u32(o + 4 * i) for i in range(4))
        self.n_labels, self.m = u64(o + 16), u32(o + 24)
        if self.n_wires < 1 + self.n_pub_out + self.n_pub_in:
            raise ValueError(f"{path}: {h}: nWires = {self.n_wires} < 1 + nPubOut + nPubIn = {1 + self.n_pub_out + self.n_pub_in}")
        coff, csize = secs[2]
        self.constraints = mm[coff:coff + csize]
        self._mm = mm

    @property
    def ni0(self):
        """formatted inputs before padding: One, the public outputs, the public inputs"""
        return 1 + self.n_pub_out + self.n_pub_in

    def info(self):
        return CircomInfo(self.n_wires, self.n_pub_out, self.n_pub_in, self.n_prv_in, self.m)


class WtnsFile:
    """The framing of one .wtns file: n8, prime, n_witness and `values`, an (n_witness, n8) uint8 view of section 2."""

    def __init__(self, path):
        self.path = path
        mm, secs, u32, _ = _container(path, "wtns", 2, WTNS_SECTIONS, (1, 2))
        hoff, hsize = secs[1]
        h = _section(WTNS_SECTIONS, 1)
        if hsize < 4:
            raise ValueError(f"{path}: {h} is too short")
        n8 = u32(hoff)
        if hsize != 8 + n8:
            raise ValueError(f"{path}: {h} has {hsize} bytes, n8 = {n8} needs {8 + n8}")
        if n8 != 32:
            raise ValueError(f"{path}: {h}: n8 = {n8}, only 32-byte fields are supported")
        self.n8 = n8
        self.prime = int.from_bytes(bytes(mm[hoff + 4:hoff + 4 + n8]), "little")
        self.n_witness = u32(hoff + 4 + n8)
        woff, wsize = secs[2]
        if wsize != self.n_witness * n8:
            raise ValueError(f"{path}: {_section(WTNS_SECTIONS, 2)} has {wsize} bytes, nWitness = {self.n_witness} needs {self.n_witness * n8}")
        self.values = mm[woff:woff + wsize].reshape(self.n_witness, n8)


def read_r1cs(path):
    return R1csFile(path)


def read_wtns(path):
    return WtnsFile(path)


def check_prime(path, section, prime, curve_id):
    """the file's prime must be the Fr modulus of curve_id; a mismatch names the curve the prime belongs to, if any"""
    if prime == fields.FR_MODULUS[curve_id]:
        return
    names = {v: k for k, v in fields.CURVE_IDS.items()}
    other = curve_of_prime(prime)
    what = f"the {names[other]} scalar field" if other is not None else "the scalar field of no supported curve"
    raise ValueError(f"{path}: {section}: the prime {prime:#x} is {what}, this Marlin instance is {names[curve_id]}")


def constraint_rows(f):
    """The host walk over section 2 (b2m_circom_constraint_rows): three term-count prefix sums (u64[m + 1] each).  A
    truncated section, or one longer than its m constraints, raises naming the section and the constraint."""
    rps = [np.zeros(f.m + 1, dtype=np.uint64) for _ in range(3)]
    end, bc, br = ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_int(0)
    data = f.constraints
    L = _lib.lib()
    rc = L.b2m_circom_constraint_rows(data.ctypes.data if len(data) else None, len(data), f.m, *[_lib.ptr(r) for r in rps], ctypes.byref(end),
                                      ctypes.byref(bc), ctypes.byref(br))
    sec = _section(R1CS_SECTIONS, 2)
    if rc == _lib.ERR_SERIALIZATION:
        raise ValueError(f"{f.path}: {sec}: {L.b2m_last_error().decode()}")
    _lib.check(rc)
    if end.value != len(data):
        raise ValueError(f"{f.path}: {sec} has {len(data)} bytes, its {f.m} constraints take {end.value}")
    return rps


def term_offset(rps, k, j, i):
    """byte offset in section 2 of term i of LC j (0/1/2 = A/B/C) of constraint k"""
    before = sum(int(r[k]) for r in rps) + sum(int(rps[q][k + 1] - rps[q][k]) for q in range(j))
    return 4 * (3 * k + j) + TERM_BYTES * (before + i) + 4
