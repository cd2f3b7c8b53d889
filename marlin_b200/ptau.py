"""snarkjs Powers-of-Tau (`.ptau`) files: the section framing, read through a memory map.

Layout [U snarkjs binfileutils, powersoftau_new.js, utils.writePTauHeader]: the magic `ptau`, u32 version (1), u32 section
count, then the sections in any order, each a u32 id, a u64 byte size and the data.  Section 1 (header) is u32 n8 (bytes of
an Fq), q as n8 little-endian bytes, u32 power, u32 ceremonyPower.  Section 2 `tauG1` holds 2^(power+1) - 1 G1 points,
section 3 `tauG2` 2^power G2 points, section 4 `alphaTauG1` 2^power G1 points, all in snarkjs's uncompressed "LEM" form
(b2m_g1_decode_lem / b2m_g2_decode_lem decode them).  Sections 5 (betaTauG1), 6 (betaG2), 7 (contributions) and the
Lagrange sections 12-15 of a prepared file are not read.  Files reach hundreds of GB: nothing beyond the section table and
the point prefixes a caller slices is read.
"""
import numpy as np

from . import _lib, fields

SECTION_NAMES = {1: "header", 2: "tauG1", 3: "tauG2", 4: "alphaTauG1", 5: "betaTauG1", 6: "betaG2", 7: "contributions"}
# q of the header -> curve id; snarkjs makes no BLS12-377 file
CURVE_OF_Q = {fields.FQ_MODULUS[_lib.CURVE_BN254]: _lib.CURVE_BN254, fields.FQ_MODULUS[_lib.CURVE_BLS12_381]: _lib.CURVE_BLS12_381}


def _section(sid):
    return f"section {sid} ({SECTION_NAMES[sid]})" if sid in SECTION_NAMES else f"section {sid}"


class PtauFile:
    """The framing of one .ptau file.  curve_id, n8, power, ceremony_power; tau_g1(n), tau_g2(n), alpha_tau_g1(n) are (n, point
    bytes) uint8 views of the first n points of sections 2-4 (memory-mapped: only what is read is loaded)."""

    def __init__(self, path):
        self.path = path
        mm = np.memmap(path, dtype=np.uint8, mode="r")
        size = len(mm)

        def u32(off):
            return int.from_bytes(bytes(mm[off:off + 4]), "little")

        def u64(off):
            return int.from_bytes(bytes(mm[off:off + 8]), "little")

        if size < 12 or bytes(mm[:4]) != b"ptau":
            raise ValueError(f"{path}: not a .ptau file (the magic is not 'ptau')")
        if u32(4) != 1:
            raise ValueError(f"{path}: .ptau version {u32(4)}, only version 1 is known")
        n_sections = u32(8)
        self.sections = {}
        off = 12
        for s in range(n_sections):
            if size - off < 12:
                raise ValueError(f"{path}: the header of section entry {s} runs past the end of the file")
            sid, ssize = u32(off), u64(off + 4)
            off += 12
            if ssize > size - off:
                raise ValueError(f"{path}: {_section(sid)} of {ssize} bytes runs past the end of the file")
            if sid in (1, 2, 3, 4) and sid in self.sections:
                raise ValueError(f"{path}: {_section(sid)} appears more than once")
            self.sections.setdefault(sid, (off, ssize))
            off += ssize
        for sid in (1, 2, 3, 4):
            if sid not in self.sections:
                raise ValueError(f"{path}: {_section(sid)} is missing")
        hoff, hsize = self.sections[1]
        if hsize < 4:
            raise ValueError(f"{path}: {_section(1)} is too short")
        n8 = u32(hoff)
        if hsize != 4 + n8 + 8:
            raise ValueError(f"{path}: {_section(1)} has {hsize} bytes, n8 = {n8} needs {4 + n8 + 8}")
        q = int.from_bytes(bytes(mm[hoff + 4:hoff + 4 + n8]), "little")
        if q not in CURVE_OF_Q:
            raise ValueError(f"{path}: {_section(1)}: q = {q:#x} is neither the BN254 nor the BLS12-381 base-field modulus")
        self.curve_id = CURVE_OF_Q[q]
        if n8 != 8 * _lib.LIMBS[self.curve_id][1]:
            raise ValueError(f"{path}: {_section(1)}: n8 = {n8} does not fit q")
        self.n8 = n8
        self.power, self.ceremony_power = u32(hoff + 4 + n8), u32(hoff + 8 + n8)
        if self.power < 1:
            raise ValueError(f"{path}: {_section(1)}: power {self.power} < 1")
        self.counts = {2: 2 ** (self.power + 1) - 1, 3: 2 ** self.power, 4: 2 ** self.power}
        self.point_bytes = {2: 2 * n8, 3: 4 * n8, 4: 2 * n8}
        for sid in (2, 3, 4):
            want = self.counts[sid] * self.point_bytes[sid]
            if self.sections[sid][1] != want:
                raise ValueError(f"{path}: {_section(sid)} has {self.sections[sid][1]} bytes, power {self.power} needs {want}")
        self._mm = mm

    def _points(self, sid, n):
        if n > self.counts[sid]:
            raise ValueError(f"{self.path}: {_section(sid)} holds {self.counts[sid]} points, not {n}")
        off = self.sections[sid][0]
        pb = self.point_bytes[sid]
        return self._mm[off:off + n * pb].reshape(n, pb)

    def tau_g1(self, n):
        return self._points(2, n)

    def tau_g2(self, n):
        return self._points(3, n)

    def alpha_tau_g1(self, n):
        return self._points(4, n)

    @property
    def max_degree(self):
        """the largest D a MarlinKZG10 SRS from this file can have: tauG1 holds D + 1 = 2^(power+1) - 1 powers"""
        return 2 ** (self.power + 1) - 2


def power_for_degree(D):
    """the smallest .ptau power whose tauG1 holds D + 1 powers"""
    p = 1
    while 2 ** (p + 1) - 2 < D:
        p += 1
    return p


def read_ptau(path):
    return PtauFile(path)
