"""SRS files in ark-serialize layout (SURVEY.md section 8 f-3): `kzg10::UniversalParams<E>` written field by field with
`CanonicalSerialize::serialize_uncompressed` [U ark-poly-commit 0.3 kzg10/data_structures.rs, ark-serialize 0.3]:

    powers_of_g        : Vec<G1Affine>             u64-LE length, then the points
    powers_of_gamma_g  : BTreeMap<usize, G1Affine> u64-LE length, then (u64-LE key, point) in ascending key order
    h, beta_h          : G2Affine
    neg_powers_of_h    : BTreeMap<usize, G2Affine> as above (SonicKZG10: the entries its `trim` reads, max_degree - bound)

A point is its canonical little-endian coordinates (x || y; over Fq2: c0 || c1 each) with the infinity flag in bit 6 of the
last byte.  tools/replay_rs reads this file with `deserialize_unchecked` into the public fields of `UniversalParams`, so an SRS
made on the GPU can be replayed through the real `ark_marlin::Marlin::{index, prove, verify}`.  All group arithmetic and the
Montgomery <-> canonical conversions happen in libb2m (GPU for G1, host C++ for the few G2 points); this module only moves bytes.
"""
import os
import struct
from collections.abc import Mapping

import numpy as np

from . import _lib

MAGIC = b"B2MSRS01"  # 8-byte tag + curve id (u64) ahead of the ark-serialize payload, so that a wrong-curve load fails loudly


def fq_bytes(curve_id):
    return 8 * _lib.LIMBS[curve_id][1]


def write_srs(path, curve_id, powers, gamma, h, beta_h, neg_powers):
    """powers: bytes (n * 2 * fq_bytes); gamma: {index: bytes}; h, beta_h: bytes (4 * fq_bytes); neg_powers: {index: bytes}"""
    g1, g2 = 2 * fq_bytes(curve_id), 4 * fq_bytes(curve_id)
    assert len(powers) % g1 == 0 and len(h) == g2 and len(beta_h) == g2
    with open(path, "wb") as f:
        f.write(MAGIC + struct.pack("<Q", curve_id))
        f.write(struct.pack("<Q", len(powers) // g1))
        f.write(powers)
        f.write(struct.pack("<Q", len(gamma)))
        for k in sorted(gamma):
            assert len(gamma[k]) == g1
            f.write(struct.pack("<Q", k) + gamma[k])
        f.write(h + beta_h)
        f.write(struct.pack("<Q", len(neg_powers)))
        for k in sorted(neg_powers):
            assert len(neg_powers[k]) == g2
            f.write(struct.pack("<Q", k) + neg_powers[k])


def read_srs(path):
    """-> dict(curve_id, powers (bytes), gamma {index: bytes}, h, beta_h, neg_powers {index: bytes})"""
    with open(path, "rb") as f:
        head = f.read(16)
        if head[:8] != MAGIC:
            raise ValueError(f"{path}: not a b2m SRS file")
        curve_id = struct.unpack("<Q", head[8:])[0]
        if curve_id not in _lib.LIMBS:
            raise ValueError(f"{path}: unknown curve id {curve_id}")
        g1, g2 = 2 * fq_bytes(curve_id), 4 * fq_bytes(curve_id)

        def u64():
            b = f.read(8)
            if len(b) != 8:
                raise ValueError(f"{path}: truncated")
            return struct.unpack("<Q", b)[0]

        def blob(n):
            b = f.read(n)
            if len(b) != n:
                raise ValueError(f"{path}: truncated")
            return b

        n = u64()
        powers = blob(n * g1)
        gamma = {}
        for _ in range(u64()):
            k = u64()
            gamma[k] = blob(g1)
        h, beta_h = blob(g2), blob(g2)
        neg = {}
        for _ in range(u64()):
            k = u64()
            neg[k] = blob(g2)
        if f.read(1):
            raise ValueError(f"{path}: trailing bytes")
    return {"curve_id": curve_id, "powers": powers, "gamma": gamma, "h": h, "beta_h": beta_h, "neg_powers": neg}


def g2_setup(curve_id, r, beta, max_degree, degree_bounds):
    """h (the standard G2 generator), beta * h and beta^-(max_degree - d) * h per enforced bound d, as uncompressed bytes."""
    L = _lib.lib()
    exps = [1, beta % r] + [pow(pow(beta % r, max_degree - d, r), -1, r) for d in sorted(set(degree_bounds))]
    sc = _lib.ints_to_limbs(exps, 4)
    g2 = 4 * fq_bytes(curve_id)
    out = np.zeros(len(exps) * g2, dtype=np.uint8)
    _lib.check(L.b2m_g2_scalar_muls(curve_id, None, _lib.ptr(sc), len(exps), _lib.ptr(out)))
    raw = out.tobytes()
    pts = [raw[i * g2:(i + 1) * g2] for i in range(len(exps))]
    return pts[0], pts[1], {max_degree - d: pts[2 + i] for i, d in enumerate(sorted(set(degree_bounds)))}


# ---- raw arkworks layout ----------------------------------------------------------------------------------------------------
# `kzg10::UniversalParams<E>` exactly as `CanonicalSerialize::serialize` (compressed) or `serialize_uncompressed` writes it
# [U ark-poly-commit 0.3, ark-serialize 0.3]: the fields above in the same order, no header.  A compressed G1 point is x alone
# (sizeof(Fq) bytes), a compressed G2 point x.c0 || x.c1, flags in the top bits of the last byte.  Marlin.load_ark_srs decodes
# and validates every point on the GPU; this module only checks the framing.

def point_sizes(curve_id, compressed):
    """(G1, G2) point sizes in bytes of the compressed or uncompressed form"""
    nb = fq_bytes(curve_id)
    return (nb, 2 * nb) if compressed else (2 * nb, 4 * nb)


def read_ark(path, curve_id, compressed):
    """Parse a raw `UniversalParams` file.  Every length field is checked against the bytes left in the file before anything
    is sliced, and truncation, trailing bytes and BTreeMap keys that are not strictly ascending are rejected (ValueError).
    -> dict(powers: uint8 (n, g1), gamma_keys: uint64 (m,), gamma: uint8 (m, g1), h, beta_h: uint8 (g2,),
            neg_keys: uint64 (k,), neg: uint8 (k, g2)); `powers` is a read-only view of the memory-mapped file."""
    if curve_id not in _lib.LIMBS:
        raise ValueError(f"unknown curve id {curve_id}")
    g1, g2 = point_sizes(curve_id, compressed)
    size = os.path.getsize(path)
    buf = np.memmap(path, dtype=np.uint8, mode="r") if size else np.zeros(0, dtype=np.uint8)
    pos = 0

    def u64(what):
        nonlocal pos
        if size - pos < 8:
            raise ValueError(f"{path}: truncated in the length of {what}")
        v = int.from_bytes(bytes(buf[pos:pos + 8]), "little")
        pos += 8
        return v

    def take(count, stride, what):
        nonlocal pos
        if count > (size - pos) // stride:
            raise ValueError(f"{path}: {what} claims {count} entries of {stride} bytes, the file has {size - pos} bytes left")
        a = buf[pos:pos + count * stride].reshape(count, stride)
        pos += count * stride
        return a

    def btree(point, what):
        ent = take(u64(what), 8 + point, what)
        keys = np.ascontiguousarray(ent[:, :8]).view("<u8").reshape(-1).astype(np.uint64)
        if len(keys) > 1 and not bool(np.all(keys[1:] > keys[:-1])):
            raise ValueError(f"{path}: the keys of {what} are not strictly ascending")
        return keys, np.ascontiguousarray(ent[:, 8:])

    powers = take(u64("powers_of_g"), g1, "powers_of_g")
    gamma_keys, gamma = btree(g1, "powers_of_gamma_g")
    h = np.ascontiguousarray(take(1, g2, "h")[0])
    beta_h = np.ascontiguousarray(take(1, g2, "beta_h")[0])
    neg_keys, neg = btree(g2, "neg_powers_of_h")
    if pos != size:
        raise ValueError(f"{path}: {size - pos} trailing bytes")
    return {"powers": powers, "gamma_keys": gamma_keys, "gamma": gamma, "h": h, "beta_h": beta_h, "neg_keys": neg_keys, "neg": neg}


def write_ark(path, curve_id, compressed, powers, gamma_keys, gamma, h, beta_h, neg_keys, neg):
    """Write a raw `UniversalParams` file (read_ark's layout); points are byte arrays already in the chosen form."""
    g1, g2 = point_sizes(curve_id, compressed)

    def btree(keys, pts, point):
        keys = np.asarray(keys, dtype=np.uint64)
        pts = np.asarray(pts, dtype=np.uint8).reshape(len(keys), point)
        if len(keys) > 1 and not bool(np.all(keys[1:] > keys[:-1])):
            raise ValueError("BTreeMap keys must be strictly ascending")
        ent = np.empty((len(keys), 8 + point), dtype=np.uint8)
        ent[:, :8] = keys.astype("<u8").view(np.uint8).reshape(-1, 8)
        ent[:, 8:] = pts
        return struct.pack("<Q", len(keys)), ent

    powers = np.asarray(powers, dtype=np.uint8).reshape(-1, g1)
    h, beta_h = np.asarray(h, dtype=np.uint8).reshape(g2), np.asarray(beta_h, dtype=np.uint8).reshape(g2)
    gl, ge = btree(gamma_keys, gamma, g1)
    nl, ne = btree(neg_keys, neg, g2)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(powers)))
        f.write(memoryview(np.ascontiguousarray(powers)))
        f.write(gl)
        f.write(memoryview(ge))
        f.write(memoryview(h))
        f.write(memoryview(beta_h))
        f.write(nl)
        f.write(memoryview(ne))


class G2Points(Mapping):
    """{index: uncompressed G2 bytes} over one contiguous array (keys sorted ascending), so that millions of
    neg_powers_of_h cost one buffer rather than one Python object each."""

    def __init__(self, keys, points):
        self.keys_arr = np.asarray(keys, dtype=np.uint64)
        points = np.asarray(points, dtype=np.uint8)
        self.points = points if points.ndim == 2 else points.reshape(len(self.keys_arr), -1)

    def _find(self, k):
        if not isinstance(k, (int, np.integer)) or k < 0:
            return -1
        i = int(np.searchsorted(self.keys_arr, np.uint64(k)))
        return i if i < len(self.keys_arr) and int(self.keys_arr[i]) == k else -1

    def __getitem__(self, k):
        i = self._find(k)
        if i < 0:
            raise KeyError(k)
        return self.points[i].tobytes()

    def __contains__(self, k):
        return self._find(k) >= 0

    def __iter__(self):
        return (int(k) for k in self.keys_arr)

    def __len__(self):
        return len(self.keys_arr)
