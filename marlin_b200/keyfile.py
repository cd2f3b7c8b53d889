"""Index key files in ark-serialize layout: the `IndexProverKey` and `IndexVerifierKey` that `Marlin::index` returns
[reference src/data_structures.rs:24-80, src/ahp/indexer.rs:28-127, src/ahp/constraint_systems.rs:87-123], written field by
field as `CanonicalSerialize::serialize` (compressed points) or `serialize_uncompressed` writes them, with no header.

The layouts below are recalled from ark-serialize / ark-poly / ark-poly-commit 0.3 [U] and are not yet pinned against the
real types: the tests compare with an independent writer built from the same recollection.  tools/replay_rs (source, run
where a Rust toolchain and the arkworks crates are available) is the check that pins them: it `deserialize`s the files
tools/make_replay_kit.py writes into the real `IndexProverKey` / `IndexVerifierKey` and byte-diffs them against its own
`Marlin::index` output.

`usize` is a u64 LE value; `Vec<T>` and `String` are a u64 length and then the items or bytes; `Option<T>` is one byte (0 or 1) and then the value; a tuple is its members in order; `PhantomData` writes nothing; F is its canonical
32-byte LE value; G1 / G2 points are as in srsfile.point_sizes.

    IndexVerifierKey  index_info     num_variables, num_constraints, num_non_zero, num_instance_variables
                      index_comms    Vec of 6 PC::Commitment: MarlinKZG10 G1 + Option<shifted G1> (always None here),
                                     SonicKZG10 a bare G1
                      verifier_key   MarlinKZG10: g, gamma_g, h, beta_h, Option<Vec<(usize, G1)>> shift powers,
                                                  max_degree, supported_degree
                                     SonicKZG10:  g, gamma_g, h, beta_h, Option<Vec<(usize, G2)>> neg powers of h,
                                                  supported_degree, max_degree
    IndexProverKey    index_vk       as above
                      index_comm_rands  Vec of 6 empty randomness values: MarlinKZG10 u64 0 + None, SonicKZG10 u64 0
                      index          index_info; a, b, c as Vec<Vec<(F, usize)>>; joint_arith = six LabeledPolynomial
                                     (label String, Vec<F> coefficients without trailing zeros, degree_bound None,
                                     hiding_bound None) in the order row, col, a_val, b_val, c_val, row_col, then
                                     evals_on_K in the order row, col, row_col, val_a, val_b, val_c, each Vec<F> + domain
                                     (u8 tag 0, size u64, log_size_of_group u32, five F: b2m_domain_ark)
                      committer_key  MarlinKZG10: powers, Option<shifted_powers>, powers_of_gamma_g,
                                                  Option<enforced_degree_bounds>, max_degree
                                     SonicKZG10:  powers_of_g, powers_of_gamma_g, Option<shifted_powers_of_g>,
                                                  Option<BTreeMap<usize, Vec<G1>>> shifted_powers_of_gamma_g,
                                                  Option<enforced_degree_bounds>, max_degree

This module only frames bytes: every length is checked against the bytes left before anything is sliced, and truncation,
trailing bytes, option bytes other than 0 / 1, map keys that are not strictly ascending, a wrong label or domain tag and
non-empty commitment randomness raise ValueError naming the field.  Points and field elements are decoded and validated on
the GPU by Marlin.load_index / Marlin.load_verifier_key.  Vectors are returned as (n, 32) or (n, point size) uint8 views of
the memory-mapped file.
"""
import ctypes
import os
import struct

import numpy as np

from . import _lib
from .srsfile import point_sizes

FR_BYTES = 32
DOMAIN_BYTES = 8 + 4 + 5 * FR_BYTES
POLY_LABELS = ("row", "col", "a_val", "b_val", "c_val", "row_col")   # joint_arith polynomials, index-polynomial order
EVAL_NAMES = ("row", "col", "row_col", "val_a", "val_b", "val_c")    # evals_on_K fields, in file order
EVAL_OF_POLY = (0, 1, 3, 4, 5, 2)                                    # evals_on_K position of polynomial i
MATRICES = ("a", "b", "c")


class _Reader:
    def __init__(self, path):
        self.path = path
        self.size = os.path.getsize(path)
        self.buf = np.memmap(path, dtype=np.uint8, mode="r") if self.size else np.zeros(0, dtype=np.uint8)
        self.pos = 0

    def fail(self, field, msg):
        raise ValueError(f"{self.path}: {field}: {msg}")

    def _int(self, n, field):
        if self.size - self.pos < n:
            self.fail(field, f"truncated ({self.size - self.pos} bytes left, {n} needed)")
        v = int.from_bytes(bytes(self.buf[self.pos:self.pos + n]), "little")
        self.pos += n
        return v

    def u64(self, field):
        return self._int(8, field)

    def u8(self, field):
        return self._int(1, field)

    def option(self, field):
        b = self.u8(field)
        if b > 1:
            self.fail(field, f"option byte {b} is neither 0 nor 1")
        return b == 1

    def take(self, count, stride, field):
        if count > (self.size - self.pos) // stride:
            self.fail(field, f"claims {count} entries of {stride} bytes, the file has {self.size - self.pos} bytes left")
        a = self.buf[self.pos:self.pos + count * stride].reshape(count, stride)
        self.pos += count * stride
        return a

    def vec(self, stride, field):
        return self.take(self.u64(field), stride, field)

    def keyed(self, stride, field):
        """Vec<(usize, T)> -> (keys uint64, items (n, stride))"""
        ent = self.vec(8 + stride, field)
        return np.ascontiguousarray(ent[:, :8]).view("<u8").reshape(-1).astype(np.uint64), ent[:, 8:]

    def matrix(self, field):
        """Matrix<F> = Vec<Vec<(F, usize)>> -> (row_ptr uint64 (n + 1), col uint64 (nnz), coeff uint8 (nnz, 32)).  The row
        lengths are a chain of offsets, walked in libb2m (b2m_ark_matrix_rows); the entries are then de-interleaved with one
        mask."""
        nrows = self.u64(field)
        start, size, buf = self.pos, self.size, self.buf
        if nrows > (size - start) // 8:
            self.fail(field, f"claims {nrows} rows, the file has {size - start} bytes left")
        row_ptr = np.zeros(nrows + 1, dtype=np.uint64)
        end, bad_row, bad_reason = ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_int(0)
        rc = _lib.lib().b2m_ark_matrix_rows(buf[start:].ctypes.data if size > start else None, size - start, nrows, FR_BYTES + 8,
                                            _lib.ptr(row_ptr), ctypes.byref(end), ctypes.byref(bad_row), ctypes.byref(bad_reason))
        if rc == _lib.ERR_SERIALIZATION:
            at = start + end.value  # the failing row's length field
            if bad_reason.value == 1:
                self.fail(f"{field}[{bad_row.value}]", "truncated in the row length")
            n = struct.unpack_from("<Q", buf, at)[0]
            self.fail(f"{field}[{bad_row.value}]", f"claims {n} entries, the file has {size - at - 8} bytes left")
        _lib.check(rc)
        pos = start + end.value
        self.pos = pos
        section = buf[start:pos]
        keep = np.ones(pos - start, dtype=bool)
        hdr = 8 * np.arange(nrows, dtype=np.int64) + (FR_BYTES + 8) * row_ptr[:-1].astype(np.int64)
        keep[(hdr[:, None] + np.arange(8)).reshape(-1)] = False
        ent = section[keep].reshape(-1, FR_BYTES + 8)
        col = np.ascontiguousarray(ent[:, FR_BYTES:]).view("<u8").reshape(-1).astype(np.uint64)
        return row_ptr, col, np.ascontiguousarray(ent[:, :FR_BYTES])

    def end(self):
        if self.pos != self.size:
            raise ValueError(f"{self.path}: {self.size - self.pos} trailing bytes")


def _read_vk(r, field, curve_id, pc, compressed):
    g1, g2 = point_sizes(curve_id, compressed)
    marlin = pc == _lib.PC_MARLIN_KZG10
    info = tuple(r.u64(f"{field}.index_info.{k}") for k in ("num_variables", "num_constraints", "num_non_zero", "num_instance_variables"))
    n = r.u64(f"{field}.index_comms")
    if n != 6:
        r.fail(f"{field}.index_comms", f"holds {n} commitments, an index has 6")
    ent = r.take(6, g1 + (1 if marlin else 0), f"{field}.index_comms")
    if marlin:
        flags = ent[:, g1]
        bad = np.flatnonzero(flags != 0)
        if len(bad):
            i = int(bad[0])
            r.fail(f"{field}.index_comms[{i}].shifted_comm", "is not None (index polynomials have no degree bound)" if flags[i] == 1
                   else f"option byte {int(flags[i])} is neither 0 nor 1")
    vk = {"info": info, "comms": np.ascontiguousarray(ent[:, :g1])}
    vf = f"{field}.verifier_key"
    vk["g"] = r.take(1, g1, f"{vf}.g")[0]
    vk["gamma_g"] = r.take(1, g1, f"{vf}.gamma_g")[0]
    vk["h"] = r.take(1, g2, f"{vf}.h")[0]
    vk["beta_h"] = r.take(1, g2, f"{vf}.beta_h")[0]
    name = "degree_bounds_and_shift_powers" if marlin else "degree_bounds_and_neg_powers_of_h"
    if r.option(f"{vf}.{name}"):
        vk["bounds"], vk["bound_points"] = r.keyed(g1 if marlin else g2, f"{vf}.{name}")
    else:
        vk["bounds"], vk["bound_points"] = np.zeros(0, dtype=np.uint64), np.zeros((0, g1 if marlin else g2), dtype=np.uint8)
    if marlin:
        vk["max_degree"], vk["supported_degree"] = r.u64(f"{vf}.max_degree"), r.u64(f"{vf}.supported_degree")
    else:
        vk["supported_degree"], vk["max_degree"] = r.u64(f"{vf}.supported_degree"), r.u64(f"{vf}.max_degree")
    return vk


def read_verifier_key(path, curve_id, pc, compressed):
    """Parse an `IndexVerifierKey` file -> dict(info (4 ints), comms (6, g1), g, gamma_g, h, beta_h, bounds uint64 (n,),
    bound_points (n, g1 or g2), supported_degree, max_degree)."""
    r = _Reader(path)
    vk = _read_vk(r, "index_vk", curve_id, pc, compressed)
    r.end()
    return vk


def read_prover_key(path, curve_id, pc, compressed):
    """Parse an `IndexProverKey` file -> dict(vk (as read_verifier_key), index, ck).  index = dict(info, matrices [(row_ptr,
    col, coeff bytes)] * 3, coeffs [6 x (n_i, 32)] and evals [6 x (K, 32)] in index-polynomial order, domains [6 x bytes]).
    ck: MarlinKZG10 dict(powers, shifted (or None), gamma, bounds (or None), max_degree); SonicKZG10 dict(powers, gamma,
    shifted, shifted_gamma ({bound: (n, g1)} or None), bounds, max_degree)."""
    g1, _ = point_sizes(curve_id, compressed)
    marlin = pc == _lib.PC_MARLIN_KZG10
    r = _Reader(path)
    vk = _read_vk(r, "index_vk", curve_id, pc, compressed)
    n = r.u64("index_comm_rands")
    if n != 6:
        r.fail("index_comm_rands", f"holds {n} values, an index has 6")
    for i in range(6):
        f = f"index_comm_rands[{i}]"
        if r.u64(f"{f}.blinding_polynomial") != 0:
            r.fail(f"{f}.blinding_polynomial", "is not empty (index polynomials are committed without hiding)")
        if marlin and r.option(f"{f}.shifted_rand"):
            r.fail(f"{f}.shifted_rand", "is not None (index polynomials have no degree bound)")
    info = tuple(r.u64(f"index.index_info.{k}") for k in ("num_variables", "num_constraints", "num_non_zero", "num_instance_variables"))
    if info != vk["info"]:
        r.fail("index.index_info", f"{info} differs from index_vk.index_info {vk['info']}")
    mats = [r.matrix(f"index.{m}") for m in MATRICES]
    coeffs = []
    for label in POLY_LABELS:
        f = f"index.joint_arith.{label}"
        got = bytes(r.vec(1, f"{f}.label").reshape(-1))
        if got != label.encode():
            r.fail(f"{f}.label", f"is {got!r}, expected {label!r}")
        coeffs.append(r.vec(FR_BYTES, f"{f}.polynomial"))
        if r.option(f"{f}.degree_bound"):
            r.fail(f"{f}.degree_bound", "is not None")
        if r.option(f"{f}.hiding_bound"):
            r.fail(f"{f}.hiding_bound", "is not None")
    evals, domains = [None] * 6, [None] * 6
    for name in EVAL_NAMES:
        f = f"index.joint_arith.evals_on_K.{name}"
        ev = r.vec(FR_BYTES, f"{f}.evals")
        tag = r.u8(f"{f}.domain")
        if tag != 0:
            r.fail(f"{f}.domain", f"tag {tag} is not 0 (Radix2)")
        dom = bytes(r.take(1, DOMAIN_BYTES, f"{f}.domain")[0])
        i = EVAL_OF_POLY.index(EVAL_NAMES.index(name))
        evals[i], domains[i] = ev, dom
    index = {"info": info, "matrices": mats, "coeffs": coeffs, "evals": evals, "domains": domains}
    ck = {}
    if marlin:
        ck["powers"] = r.vec(g1, "committer_key.powers")
        ck["shifted"] = r.vec(g1, "committer_key.shifted_powers") if r.option("committer_key.shifted_powers") else None
        ck["gamma"] = r.vec(g1, "committer_key.powers_of_gamma_g")
    else:
        ck["powers"] = r.vec(g1, "committer_key.powers_of_g")
        ck["gamma"] = r.vec(g1, "committer_key.powers_of_gamma_g")
        ck["shifted"] = r.vec(g1, "committer_key.shifted_powers_of_g") if r.option("committer_key.shifted_powers_of_g") else None
        ck["shifted_gamma"] = None
        f = "committer_key.shifted_powers_of_gamma_g"
        if r.option(f):
            m, prev = {}, None
            for _ in range(r.u64(f)):
                k = r.u64(f"{f} key")
                if prev is not None and k <= prev:
                    r.fail(f, f"key {k} after {prev}: the keys are not strictly ascending")
                m[k] = r.vec(g1, f"{f}[{k}]")
                prev = k
            ck["shifted_gamma"] = m
    ck["bounds"] = [int(x) for x in r.vec(8, "committer_key.enforced_degree_bounds").view("<u8").reshape(-1)] \
        if r.option("committer_key.enforced_degree_bounds") else None
    ck["max_degree"] = r.u64("committer_key.max_degree")
    r.end()
    return {"vk": vk, "index": index, "ck": ck}


# ---- writers ----------------------------------------------------------------------------------------------------------
def _u64(v):
    return struct.pack("<Q", v)


def _vec(a):
    a = np.ascontiguousarray(a, dtype=np.uint8)
    return [_u64(len(a)), memoryview(a.reshape(-1))]


def _keyed(keys, pts):
    keys = np.asarray(keys, dtype=np.uint64)
    pts = np.asarray(pts, dtype=np.uint8).reshape(len(keys), -1)
    ent = np.empty((len(keys), 8 + pts.shape[1]), dtype=np.uint8)
    ent[:, :8] = keys.astype("<u8").view(np.uint8).reshape(-1, 8)
    ent[:, 8:] = pts
    return _vec(ent)


def _matrix(row_ptr, col, coeff):
    row_ptr = np.asarray(row_ptr, dtype=np.int64)
    nrows, ne = len(row_ptr) - 1, int(row_ptr[-1])
    ent = np.empty((ne, FR_BYTES + 8), dtype=np.uint8)
    ent[:, :FR_BYTES] = np.asarray(coeff, dtype=np.uint8).reshape(-1, FR_BYTES)[:ne]
    ent[:, FR_BYTES:] = np.asarray(col[:ne], dtype=np.uint64).astype("<u8").view(np.uint8).reshape(-1, 8)
    out = np.empty(8 * nrows + (FR_BYTES + 8) * ne, dtype=np.uint8)
    hdr = 8 * np.arange(nrows, dtype=np.int64) + (FR_BYTES + 8) * row_ptr[:-1]
    is_hdr = np.zeros(len(out), dtype=bool)
    is_hdr[(hdr[:, None] + np.arange(8)).reshape(-1)] = True
    out[is_hdr] = np.diff(row_ptr).astype("<u8").view(np.uint8)
    out[~is_hdr] = ent.reshape(-1)
    return [_u64(nrows), memoryview(out)]


def strip_zeros(coeffs):
    """`DensePolynomial::from_coefficients_vec` drops zero high coefficients: (n, 32) -> the prefix up to the last non-zero"""
    nz = np.flatnonzero(np.asarray(coeffs).any(axis=1))
    return coeffs[:int(nz[-1]) + 1] if len(nz) else coeffs[:0]


def _vk_parts(pc, vk):
    marlin = pc == _lib.PC_MARLIN_KZG10
    out = [b"".join(_u64(v) for v in vk["info"]), _u64(6)]
    comms = np.asarray(vk["comms"], dtype=np.uint8)
    for c in comms:
        out += [memoryview(np.ascontiguousarray(c)), b"\x00" if marlin else b""]
    out += [memoryview(np.ascontiguousarray(vk[k], dtype=np.uint8).reshape(-1)) for k in ("g", "gamma_g", "h", "beta_h")]
    out += [b"\x01"] + _keyed(vk["bounds"], vk["bound_points"])
    if marlin:
        out += [_u64(vk["max_degree"]), _u64(vk["supported_degree"])]
    else:
        out += [_u64(vk["supported_degree"]), _u64(vk["max_degree"])]
    return out


def _write(path, parts):
    with open(path, "wb") as f:
        for p in parts:
            f.write(p)


def write_verifier_key(path, pc, vk):
    """vk as read_verifier_key returns it (points already in the chosen form)"""
    _write(path, _vk_parts(pc, vk))


def write_prover_key(path, pc, vk, index, ck):
    """Arguments as read_prover_key returns them; index["coeffs"] may carry trailing zero coefficients (they are stripped)."""
    marlin = pc == _lib.PC_MARLIN_KZG10
    parts = _vk_parts(pc, vk)
    parts += [_u64(6)] + [_u64(0) + (b"\x00" if marlin else b"")] * 6
    parts.append(b"".join(_u64(v) for v in index["info"]))
    for m in index["matrices"]:
        parts += _matrix(*m)
    for label, co in zip(POLY_LABELS, index["coeffs"]):
        parts += [_u64(len(label)), label.encode()] + _vec(strip_zeros(np.asarray(co, dtype=np.uint8).reshape(-1, FR_BYTES))) + [b"\x00\x00"]
    for name in EVAL_NAMES:
        i = EVAL_OF_POLY.index(EVAL_NAMES.index(name))
        parts += _vec(index["evals"][i]) + [b"\x00", bytes(index["domains"][i])]
    opt = lambda a: [b"\x01"] + _vec(a) if a is not None else [b"\x00"]
    bounds = [b"\x01", _u64(len(ck["bounds"])), b"".join(_u64(b) for b in ck["bounds"])] if ck["bounds"] is not None else [b"\x00"]
    if marlin:
        parts += _vec(ck["powers"]) + opt(ck["shifted"]) + _vec(ck["gamma"])
    else:
        parts += _vec(ck["powers"]) + _vec(ck["gamma"]) + opt(ck["shifted"])
        if ck["shifted_gamma"] is None:
            parts.append(b"\x00")
        else:
            parts += [b"\x01", _u64(len(ck["shifted_gamma"]))]
            for k in sorted(ck["shifted_gamma"]):
                parts += [_u64(k)] + _vec(ck["shifted_gamma"][k])
    parts += bounds + [_u64(ck["max_degree"])]
    _write(path, parts)
