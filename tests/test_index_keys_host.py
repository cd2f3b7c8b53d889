"""CPU: framing of arkworks index key files (marlin_b200/keyfile.py).  Files written by the independent oracle writer
(tests/index_key_oracle.py) parse into the oracle's values for both curves, both PC schemes and both point forms, and write
back byte for byte; truncation at every section boundary, a trailing byte, a bad option byte, a length running past the end,
unsorted map keys, a wrong label, a wrong domain tag and non-empty commitment randomness each raise an error naming the
field."""
import struct

import numpy as np
import pytest

from marlin_b200 import _lib, keyfile
from oracle import kzg
from oracle import marlin as omarlin
from oracle import r1cs as or1cs
from oracle import rng as orng
from oracle.params import BLS12_381, BN254

import index_key_oracle as iko

PCS = {"marlin_kzg10": (kzg.MARLIN, _lib.PC_MARLIN_KZG10), "sonic_kzg10": (kzg.SONIC, _lib.PC_SONIC_KZG10)}
CIDS = {"bls12_381": _lib.CURVE_BLS12_381, "bn254": _lib.CURVE_BN254}
_CACHE = {}


def oracle_keys(curve, pc, compressed, n=16):
    key = (curve.name, pc, compressed, n)
    if key not in _CACHE:
        f = curve.fr
        r = orng.test_rng()
        a, b = orng.field_rand(f, r), orng.field_rand(f, r)
        circ = or1cs.dummy_circuit(f, a, b, 10, n)
        osrs = omarlin.universal_setup(curve, n, n, 3 * n, beta=0x1234567, g_scalar=1, gamma=7)
        opk = omarlin.index(osrs, circ, PCS[pc][0], kzg.Engine(use_trapdoor=True))
        w = iko.KeyWriter(osrs, opk, compressed)
        _CACHE[key] = (w.prover_key(), w.verifier_key(), opk)
    return _CACHE[key]


def write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(bytes(data))
    return str(p)


@pytest.mark.parametrize("compressed", [True, False], ids=["compressed", "uncompressed"])
@pytest.mark.parametrize("pc", list(PCS))
@pytest.mark.parametrize("curve", [BLS12_381, BN254], ids=lambda c: c.name)
def test_oracle_files_parse_and_write_back(tmp_path, curve, pc, compressed):
    pk_bytes, vk_bytes, opk = oracle_keys(curve, pc, compressed)
    cid, pcid = CIDS[curve.name], PCS[pc][1]
    f = curve.fr
    d = keyfile.read_prover_key(write(tmp_path, "pk.bin", pk_bytes), cid, pcid, compressed)
    vk = keyfile.read_verifier_key(write(tmp_path, "vk.bin", vk_bytes), cid, pcid, compressed)
    idx = opk.index
    info = (idx.info.num_variables, idx.info.num_constraints, idx.info.num_non_zero, idx.info.num_instance_variables)
    assert vk["info"] == d["vk"]["info"] == d["index"]["info"] == info
    assert [int(b) for b in vk["bounds"]] == opk.ck.enforced_degree_bounds == d["ck"]["bounds"]
    assert vk["max_degree"] == d["ck"]["max_degree"] == opk.ck.max_degree
    to_int = lambda rows: [int.from_bytes(bytes(x), "little") for x in rows]
    by_label = {p.label: p for p in idx.polys}
    for i, label in enumerate(keyfile.POLY_LABELS):
        assert to_int(d["index"]["coeffs"][i]) == iko.strip(by_label[label].coeffs)
    for k, name in enumerate(keyfile.EVAL_NAMES):
        i = keyfile.EVAL_OF_POLY.index(k)
        assert to_int(d["index"]["evals"][i]) == [v % f.p for v in idx.evals[name]]
    for (row_ptr, col, coeff), rows in zip(d["index"]["matrices"], (idx.a, idx.b, idx.c)):
        flat = [e for row in rows for e in row]
        assert [int(x) for x in np.diff(row_ptr.astype(np.int64))] == [len(r) for r in rows]
        assert [int(c) for c in col] == [i for _, i in flat]
        assert to_int(coeff) == [c for c, _ in flat]
    # and back, byte for byte
    out = tmp_path / "again.bin"
    keyfile.write_prover_key(str(out), pcid, d["vk"], d["index"], d["ck"])
    assert out.read_bytes() == pk_bytes
    keyfile.write_verifier_key(str(out), pcid, vk)
    assert out.read_bytes() == vk_bytes


@pytest.mark.parametrize("pc", list(PCS))
@pytest.mark.parametrize("curve", [BLS12_381, BN254], ids=lambda c: c.name)
def test_zero_polynomial_is_stored_empty_and_writes_back(tmp_path, curve, pc):
    """An empty C matrix makes c_val the zero polynomial: the oracle file stores it with no coefficients (a `DensePolynomial`
    drops zero high coefficients), it parses as an empty vector next to |K| evaluations, and the writer, given the |K| zero
    coefficients a device index exports, strips them back to the same bytes."""
    f = curve.fr
    circ = iko.zero_c_circuit(f, 0x1234, 16)
    osrs = omarlin.universal_setup(curve, 16, 16, 48, beta=0x1234567, g_scalar=1, gamma=7)
    opk = omarlin.index(osrs, circ, PCS[pc][0], kzg.Engine(use_trapdoor=True))
    assert all(len(r) == 0 for r in opk.index.c)
    pk_bytes = iko.KeyWriter(osrs, opk, True).prover_key()
    cid, pcid = CIDS[curve.name], PCS[pc][1]
    d = keyfile.read_prover_key(write(tmp_path, "pk.bin", pk_bytes), cid, pcid, True)
    K = len(opk.index.evals["row"])
    assert len(d["index"]["coeffs"][4]) == 0 and len(d["index"]["evals"][4]) == K
    assert len(d["index"]["matrices"][2][1]) == 0
    index = dict(d["index"])
    index["coeffs"] = [np.concatenate([c, np.zeros((K - len(c), 32), dtype=np.uint8)]) for c in d["index"]["coeffs"]]
    out = tmp_path / "again.bin"
    keyfile.write_prover_key(str(out), pcid, d["vk"], index, d["ck"])
    assert out.read_bytes() == pk_bytes


def _boundaries(curve, pc, compressed):
    """byte offsets of the section boundaries of a prover key: after the verifier key, the randomness, each matrix, each
    labelled polynomial, each evaluation vector, and each field of the committer key"""
    pk_bytes, vk_bytes, opk = oracle_keys(curve, pc, compressed)
    g1 = curve.fq.nbytes if compressed else 2 * curve.fq.nbytes
    ck = opk.ck
    D, bounds = ck.max_degree, ck.enforced_degree_bounds
    marks = [len(vk_bytes), len(vk_bytes) + 8 + 6 * (9 if pc == "marlin_kzg10" else 8)]
    at = marks[-1] + 32
    idx = opk.index
    for m in (idx.a, idx.b, idx.c):
        at += 8 + sum(8 + 40 * len(r) for r in m)
        marks.append(at)
    by_label = {p.label: p for p in idx.polys}
    for label in keyfile.POLY_LABELS:
        at += 8 + len(label) + 8 + 32 * len(iko.strip(by_label[label].coeffs)) + 2
        marks.append(at)
    K = len(idx.evals["row"])
    for _ in range(6):
        at += 8 + 32 * K + 1 + keyfile.DOMAIN_BYTES
        marks.append(at)
    powers = 8 + g1 * (ck.supported_degree + 1)
    shifted = 1 + 8 + g1 * (bounds[-1] + 1)
    gamma = 8 + 3 * g1
    if pc == "marlin_kzg10":
        fields = [powers, shifted, gamma]
    else:
        fields = [powers, gamma, shifted, 1 + 8 + sum(16 + g1 * len([i for i in range(3) if D - d + i < D + 2]) for d in bounds)]
    for size in fields + [1 + 8 + 8 * len(bounds)]:
        at += size
        marks.append(at)
    assert at + 8 == len(pk_bytes)  # max_degree closes the file
    return pk_bytes, marks


@pytest.mark.parametrize("pc", list(PCS))
def test_truncation_at_every_section_boundary_and_trailing_byte(tmp_path, pc):
    curve, compressed = BLS12_381, True
    pk_bytes, marks = _boundaries(curve, pc, compressed)
    cid, pcid = CIDS[curve.name], PCS[pc][1]
    for cut in sorted(set(marks + [m - 1 for m in marks] + [1, 8, 40, len(pk_bytes) - 1])):
        if cut >= len(pk_bytes):
            continue
        with pytest.raises(ValueError) as e:
            keyfile.read_prover_key(write(tmp_path, "cut.bin", pk_bytes[:cut]), cid, pcid, compressed)
        assert "truncated" in str(e.value) or "bytes left" in str(e.value), (cut, str(e.value))
        assert ": " in str(e.value).split("cut.bin", 1)[1]
    with pytest.raises(ValueError, match="1 trailing bytes"):
        keyfile.read_prover_key(write(tmp_path, "long.bin", pk_bytes + b"\x00"), cid, pcid, compressed)
    _, vk_bytes, _ = oracle_keys(curve, pc, compressed)
    with pytest.raises(ValueError, match="1 trailing bytes"):
        keyfile.read_verifier_key(write(tmp_path, "vlong.bin", vk_bytes + b"\x00"), cid, pcid, compressed)


def test_bad_option_byte_names_the_field(tmp_path):
    curve, pc, compressed = BLS12_381, "marlin_kzg10", True
    pk_bytes, _, _ = oracle_keys(curve, pc, compressed)
    vk_len = len(oracle_keys(curve, pc, compressed)[1])
    data = bytearray(pk_bytes)
    data[vk_len + 8 + 8] = 2  # index_comm_rands[0].shifted_rand
    with pytest.raises(ValueError, match=r"index_comm_rands\[0\]\.shifted_rand: option byte 2"):
        keyfile.read_prover_key(write(tmp_path, "opt.bin", data), 0, _lib.PC_MARLIN_KZG10, compressed)
    # the option of the verifier key's shift powers
    g1 = 48
    at = 32 + 8 + 6 * (g1 + 1) + 2 * g1 + 2 * 2 * g1
    data = bytearray(pk_bytes)
    data[at] = 7
    with pytest.raises(ValueError, match="index_vk.verifier_key.degree_bounds_and_shift_powers: option byte 7"):
        keyfile.read_prover_key(write(tmp_path, "opt2.bin", data), 0, _lib.PC_MARLIN_KZG10, compressed)
    # a non-empty blinding polynomial
    data = bytearray(pk_bytes)
    data[vk_len + 8] = 1
    with pytest.raises(ValueError, match=r"index_comm_rands\[0\]\.blinding_polynomial: is not empty"):
        keyfile.read_prover_key(write(tmp_path, "rand.bin", data), 0, _lib.PC_MARLIN_KZG10, compressed)


def test_length_past_the_end_names_the_field(tmp_path):
    curve, pc, compressed = BN254, "sonic_kzg10", False
    pk_bytes, _, opk = oracle_keys(curve, pc, compressed)
    _, marks = _boundaries(curve, pc, compressed)
    data = bytearray(pk_bytes)
    # the length of index.joint_arith.row.polynomial (after its 8 + 3 label bytes)
    at = marks[4] + 8 + 3
    data[at:at + 8] = struct.pack("<Q", 1 << 40)
    with pytest.raises(ValueError, match=r"index\.joint_arith\.row\.polynomial: claims 1099511627776 entries"):
        keyfile.read_prover_key(write(tmp_path, "len.bin", data), 1, _lib.PC_SONIC_KZG10, compressed)
    data = bytearray(pk_bytes)
    data[marks[1] + 32:marks[1] + 40] = struct.pack("<Q", 1 << 50)  # rows of index.a
    with pytest.raises(ValueError, match=r"index\.a: claims"):
        keyfile.read_prover_key(write(tmp_path, "rows.bin", data), 1, _lib.PC_SONIC_KZG10, compressed)


def test_unsorted_sonic_map_keys_wrong_label_and_wrong_domain_tag(tmp_path):
    curve, pc, compressed = BLS12_381, "sonic_kzg10", True
    pk_bytes, _, opk = oracle_keys(curve, pc, compressed)
    _, marks = _boundaries(curve, pc, compressed)
    cid, pcid = 0, _lib.PC_SONIC_KZG10
    # shifted_powers_of_gamma_g: swap the two keys
    bounds = opk.ck.enforced_degree_bounds
    assert len(bounds) == 2
    g1 = 48
    tail = 1 + 8 + 8 * len(bounds) + 8  # enforced bounds option + vec, max_degree
    entry = 8 + 8 + 3 * g1
    start = len(pk_bytes) - tail - 2 * entry
    assert struct.unpack_from("<Q", pk_bytes, start)[0] == bounds[0]
    data = bytearray(pk_bytes)
    data[start:start + 8] = struct.pack("<Q", bounds[1])
    data[start + entry:start + entry + 8] = struct.pack("<Q", bounds[0])
    with pytest.raises(ValueError, match="committer_key.shifted_powers_of_gamma_g: key .* not strictly ascending"):
        keyfile.read_prover_key(write(tmp_path, "keys.bin", data), cid, pcid, compressed)
    # a wrong label
    data = bytearray(pk_bytes)
    data[marks[4] + 8:marks[4] + 11] = b"raw"
    with pytest.raises(ValueError, match=r"index\.joint_arith\.row\.label: is b'raw', expected 'row'"):
        keyfile.read_prover_key(write(tmp_path, "label.bin", data), cid, pcid, compressed)
    # a wrong domain tag (evals_on_K.col: after its evaluations)
    K = len(opk.index.evals["row"])
    at = marks[11] + 8 + 32 * K
    data = bytearray(pk_bytes)
    assert data[at] == 0
    data[at] = 1
    with pytest.raises(ValueError, match=r"index\.joint_arith\.evals_on_K\.col\.domain: tag 1 is not 0"):
        keyfile.read_prover_key(write(tmp_path, "tag.bin", data), cid, pcid, compressed)


def test_other_curve_or_scheme_fails_in_framing(tmp_path):
    pk_bytes, vk_bytes, _ = oracle_keys(BLS12_381, "marlin_kzg10", True)
    p, v = write(tmp_path, "pk.bin", pk_bytes), write(tmp_path, "vk.bin", vk_bytes)
    for cid, pcid in ((1, _lib.PC_MARLIN_KZG10), (0, _lib.PC_SONIC_KZG10), (1, _lib.PC_SONIC_KZG10)):
        with pytest.raises(ValueError):
            keyfile.read_prover_key(p, cid, pcid, True)
        with pytest.raises(ValueError):
            keyfile.read_verifier_key(v, cid, pcid, True)
    with pytest.raises(ValueError):
        keyfile.read_prover_key(p, 0, _lib.PC_MARLIN_KZG10, False)
