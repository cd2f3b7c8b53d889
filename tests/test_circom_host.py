"""CPU: circom `.r1cs` / `.wtns` framing (marlin_b200/circom.py), the host walk over the constraint section
(b2m_circom_constraint_rows) and the padding rule `from_rows` and the circom loader share (r1cs.Shape).  No GPU."""
import ctypes
import os
import struct

import numpy as np
import pytest

import circom_writer as cw
from marlin_b200 import _lib, circom, fields
from marlin_b200 import r1cs as gr1cs

BN, BLS = _lib.CURVE_BN254, _lib.CURVE_BLS12_381
P_BN = fields.FR_MODULUS[BN]
CONS = [([(2, 1)], [(3, 5), (1, 2)], [(1, 1)]),
        ([], [(2, 7)], []),
        ([(3, P_BN - 1), (0, 4), (3, 9)], [(1, 1)], [(2, 3)])]


def r1cs_file(tmp_path, name="c.r1cs", cons=CONS, **kw):
    return cw.write_r1cs(os.path.join(tmp_path, name), P_BN, 4, 1, 1, cons, **kw)


def walk_arrays(data, m):
    rps = [np.zeros(m + 1, dtype=np.uint64) for _ in range(3)]
    end, bc, br = ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_int(0)
    buf = np.frombuffer(bytes(data), dtype=np.uint8) if len(data) else np.zeros(1, dtype=np.uint8)
    rc = _lib.lib().b2m_circom_constraint_rows(_lib.ptr(buf), len(data), m, *[_lib.ptr(r) for r in rps], ctypes.byref(end), ctypes.byref(bc),
                                               ctypes.byref(br))
    return rc, rps, end.value, bc.value, br.value, _lib.lib().b2m_last_error().decode()


def test_sections_load_in_any_order_and_unread_ones_are_ignored(tmp_path):
    for order in ([1, 2, 3], [2, 1, 3], [3, 2, 1], [2, 3, 1]):
        extra = [[99, b"\x00" * 17], [6, b"garbage"]]
        f = circom.read_r1cs(r1cs_file(tmp_path, f"o{''.join(map(str, order))}.r1cs", order=order, extra=extra))
        assert (f.n8, f.prime, f.n_wires, f.n_pub_out, f.n_pub_in, f.m) == (32, P_BN, 4, 1, 1, 3)
        assert f.ni0 == 3
        assert bytes(f.constraints) == cw.constraints_bytes(CONS)
        rps = circom.constraint_rows(f)
        assert [list(map(int, r)) for r in rps] == [[0, 1, 1, 4], [0, 2, 3, 4], [0, 1, 1, 2]]
    # no label section at all
    f = circom.read_r1cs(r1cs_file(tmp_path, "nolabels.r1cs", labels=False))
    assert f.m == 3
    assert circom.curve_of_prime(f.prime) == BN


def test_term_offsets_follow_the_prefix_sums():
    data = cw.constraints_bytes(CONS)
    rc, rps, end, _, _, _ = walk_arrays(data, 3)
    assert rc == 0 and end == len(data)
    for k, con in enumerate(CONS):
        for j, lc in enumerate(con):
            for i, (w, c) in enumerate(lc):
                off = circom.term_offset(rps, k, j, i)
                assert struct.unpack_from("<I", data, off)[0] == w
                assert int.from_bytes(data[off + 4:off + 36], "little") == c


def test_walk_names_the_constraint_and_matrix():
    data = cw.constraints_bytes(CONS)
    # truncated inside constraint 2's A term count
    lc2 = len(cw.constraints_bytes(CONS[:2]))
    rc, _, end, bc, br, msg = walk_arrays(data[:lc2 + 2], 3)
    assert (rc, bc, br, end) == (_lib.ERR_SERIALIZATION, 2, 1, lc2)
    assert "constraints[2].A: truncated in the term count" in msg
    # terms of constraint 0's B run past the end
    b0 = len(cw.lc_bytes(CONS[0][0]))
    rc, _, end, bc, br, msg = walk_arrays(data[:b0 + 4 + 36 + 10], 3)
    assert (rc, bc, br, end) == (_lib.ERR_SERIALIZATION, 0, 2, b0)
    assert "constraints[0].B: 2 terms run past the end" in msg
    # a missing C count of the last constraint
    rc, _, _, bc, br, msg = walk_arrays(data[:len(data) - len(cw.lc_bytes(CONS[2][2]))], 3)
    assert (bc, br) == (2, 1) and "constraints[2].C" in msg
    # overlong: the walk stops at m constraints and reports where
    rc, rps, end, _, _, _ = walk_arrays(data + b"\x00" * 12, 3)
    assert rc == 0 and end == len(data)
    # m = 0 on an empty section
    rc, rps, end, _, _, _ = walk_arrays(b"", 0)
    assert rc == 0 and end == 0 and [int(r[0]) for r in rps] == [0, 0, 0]


def framing_error(tmp_path, secs, magic=b"r1cs", version=1, reader=circom.read_r1cs):
    path = cw.write(os.path.join(tmp_path, "bad"), magic, version, secs)
    with pytest.raises(ValueError) as e:
        reader(path)
    return str(e.value)


def test_every_r1cs_framing_error_is_named(tmp_path):
    secs = cw.r1cs_sections(P_BN, 4, 1, 1, CONS)
    assert "the magic is not 'r1cs'" in framing_error(tmp_path, secs, magic=b"wtns")
    assert ".r1cs version 2" in framing_error(tmp_path, secs, version=2)
    assert "section 1 (header) is missing" in framing_error(tmp_path, secs[1:])
    assert "section 2 (constraints) is missing" in framing_error(tmp_path, [secs[0], secs[2]])
    assert "section 1 (header) appears more than once" in framing_error(tmp_path, secs + [secs[0]])
    assert "section 2 (constraints) appears more than once" in framing_error(tmp_path, secs + [secs[1]])
    # a section past the end of the file
    path = cw.write(os.path.join(tmp_path, "cut.r1cs"), b"r1cs", 1, secs)
    with open(path, "r+b") as fh:
        fh.truncate(os.path.getsize(path) - 5)
    with pytest.raises(ValueError, match=r"section 3 \(wire2LabelId\) of \d+ bytes runs past the end of the file"):
        circom.read_r1cs(path)
    hdr = bytearray(secs[0][1])
    assert "section 1 (header) has 63 bytes, n8 = 32 needs 64" in framing_error(tmp_path, [[1, hdr[:-1]]] + secs[1:])
    n8_16 = cw.r1cs_header(P_BN % (1 << 128), 4, 1, 1, 0, 3, n8=16)
    assert "n8 = 16, only 32-byte fields" in framing_error(tmp_path, [[1, n8_16]] + secs[1:])
    assert "PLONK custom gates" in framing_error(tmp_path, secs + [[4, b"\x00" * 8]])
    assert "section 5 (customGatesApplication)" in framing_error(tmp_path, secs + [[5, b"\x00" * 8]])
    with open(os.path.join(tmp_path, "short"), "wb") as fh:
        fh.write(b"r1cs")
    with pytest.raises(ValueError, match="not a .r1cs file"):
        circom.read_r1cs(os.path.join(tmp_path, "short"))
    # a section-2 size that disagrees with the walk
    longer = [secs[0], [2, secs[1][1] + b"\x00" * 12], secs[2]]
    f = circom.read_r1cs(cw.write(os.path.join(tmp_path, "long.r1cs"), b"r1cs", 1, longer))
    with pytest.raises(ValueError, match=r"section 2 \(constraints\) has \d+ bytes, its 3 constraints take \d+"):
        circom.constraint_rows(f)
    shorter = [secs[0], [2, secs[1][1][:-3]], secs[2]]
    f = circom.read_r1cs(cw.write(os.path.join(tmp_path, "short.r1cs"), b"r1cs", 1, shorter))
    with pytest.raises(ValueError, match=r"section 2 \(constraints\): constraints\[2\].C: 1 terms run past the end"):
        circom.constraint_rows(f)


def test_prime_mismatch_names_the_curve():
    circom.check_prime("x.r1cs", "section 1 (header)", P_BN, BN)
    with pytest.raises(ValueError, match="the bn254 scalar field, this Marlin instance is bls12_381"):
        circom.check_prime("x.r1cs", "section 1 (header)", P_BN, BLS)
    with pytest.raises(ValueError, match="the scalar field of no supported curve"):
        circom.check_prime("x.r1cs", "section 1 (header)", P_BN + 2, BN)


def test_every_wtns_framing_error_is_named(tmp_path):
    secs = cw.wtns_sections(P_BN, [1, 2, 3, 4])
    rd = circom.read_wtns
    f = rd(cw.write(os.path.join(tmp_path, "ok.wtns"), b"wtns", 2, secs[::-1] + [[7, b"xyz"]]))
    assert (f.n8, f.prime, f.n_witness) == (32, P_BN, 4)
    assert [int.from_bytes(bytes(v), "little") for v in f.values] == [1, 2, 3, 4]
    assert "the magic is not 'wtns'" in framing_error(tmp_path, secs, magic=b"r1cs", version=2, reader=rd)
    assert ".wtns version 1" in framing_error(tmp_path, secs, magic=b"wtns", version=1, reader=rd)
    assert "section 2 (witness) is missing" in framing_error(tmp_path, secs[:1], magic=b"wtns", version=2, reader=rd)
    assert "section 1 (header) appears more than once" in framing_error(tmp_path, secs + secs[:1], magic=b"wtns", version=2, reader=rd)
    bad_n8 = struct.pack("<I", 48) + P_BN.to_bytes(48, "little") + struct.pack("<I", 4)
    assert "n8 = 48, only 32-byte fields" in framing_error(tmp_path, [[1, bad_n8], secs[1]], magic=b"wtns", version=2, reader=rd)
    assert "section 1 (header) has 39 bytes, n8 = 32 needs 40" in framing_error(tmp_path, [[1, secs[0][1][:-1]], secs[1]], magic=b"wtns", version=2, reader=rd)
    assert "section 2 (witness) has 96 bytes, nWitness = 4 needs 128" in framing_error(tmp_path, [secs[0], [2, secs[1][1][:96]]], magic=b"wtns",
                                                                                        version=2, reader=rd)


@pytest.mark.parametrize("ni0", [1, 2, 3, 5, 17])
def test_shape_is_the_padding_from_rows_applies(ni0):
    for n_wit, nc in ((3, 40), (40, 3), (6, 6 + 1)):  # more constraints, more variables, nearly square
        inst = [1] + list(range(2, ni0 + 1))
        wit = list(range(100, 100 + n_wit))
        # one row per witness and instance variable, to see every column move
        rows = [[(1, i)] for i in range(ni0 + n_wit)][:nc] + [[] for _ in range(max(nc - ni0 - n_wit, 0))]
        r = gr1cs.from_rows(BN, rows, [[]] * nc, [[]] * nc, inst, wit)
        sh = gr1cs.Shape(ni0, n_wit, nc)
        assert r.num_instance == sh.ni and sh.shift == sh.ni - ni0
        assert r.num_constraints == r.num_variables == sh.size
        assert len(r.witness) == n_wit + sh.pad_witness and r.num_constraints == nc + sh.pad_rows
        assert (sh.pad_rows == 0) or (sh.pad_witness == 0)
        cols = [int(x) for x in r.a[1][:int(r.a[0][-1])]]
        assert cols == [sh.column(i) for i in range(min(nc, ni0 + n_wit))]
