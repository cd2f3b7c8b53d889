"""CPU: the Level-1 `PC::check_combinations` bookkeeping (csrc/pc_check.hpp, built through tests/host/pc_check_host_shim.cpp) on
the arrays `api.pc_check_arrays` marshals, against the oracle (oracle/kzg.py::check_combinations).  The terms of every opening
point, evaluated in G1 through the SRS trapdoor, vanish exactly when the oracle accepts; upstream's `Err` cases and the
malformed inputs are named."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import pc_check_oracle as P
from marlin_b200 import _lib, api
from oracle import ec, kzg
from oracle import transcript as T
from oracle.params import BLS12_381, BN254

HERE = os.path.dirname(os.path.abspath(__file__))
CONFIGS = [(ci, c, sch) for ci, c in ((0, BLS12_381), (1, BN254)) for sch in (kzg.MARLIN, kzg.SONIC)]
IDS = [f"{c.name}-{sch}" for _, c, sch in CONFIGS]
_PP = {}


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    src = os.path.join(HERE, "host", "pc_check_host_shim.cpp")
    so = str(tmp_path_factory.mktemp("pc_check_host") / "libpc_check_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DB2M_HOST_LIGHT_INLINE", "-shared", "-fPIC", "-x", "c++", src, "-o", so])
    L = ctypes.CDLL(so)
    L.pc_terms_host.restype = ctypes.c_long
    L.pc_terms_host.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
                                ctypes.c_uint32, ctypes.c_void_p, ctypes.c_char_p, ctypes.c_size_t]
    L.pc_points_host.restype = ctypes.c_size_t
    L.pc_points_host.argtypes = [ctypes.c_int, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p]
    return L


def pp_for(curve):
    if curve.name not in _PP:
        _PP[curve.name] = P.pp_for(curve)
    return _PP[curve.name]


def pc_id(sch):
    return _lib.PC_MARLIN_KZG10 if sch == kzg.MARLIN else _lib.PC_SONIC_KZG10


def no_gpu(limbs):
    raise AssertionError("the test sets carry compressed bytes")


def arrays(ci, sets, identity=False):
    return api.pc_check_arrays(ci, sets, identity, no_gpu)


def run_terms(L, ci, sch, arrs, s=0, n=None):
    """(terms per point, or -1 malformed, or the error string)"""
    ptrs = (ctypes.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    n = len(arrs[0]) - 1 if n is None else n
    b = np.asarray(P.BOUNDS, dtype=np.uint64)
    out = np.zeros(1 << 16, dtype=np.uint32)
    err = ctypes.create_string_buffer(512)
    rc = L.pc_terms_host(ci, pc_id(sch), n, ptrs, s, b.ctypes.data, len(b), 2 + len(b), out.ctypes.data, err, 512)
    if rc == -2:
        return err.value.decode()
    if rc == -1:
        return -1
    nw = 8
    fr = (BLS12_381 if ci == 0 else BN254).fr
    val = lambda o: fr.from_mont(sum(int(out[o + i]) << (32 * i) for i in range(nw)))  # noqa: E731
    pts, o = [], 0
    while o < rc:
        npl, nb = int(out[o]), int(out[o + 1])
        o += 2
        plain, bounded = [], []
        for _ in range(npl):
            plain.append((int(out[o]), val(o + 1)))
            o += 1 + nw
        for _ in range(nb):
            bounded.append((int(out[o]), int(out[o + 1]), val(o + 2)))
            o += 2 + nw
        z = val(o)
        w = int(out[o + nw])
        o += nw + 1
        pts.append((plain, bounded, z, w))
    return pts


def slot_points(L, ci, sch, arrs, oset, s=0):
    """the oracle points behind set s's slots (pc_set_points order)"""
    n = len(arrs[0]) - 1
    fq_bytes = 48 if ci == 0 else 32
    ptrs = (ctypes.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    kind = np.zeros(256, dtype=np.uint32)
    idx = np.zeros(256, dtype=np.uint64)
    k = L.pc_points_host(pc_id(sch), n, ptrs, s, fq_bytes, kind.ctypes.data, idx.ctypes.data)
    by_label = {p.label: c for p, c in zip(oset.polys, oset.comms)}
    labels = sorted(by_label)
    out = []
    for j in range(k):
        i = int(idx[j]) - int(arrs[0][s]) if kind[j] < 2 else int(idx[j]) - int(arrs[9][s])
        out.append(oset.proofs[i][0] if kind[j] == 2 else by_label[labels[i]].shifted if kind[j] == 1 else by_label[labels[i]].comm)
    return out


def equations_hold(curve, pp, sch, terms, pts):
    """per point: plain + z W - beta W + sum_k beta^-(D - d_k) bounded_k == O, the pairing equation through the trapdoor"""
    r = curve.fr.p
    shared = [pp.g, pp.gamma_g] + ([pp.powers_of_g[P.D - d] for d in P.BOUNDS] if sch == kzg.MARLIN else [])
    base = lambda b: shared[b] if b < len(shared) else pts[b - 2 - len(P.BOUNDS)]  # noqa: E731
    ok = []
    for plain, bounded, z, w in terms:
        bases = [base(b) for b, _ in plain] + [base(w)]
        scalars = [c for _, c in plain] + [(z - pp.beta) % r]
        for k, b, c in bounded:
            bases.append(base(b))
            scalars.append(c * pow(pow(pp.beta, P.D - P.BOUNDS[k], r), -1, r) % r)
        ok.append(ec.msm_naive(curve, bases, scalars) is None)
    return ok


@pytest.mark.parametrize("ci,curve,sch", CONFIGS, ids=IDS)
def test_terms_vanish_exactly_when_the_oracle_accepts(hostlib, ci, curve, sch):
    pp = pp_for(curve)
    ck = P.ck_for(pp, sch)
    for seed, bounded in ((1, (12,)), (2, (12, 20)), (3, ())):
        o = P.random_set(ck, seed, bounded=bounded)
        assert o.check() is True
        tampered = P.random_set(ck, seed, bounded=bounded)
        key = sorted(tampered.evaluations)[seed % len(tampered.evaluations)]
        tampered.evaluations[key] = (tampered.evaluations[key] + 1) % curve.fr.p
        assert tampered.check() is False
        for oset, want in ((o, True), (tampered, False)):
            arrs = arrays(ci, [oset.api_set()])
            terms = run_terms(hostlib, ci, sch, arrs)
            assert len(terms) == 2
            held = equations_hold(curve, pp, sch, terms, slot_points(hostlib, ci, sch, arrs, oset))
            assert all(held) == want
            if sch == kzg.SONIC and bounded:
                assert any(t[1] for t in terms)  # the bounded LCs went to their bounds' pairings


@pytest.mark.parametrize("ci,curve,sch", CONFIGS[:2], ids=IDS[:2])
def test_batch_check_identity_lcs(hostlib, ci, curve, sch):
    """batch_check's LCs (one per commitment, coefficient one, the commitment's label) give the terms of explicit ones"""
    o = P.random_set(P.ck_for(pp_for(curve), sch), 5, bounded=(20,))
    s = o.api_set()
    labels = sorted(s.commitments)
    query = [(l, ("z", 1234567)) for l in labels]
    evals = {(l, 1234567): 1 for l in labels}
    s_id = api.OpeningSet(s.commitments, query, evals, [s.proofs[0]], s.challenge, degree_bounds=s.degree_bounds, shifted=s.shifted)
    s_lc = api.OpeningSet(s.commitments, query, evals, [s.proofs[0]], s.challenge, lcs=[(l, [(1, l)]) for l in reversed(labels)],
                          degree_bounds=s.degree_bounds, shifted=s.shifted)
    a, b = arrays(ci, [s_id], identity=True), arrays(ci, [s_lc])
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert run_terms(hostlib, ci, sch, a) == run_terms(hostlib, ci, sch, b)


def mutate(arrs, k, fn):
    arrs = [a.copy() for a in arrs]
    fn(arrs[k])
    return arrs


@pytest.mark.parametrize("sch", [kzg.MARLIN, kzg.SONIC])
def test_errors_and_malformed_sets(hostlib, sch):
    ci, curve = 0, BLS12_381
    o = P.random_set(P.ck_for(pp_for(curve), sch), 7, bounded=(12,))
    s = o.api_set()
    base = arrays(ci, [s])
    labels = sorted(s.commitments)
    bi = labels.index("b0")
    lcs = sorted(lc.label for lc in o.lcs)
    t_b = int(base[6][lcs.index("lc_b0")])   # the bounded LC's one term
    t_mix = int(base[6][lcs.index("mix")])   # mix's first term

    def err(arrs):
        r = run_terms(hostlib, ci, sch, arrs)
        assert isinstance(r, str), r
        return r
    assert "EquationHasDegreeBounds" in err(mutate(base, 7, lambda a: a.__setitem__(t_mix, bi)))
    assert "is not one" in err(mutate(base, 8, lambda a: a.__setitem__(t_b, _lib.ints_to_limbs([12345], 4)[0])))
    assert "not enforced" in err(mutate(base, 2, lambda a: a.__setitem__(bi, 13)))
    assert "names commitment" in err(mutate(base, 7, lambda a: a.__setitem__(t_mix, len(labels))))
    assert "names LC" in err(mutate(base, 15, lambda a: a.__setitem__(0, len(lcs))))
    assert "names point" in err(mutate(base, 16, lambda a: a.__setitem__(0, 2)))
    q = np.flatnonzero(base[16] == base[16][1])  # two queries at one point: give the second the first's LC
    assert "repeats" in err(mutate(base, 15, lambda a: a.__setitem__(q[1], a[q[0]])))
    extra = list(base)  # a third point (and proof) that no query names
    extra[9] = np.array([0, 3], dtype=np.uint64)
    extra[10] = np.concatenate([base[10], base[10][:1]])
    extra[11] = np.concatenate([base[11], base[11][:1]])
    extra[12] = np.concatenate([base[12], np.zeros(1, dtype=np.int32)])
    extra[13] = np.concatenate([base[13], np.zeros(32, dtype=np.uint8)])
    assert "point 2 has no query" in err(extra)
    r = curve.fr.p
    ev = mutate(base, 17, lambda a: a.__setitem__(slice(0, 32), np.frombuffer(r.to_bytes(32, "little"), dtype=np.uint8)))
    assert run_terms(hostlib, ci, sch, ev) == -1  # an evaluation equal to r
    rv_at = int(np.flatnonzero(base[12])[0])
    rv = mutate(base, 13, lambda a: a.__setitem__(slice(32 * rv_at, 32 * rv_at + 32), np.frombuffer((r + 5).to_bytes(32, "little"), dtype=np.uint8)))
    assert run_terms(hostlib, ci, sch, rv) == -1  # random_v not below r
    no_shift = mutate(base, 3, lambda a: a.__setitem__(bi, 0))
    assert run_terms(hostlib, ci, sch, no_shift) == (-1 if sch == kzg.MARLIN else run_terms(hostlib, ci, sch, base))
    assert T.g1_compressed(curve, o.comms[[p.label for p in o.polys].index("b0")].comm) == bytes(base[1][bi])
