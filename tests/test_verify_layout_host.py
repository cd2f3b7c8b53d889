"""CPU: the G2 grouping of a batch over several verifier keys (csrc/verify_layout.hpp): which keys share a pairing product and
which pairing slot each key's h, beta h and SonicKZG10 bound points take in the call's G2 set."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
PB = 8  # bytes per point: the grouping compares encodings only


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    src = os.path.join(HERE, "host", "verify_layout_host_shim.cpp")
    so = str(tmp_path_factory.mktemp("verify_layout_host") / "libverify_layout_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", src, "-o", so])
    lib = ctypes.CDLL(so)
    lib.g2_layout_host.restype = ctypes.c_size_t
    return lib


def pt(name):
    return name.encode().ljust(PB, b"\0")


def layout(lib, keys):
    """keys: per key its point names (h, beta h, bounds...) -> (groups, per key point indices, [(group, key, key point)] of the set)"""
    bufs = [np.frombuffer(b"".join(pt(x) for x in k), dtype=np.uint8).copy() for k in keys]
    ptrs = (ctypes.c_void_p * len(keys))(*[b.ctypes.data for b in bufs])
    counts = (ctypes.c_size_t * len(keys))(*[len(k) for k in keys])
    total = sum(len(k) for k in keys)
    group = (ctypes.c_uint32 * len(keys))()
    point, gop, sk, sp = [(ctypes.c_uint32 * total)() for _ in range(4)]
    n_points = ctypes.c_size_t()
    n_groups = lib.g2_layout_host(len(keys), ptrs, counts, PB, group, point, gop, sk, sp, ctypes.byref(n_points))
    per_key, o = [], 0
    for k in keys:
        per_key.append(list(point[o:o + len(k)]))
        o += len(k)
    assert max(group[:len(keys)]) + 1 == n_groups
    return list(group), per_key, [(gop[i], sk[i], sp[i]) for i in range(n_points.value)]


def resolve(keys, per_key, src):
    """the point name each key point refers to through the call's set"""
    return [[keys[src[q][1]][src[q][2]] for q in qs] for qs in per_key]


@pytest.mark.parametrize("key", [["h", "bh"], ["h", "bh", "n6", "n14"], ["h", "bh", "n14", "n6", "n30"]], ids=["marlin", "sonic", "sonic3"])
def test_one_key_is_its_own_layout(hostlib, key):
    """h, beta h, then the bounds in order: the G2 indices b2m_verify_batch has always used"""
    groups, per_key, src = layout(hostlib, [key])
    assert groups == [0]
    assert per_key == [list(range(len(key)))]
    assert src == [(0, 0, j) for j in range(len(key))]


def test_equal_h_and_beta_h_share_a_group(hostlib):
    keys = [["h", "bh"], ["h", "bh", "n6"], ["h", "bh2"], ["h2", "bh"], ["h", "bh"], ["h2", "bh"]]
    groups, per_key, src = layout(hostlib, keys)
    assert groups == [0, 0, 1, 2, 0, 2]
    # a group's h and beta h are one pair of slots, listed by its first key
    assert per_key[0][:2] == per_key[1][:2] == per_key[4][:2]
    assert per_key[3][:2] == per_key[5][:2]
    assert len({tuple(p[:2]) for p in per_key}) == 3
    assert resolve(keys, per_key, src) == keys
    for g, qs in zip(groups, per_key):
        assert all(src[q][0] == g for q in qs)


def test_sonic_points_deduplicated_within_a_group_only(hostlib):
    keys = [["h", "bh", "x", "y"], ["h", "bh", "y", "z"], ["h2", "bh2", "x", "y"], ["h", "bh", "z", "x"]]
    groups, per_key, src = layout(hostlib, keys)
    assert groups == [0, 0, 1, 0]
    assert per_key[1][2] == per_key[0][3]  # y of group 0: one slot
    assert per_key[3][2:] == [per_key[1][3], per_key[0][2]]
    assert not set(per_key[2]) & set(per_key[0] + per_key[1] + per_key[3])  # group 1 has slots of its own
    assert len(src) == 2 + 3 + 2 + 2
    assert resolve(keys, per_key, src) == keys


def test_bound_point_equal_to_h_keeps_its_slot(hostlib):
    """a bound d = D gives beta^0 h = h: it stays a slot of its own, as in the one-key layout"""
    groups, per_key, src = layout(hostlib, [["h", "bh", "h"]])
    assert per_key == [[0, 1, 2]]
