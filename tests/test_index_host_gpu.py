"""GPU: host-resident indexes.  An index whose device-resident byte model does not fit keeps its twelve |K|-vectors (the
coefficients and evaluations on K of row, col, a_val, b_val, c_val, row_col) in pinned host memory and streams them into
round 3 and the opening of every proof.  A proof is a unique function of its inputs, so every proof, key file and rng
position must equal the device-resident index's byte for byte.  B2M_INDEX_HOST=1 forces host residency."""
import hashlib
import json
import os
import re

import pytest

import test_index_keys_gpu as tk
import test_prover_gpu as tp
from marlin_b200 import _lib, api, r1cs as gr1cs
from oracle.params import BLS12_381

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
A, B = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
BENCH_BETA = 0x5eed5eed5eed5eed5eed5eed


@pytest.fixture(scope="module")
def gctx(b2m_ctx):
    c = api.Context.__new__(api.Context)
    c.handle = b2m_ctx
    return c


@pytest.fixture
def host_index(monkeypatch):
    monkeypatch.setenv("B2M_INDEX_HOST", "1")


def pinned(key):
    with open(os.path.join(HERE, "golden", "bench_proof_hashes.json")) as fh:
        return json.load(fh)[key]


def dummy_setup(m, n):
    return m.universal_setup(n, n, 3 * n, beta=BENCH_BETA, gamma=7, degree_bounds=(n - 2, 4 * n - 2))


@pytest.mark.parametrize("case", tp._golden_cases(), ids=lambda c: c["name"])
def test_golden_fixture_bytes_host_resident(gctx, host_index, case):
    """Every committed fixture (BLS12-381 under both PCs, BN254 under MarlinKZG10): vk hash, proof bytes, rng position."""
    tp.test_golden_fixture_bytes(gctx, case)


@pytest.mark.parametrize("curve_name,scheme", [("bls12_381", "marlin_kzg10"), ("bls12_381", "sonic_kzg10"), ("bn254", "marlin_kzg10")])
def test_forced_host_residency_matches_device(gctx, monkeypatch, curve_name, scheme):
    """2^12 DummyCircuit: the forced host-resident index reports it, pins 12 |K| Fr, streams each vector it reads once per
    proof, and gives the device-resident index's proofs over two consecutive proofs of one rng stream."""
    n = 1 << 12
    m = api.Marlin(curve_name, scheme, ctx=gctx)
    circ = gr1cs.dummy_circuit(m.curve_id, A, B, 10, n)
    srs = dummy_setup(m, n)
    try:
        out = {}
        for res in ("device", "host"):
            monkeypatch.setenv("B2M_INDEX_HOST", "1" if res == "host" else "0")
            pk = m.index(srs, circ)
            try:
                assert pk.residency == res
                K = 4 * n
                assert pk.host_bytes == (12 * K * 32 if res == "host" else 0)
                rng = api.ZkRng(bytes(range(32)), 12)
                proofs = [m.prove(pk, circ, rng), m.prove(pk, circ, rng)]
                t = pk.timings()
                if res == "host":  # round 3: row, col, a/b/c_val evaluations; opening: the six coefficient vectors
                    assert t["IndexStream::bytes"] == 11 * K * 32 and t["IndexStream::H2D"] > 0
                else:
                    assert "IndexStream::bytes" not in t
                out[res] = (pk.vk_bytes, proofs, rng.word_pos)
            finally:
                pk.close()
        assert out["host"] == out["device"]
    finally:
        srs.close()


def test_profile_names_the_streamed_kernels_and_copies(host_index):
    """b2m_ctx_profile: the streamed round-3 passes and opening combination run under their own names, and the copies are a
    span `index_h2d` whose units are the bytes streamed."""
    n = 1 << 12
    K = 4 * n
    ctx = api.Context(0)
    try:
        m = api.Marlin("bls12_381", "marlin_kzg10", ctx=ctx)
        circ = gr1cs.dummy_circuit(0, A, B, 10, n)
        srs = dummy_setup(m, n)
        try:
            pk = m.index(srs, circ)
            try:
                ctx.profile(True)
                m.prove(pk, circ, api.ZkRng.test_rng())
                rep = ctx.profile_report()
                ctx.profile(False)
            finally:
                pk.close()
        finally:
            srs.close()
        assert rep["index_h2d"]["units"] == 11 * K * 32 and rep["index_h2d"]["launches"] == 4
        assert rep["index_r3_denominators"]["units"] == K and rep["index_r3_f"]["units"] == K
        assert rep["index_open_lincomb"]["units"] == 2 * K
    finally:
        ctx.close()


def test_2p20_forced_host_reproduces_the_pinned_proof(gctx, host_index):
    n = 1 << 20
    m = api.Marlin("bls12_381", "marlin_kzg10", ctx=gctx)
    srs = dummy_setup(m, n)
    try:
        circ = gr1cs.dummy_circuit(0, A, B, 10, n)
        pk = m.index(srs, circ)
        try:
            assert pk.residency == "host" and pk.host_bytes == 12 * (4 * n) * 32
            proof = m.prove(pk, circ, api.ZkRng.test_rng())
        finally:
            pk.close()
        assert hashlib.sha256(proof).hexdigest() == pinned("bls12_381/marlin_kzg10/20")
    finally:
        srs.close()


@pytest.mark.parametrize("log_n", [14, 16])
def test_memory_limit_chooses_host_residency(log_n):
    """A limit between the host- and the device-resident index's model: `index` picks host residency, the proof equals the
    unlimited one's and the pool peak stays under the limit.  Without the limit the same circuit is device-resident."""
    n = 1 << log_n
    ctx = api.Context(0)
    try:
        m = api.Marlin("bls12_381", "marlin_kzg10", ctx=ctx)
        circ = gr1cs.dummy_circuit(0, A, B, 10, n)
        srs = dummy_setup(m, n)
        try:
            pk = m.index(srs, circ)
            assert pk.residency == "device"
            want = (pk.vk_bytes, m.prove(pk, circ, api.ZkRng.test_rng()))
            pk.close()
            # far too little: refused, naming the device- and the host-resident figures
            used = ctx.memory()["used"]
            _lib.check(_lib.lib().b2m_ctx_set_memory_limit(ctx.handle, used + (1 << 20)))
            with pytest.raises(_lib.B2MError) as ei:
                m.index(srs, circ)
            assert ei.value.code == _lib.ERR_MEMORY_LIMIT
            got = re.search(r"needs (\d+) bytes device-resident .* or (\d+) bytes host-resident", str(ei.value))
            assert got, str(ei.value)
            dev, host = int(got.group(1)), int(got.group(2))
            assert host < dev
            used = ctx.memory()["used"]
            limit = used + (dev + host) // 2
            _lib.check(_lib.lib().b2m_ctx_set_memory_limit(ctx.handle, limit))
            pk = m.index(srs, circ)
            try:
                assert pk.residency == "host"
                assert (pk.vk_bytes, m.prove(pk, circ, api.ZkRng.test_rng())) == want
            finally:
                pk.close()
            peak = ctx.memory()["peak"]
            assert peak <= limit, (peak, limit)
        finally:
            srs.close()
    finally:
        ctx.close()


def test_key_files_are_independent_of_residency(gctx, tmp_path, monkeypatch):
    """`save` gives the same file from either residency; `load_index` under forced host residency proves the same bytes; a
    tampered file is still reported by field, because the checks run on the device before the vectors move."""
    n = 1 << 10
    m = api.Marlin("bls12_381", "marlin_kzg10", ctx=gctx)
    circ = gr1cs.dummy_circuit(0, A, B, 10, n)
    srs = dummy_setup(m, n)
    try:
        files = {}
        for res in ("0", "1"):
            monkeypatch.setenv("B2M_INDEX_HOST", res)
            pk = m.index(srs, circ)
            try:
                files[res] = str(tmp_path / f"pk{res}.bin")
                pk.save(files[res], compressed=True)
                if res == "0":
                    want = m.prove(pk, circ, api.ZkRng.test_rng())
            finally:
                pk.close()
        assert open(files["0"], "rb").read() == open(files["1"], "rb").read()
        monkeypatch.setenv("B2M_INDEX_HOST", "1")
        pk = m.load_index(srs, files["1"], check_commitments=True)
        try:
            assert pk.residency == "host"
            assert m.prove(pk, circ, api.ZkRng.test_rng()) == want
            again = str(tmp_path / "again.bin")
            pk.save(again, compressed=True)
            assert open(again, "rb").read() == open(files["0"], "rb").read()
        finally:
            pk.close()
    finally:
        srs.close()


def test_tampered_key_file_is_named_under_host_residency(gctx, tmp_path, host_index):
    tk.test_inconsistent_coefficients_other_srs_and_tampered_commitment(gctx, tmp_path)


@pytest.mark.parametrize("curve_name,log_n", [("bls12_381", 12), ("bls12_381", 14), ("bls12_381", 16), ("bls12_381", 18), ("bn254", 12),
                                              ("bn254", 16)])
@pytest.mark.parametrize("res", ["0", "1"])
def test_model_bounds_the_pool_peak(monkeypatch, curve_name, log_n, res):
    """The pool high-water mark over setup, index and prove stays below the byte model the key was planned by (the model
    of the largest circuit of the key, which this circuit is; the host-resident term is never above the device one)."""
    monkeypatch.setenv("B2M_INDEX_HOST", res)
    n = 1 << log_n
    ctx = api.Context(0)
    try:
        m = api.Marlin(curve_name, "marlin_kzg10", ctx=ctx)
        circ = gr1cs.dummy_circuit(m.curve_id, A, B, 10, n)
        used0 = ctx.memory()["used"]
        srs = dummy_setup(m, n)
        try:
            pk = m.index(srs, circ)
            try:
                assert pk.residency == ("host" if res == "1" else "device")
                m.prove(pk, circ, api.ZkRng.test_rng())
            finally:
                pk.close()
            peak = ctx.memory()["peak"] - used0
            model = srs.layout()["model_bytes"]
            assert peak <= model, (peak, model)
        finally:
            srs.close()
    finally:
        ctx.close()


def _mem_available():
    try:
        with open("/proc/meminfo") as fh:
            for line in fh:
                if line.startswith("MemAvailable:"):
                    return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 0


NEED_HOST = 64 << 30  # 25.8 GB pinned index vectors, the circuit's host copies and the verifier's Python objects


def test_2p24_proves_on_one_gpu_with_a_host_resident_index(gctx):
    """2^24 constraints (BLS12-381, MarlinKZG10, |K| = 2^26) with no knobs: the key plans a host-resident index, the proof
    verifies on the GPU, fails for a wrong public input, and the oracle's pairing verifier accepts it."""
    import torch
    total = torch.cuda.get_device_properties(0).total_memory
    avail = _mem_available()
    if total < 80 * 10 ** 9 or avail < NEED_HOST:
        pytest.skip(f"needs a GPU of >= 80 GB (has {total / 1e9:.1f} GB) and >= {NEED_HOST / 2**30:.0f} GiB MemAvailable "
                    f"(has {avail / 2**30:.1f} GiB)")
    from oracle import kzg, marlin as omarlin
    import b2m_testutil as util
    log_n = 24
    n = 1 << log_n
    curve = BLS12_381
    m = api.Marlin("bls12_381", "marlin_kzg10", ctx=gctx)
    srs = m.universal_setup(n, n, 3 * n, beta=BENCH_BETA, gamma=7, degree_bounds=(n - 2, 4 * n - 2))
    try:
        circ = gr1cs.dummy_circuit(0, A, B, 10, n)
        pk = m.index(srs, circ)
        try:
            assert pk.residency == "host"
            proof_bytes = m.prove(pk, circ, api.ZkRng.test_rng())
            vk = m.verifier_key(pk, srs)
            try:
                c_pub = A * B % curve.fr.p
                assert m.verify(vk, [c_pub], proof_bytes, api.ZkRng(seed=bytes(32)))
                assert not m.verify(vk, [(c_pub + 1) % curve.fr.p], proof_bytes, api.ZkRng(seed=bytes(32)))
            finally:
                vk.close()
            comms = util.points_from_limbs(curve, pk.index_comms)
            lazy = kzg.UniversalParams(curve, srs.max_degree, BENCH_BETA, curve.g, 7, powers_of_g="lazy")
            ovk = omarlin.verifier_key_from_public(curve, kzg.MARLIN, lazy, n, n, 3 * (n - 1), comms)
            assert ovk.vk_bytes == pk.vk_bytes
            proof = omarlin.deserialize_proof(curve, kzg.MARLIN, proof_bytes)
            g2 = kzg.G2Key(lazy, ovk.ck.enforced_degree_bounds)
            assert omarlin.verify(ovk, [c_pub], proof, g2)
            assert not omarlin.verify(ovk, [(c_pub + 1) % curve.fr.p], proof, g2)
        finally:
            pk.close()
    finally:
        srs.close()
