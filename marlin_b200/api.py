"""Host-side mirror of the reference's public API for the accelerated path:
`Marlin::<F, PC, FS>::{universal_setup, index, prove, verify}` [reference src/lib.rs:79-433] with
F in {BLS12-381 Fr, BN254 Fr}, PC in {MarlinKZG10, SonicKZG10}, FS = SimpleHashFiatShamirRng<Blake2s, ChaChaRng>.
Every call lands in libb2m.so (include/b2m.h); nothing here computes on the CPU beyond marshalling.

Proofs are `CanonicalSerialize` bytes, the form the reference's `Marlin::verify` consumes.  `Marlin.verify_batch` checks
many proofs under one verifier key at once (G1 decoding and the folded MSMs on the GPU, a constant number of pairings per
batch on the host); `Marlin.verify` is a batch of one.
"""
import ctypes
import json
import os
import struct
import types

import numpy as np

from . import _lib, fields, srsfile

PC_IDS = {"marlin_kzg10": _lib.PC_MARLIN_KZG10, "sonic_kzg10": _lib.PC_SONIC_KZG10}
_CURVE_NAMES = {v: k for k, v in fields.CURVE_IDS.items()}


class Context:
    """One GPU (b2m_ctx).  memory_limit: device bytes an SRS created through this context plans its window tables and MSM
    passes for, and `index` checks its circuit against (None: all free device memory).  The library allocates from the
    device's default memory pool, shared by every Context on that device in the process, so the limit also counts what the
    other contexts hold."""

    def __init__(self, device=0, memory_limit=None):
        self.handle = ctypes.c_void_p()
        _lib.check(_lib.lib().b2m_ctx_create(device, ctypes.byref(self.handle)))
        if memory_limit:
            _lib.check(_lib.lib().b2m_ctx_set_memory_limit(self.handle, int(memory_limit)))

    def memory(self):
        """{"used", "peak", "reserved"}: bytes of the device's default memory pool in use, their high-water mark since the
        previous call, and bytes the pool holds from the device.  The pool is shared by every Context on the device in the
        process: the figures include their allocations, and the call restarts the high-water mark for all of them."""
        out = (ctypes.c_size_t * 3)()
        _lib.check(_lib.lib().b2m_ctx_memory(self.handle, out))
        return {"used": int(out[0]), "peak": int(out[1]), "reserved": int(out[2])}

    def launches(self):
        return int(_lib.lib().b2m_ctx_launches(self.handle))

    def profile(self, enable=True):
        _lib.check(_lib.lib().b2m_ctx_profile(self.handle, 1 if enable else 0))

    def profile_report(self):
        buf = ctypes.create_string_buffer(1 << 16)
        _lib.check(_lib.lib().b2m_ctx_profile_report(self.handle, buf, 1 << 16))
        return json.loads(buf.value.decode() or "{}")

    def close(self):
        if self.handle:
            _lib.lib().b2m_ctx_destroy(self.handle)
            self.handle = None


class ZkRng:
    """The caller's `zk_rng` as a ChaCha stream position.  Like the reference, which makes the caller pass
    `zk_rng: &mut R` [reference src/lib.rs:154], there is no implicit fixed seed: `ZkRng()` seeds from
    os.urandom(32); the public `ark_std::test_rng()` stream (ChaCha12, fixed seed -- NOT zero-knowledge, every
    blinding value is predictable) is only available through the explicit `ZkRng.test_rng()` used by tests
    and the bench."""
    TEST_RNG_SEED = bytes([1, 0, 0, 0, 23, 0, 0, 0, 200, 1, 0, 0, 210, 30, 0, 0] + [0] * 16)

    def __init__(self, seed=None, rounds=12, word_pos=0):
        self.c = _lib.Rng()
        self.c.kind = rounds
        seed = os.urandom(32) if seed is None else bytes(seed)
        if len(seed) != 32:
            raise ValueError("ZkRng seed must be 32 bytes")
        ctypes.memmove(self.c.key, seed, 32)
        self.c.word_pos = word_pos

    @classmethod
    def test_rng(cls):
        """`ark_std::test_rng()`: rand 0.8 StdRng (ChaCha12) with the public fixed seed.  Tests / benchmarks only."""
        return cls(cls.TEST_RNG_SEED, 12, 0)

    @property
    def word_pos(self):
        return int(self.c.word_pos)


class CallbackRng:
    """Any other `RngCore` behind the C ABI (B2M_RNG_CALLBACK): `next_u64` is a Python callable returning the generator's next
    64-bit output; the library pulls every random value the reference would draw through it, in the reference's order."""

    def __init__(self, next_u64):
        self._fn = next_u64
        self._cb = _lib.NEXT_U64(lambda _state: int(self._fn()) & 0xFFFFFFFFFFFFFFFF)  # kept alive with the object
        self.c = _lib.Rng()
        self.c.kind = _lib.RNG_CALLBACK
        self.c.next_u64 = self._cb
        self.c.state = None

    @property
    def word_pos(self):
        return None


class CommitterKey:
    """`PC::CommitterKey` after `PC::trim` (b2m_ck): a validated view of the device-resident SRS."""

    def __init__(self, srs, handle, pc, supported_degree, hiding_bound, degree_bounds):
        self.srs, self.handle, self.pc = srs, handle, pc
        self.supported_degree, self.hiding_bound, self.degree_bounds = supported_degree, hiding_bound, sorted(set(degree_bounds))

    def shift_power(self, bound):
        """MarlinKZG10 verifier key entry for an enforced bound: powers_of_g[max_degree - bound] (affine limbs)."""
        lq = _lib.LIMBS[self.srs.curve_id][1]
        out = np.zeros(2 * lq, dtype=np.uint64)
        _lib.check(_lib.lib().b2m_ck_shift_power(self.handle, bound, _lib.ptr(out)))
        return out

    def close(self):
        if self.handle:
            _lib.lib().b2m_ck_destroy(self.handle)
            self.handle = None


class UniversalSRS:
    """`PC::UniversalParams`, device resident (b2m_srs): G1 powers + the gamma powers the PC needs."""

    def __init__(self, ctx, curve_id, handle, max_degree, powers_limbs, gamma_limbs=None, gamma_indices=None):
        self.ctx, self.curve_id, self.handle, self.max_degree = ctx, curve_id, handle, max_degree
        self.powers_limbs, self.gamma_limbs, self.gamma_indices = powers_limbs, gamma_limbs, gamma_indices
        self.trapdoor = None  # (beta, gamma) of an insecure test SRS made by universal_setup / srs_from_trapdoor
        self.g2 = None        # (h, beta_h, {index: neg power}) as ark-serialize bytes when loaded from / written to a file
        self.ark = None       # load_ark_srs: the whole file as decoded -- every gamma power and neg_powers_of_h (save_ark)

    def layout(self):
        """The device layout of the key's MSM tables and the byte model it was chosen by (b2m_srs_layout)."""
        out = (ctypes.c_size_t * 8)()
        _lib.check(_lib.lib().b2m_srs_layout(self.handle, out))
        keys = ("window_bits", "window_tables", "max_pairs", "tables_bytes", "circuit_bytes", "msm_bytes", "model_bytes", "budget")
        return dict(zip(keys, (int(v) for v in out)))

    def save(self, path, degree_bounds=()):
        """Write the SRS as an ark-serialize file (marlin_b200/srsfile.py).  The G2 half -- h, beta h and SonicKZG10's
        beta^-(max_degree - d) h per enforced bound -- comes from the trapdoor of a test SRS, or from the file it was loaded from."""
        from . import srsfile
        L = _lib.lib()
        g1 = 2 * srsfile.fq_bytes(self.curve_id)
        n = self.max_degree + 1
        powers = np.zeros(n * g1, dtype=np.uint8)
        _lib.check(L.b2m_srs_export_g1(self.handle, 0, n, _lib.ptr(powers)))
        gam = np.zeros(len(self.gamma_indices) * g1, dtype=np.uint8)
        _lib.check(L.b2m_g1_to_uncompressed(self.ctx.handle, self.curve_id, _lib.ptr(np.ascontiguousarray(self.gamma_limbs)), len(self.gamma_indices),
                                            _lib.ptr(gam)))
        graw = gam.tobytes()
        gamma = {int(k): graw[i * g1:(i + 1) * g1] for i, k in enumerate(self.gamma_indices)}
        if self.trapdoor is not None:
            h, beta_h, neg = srsfile.g2_setup(self.curve_id, fields.FR_MODULUS[self.curve_id], self.trapdoor[0], self.max_degree, degree_bounds)
        elif self.g2 is not None:
            h, beta_h, neg = self.g2
        else:
            raise ValueError("this SRS has no G2 half (neither a trapdoor nor a source file)")
        srsfile.write_srs(path, self.curve_id, powers.tobytes(), gamma, h, beta_h, neg)

    def save_ark(self, path, compressed=True, degree_bounds=()):
        """Write the SRS as a raw arkworks `kzg10::UniversalParams` file (`serialize` or `serialize_uncompressed`, no header;
        marlin_b200/srsfile.py::read_ark).  An SRS from load_ark_srs writes everything its file held, so loading and saving in
        the same form reproduces the file byte for byte (the point at infinity, should a file hold one, is written with zero
        coordinates).  Otherwise the gamma powers are those on the device and the G2 half is made as `save` makes it."""
        from . import srsfile
        L = _lib.lib()
        cid = self.curve_id
        g1, g2 = srsfile.point_sizes(cid, compressed)
        ark = self.ark
        if ark is not None:
            gkeys, glimbs = ark["gamma_keys"], ark["gamma_limbs"]
            h, beta_h, nkeys, neg = ark["h"], ark["beta_h"], ark["neg_keys"], ark["neg"]
        else:
            gkeys, glimbs = np.asarray(self.gamma_indices, dtype=np.uint64), np.ascontiguousarray(self.gamma_limbs)
            order = np.argsort(gkeys, kind="stable")
            gkeys, glimbs = gkeys[order], np.ascontiguousarray(glimbs[order])
            if self.trapdoor is not None:
                h, beta_h, negd = srsfile.g2_setup(cid, fields.FR_MODULUS[cid], self.trapdoor[0], self.max_degree, degree_bounds)
            elif self.g2 is not None:
                h, beta_h, negd = self.g2
            else:
                raise ValueError("this SRS has no G2 half (neither a trapdoor nor a source file)")
            nkeys = np.asarray(sorted(negd), dtype=np.uint64)
            neg = np.frombuffer(b"".join(negd[int(k)] for k in nkeys), dtype=np.uint8).reshape(len(nkeys), 4 * srsfile.fq_bytes(cid))
            h, beta_h = np.frombuffer(h, dtype=np.uint8), np.frombuffer(beta_h, dtype=np.uint8)

        def g1_bytes(limbs):
            limbs = np.ascontiguousarray(limbs, dtype=np.uint64)
            out = np.zeros(len(limbs) * g1, dtype=np.uint8)
            conv = L.b2m_g1_to_compressed if compressed else L.b2m_g1_to_uncompressed
            _lib.check(conv(self.ctx.handle, cid, _lib.ptr(limbs), len(limbs), _lib.ptr(out)))
            return out

        def g2_bytes(unc):
            unc = np.ascontiguousarray(unc, dtype=np.uint8)
            if not compressed:
                return unc
            n = unc.size // (2 * g2)
            out = np.zeros(n * g2, dtype=np.uint8)
            _lib.check(L.b2m_g2_to_compressed(cid, _lib.ptr(unc), n, _lib.ptr(out)))
            return out

        srsfile.write_ark(path, cid, compressed, g1_bytes(self.powers_limbs), gkeys, g1_bytes(glimbs), g2_bytes(h), g2_bytes(beta_h), nkeys,
                          g2_bytes(neg).reshape(len(nkeys), g2))

    def close(self):
        if self.handle:
            _lib.lib().b2m_srs_destroy(self.handle)
            self.handle = None


class IndexProverKey:
    """`IndexProverKey` on the device (b2m_index).  `r1cs` supplies num_constraints, num_variables and num_instance."""

    def __init__(self, srs, handle, r1cs, pc):
        self.srs, self.handle, self.pc = srs, handle, pc
        self.num_constraints, self.num_variables = r1cs.num_constraints, r1cs.num_variables
        self.num_instance = r1cs.num_instance
        self.file_g2 = None  # (h, beta_h, {D - d: neg power}) as uncompressed bytes, when loaded from a key file
        L = _lib.lib()
        n = ctypes.c_size_t(0)
        _lib.check(L.b2m_index_vk_bytes(handle, None, 0, ctypes.byref(n)))
        buf = (ctypes.c_uint8 * n.value)()
        _lib.check(L.b2m_index_vk_bytes(handle, buf, n.value, ctypes.byref(n)))
        self.vk_bytes = bytes(buf)
        lq = _lib.LIMBS[srs.curve_id][1]
        self.index_comms = np.zeros((6, 2 * lq), dtype=np.uint64)
        _lib.check(L.b2m_index_comms(handle, _lib.ptr(self.index_comms)))

    @property
    def residency(self):
        """"device" or "host": where the index keeps its twelve |K|-vectors (b2m_index_residency)."""
        host = ctypes.c_int(0)
        _lib.check(_lib.lib().b2m_index_residency(self.handle, ctypes.byref(host), None))
        return "host" if host.value else "device"

    @property
    def host_bytes(self):
        """Pinned host bytes of a host-resident index (0 when device-resident)."""
        n = ctypes.c_size_t(0)
        _lib.check(_lib.lib().b2m_index_residency(self.handle, None, ctypes.byref(n)))
        return n.value

    def timings(self):
        buf = ctypes.create_string_buffer(4096)
        _lib.check(_lib.lib().b2m_prove_timings(self.handle, buf, 4096))
        return json.loads(buf.value.decode() or "{}")

    def info(self):
        """`IndexInfo`: (num_variables, num_constraints, num_non_zero, num_instance_variables)"""
        nv, nc, nnz = struct.unpack_from("<QQQ", self.vk_bytes, 0)
        return nv, nc, nnz, self.num_instance

    def _vk_fields(self, compressed):
        """`IndexVerifierKey` of this index as marlin_b200.keyfile writes it: the verifier key `PC::trim` makes for the
        enforced bounds {|H| - 2, |K| - 2} (sorted, deduplicated), supported_degree = the index's max degree, max_degree = D."""
        from . import srsfile
        srs, cid = self.srs, self.srs.curve_id
        nv, nc, nnz, ni = self.info()
        D = srs.max_degree
        bounds = index_degree_bounds(nc, nnz)
        h, beta_h, neg = self.file_g2 or g2_half(srs, bounds)
        powers = np.ascontiguousarray(srs.powers_limbs)
        g1 = lambda limbs: g1_to_bytes(srs.ctx, cid, limbs, compressed)
        g2 = lambda unc: g2_to_bytes(cid, unc, compressed)
        if self.pc == _lib.PC_MARLIN_KZG10:
            bound_points = g1(np.stack([powers[D - d] for d in bounds]))
        else:
            missing = [d for d in bounds if D - d not in neg]
            if missing:
                raise ValueError(f"the SRS holds no neg_powers_of_h for the degree bounds {missing}")
            bound_points = g2(np.frombuffer(b"".join(neg[D - d] for d in bounds), dtype=np.uint8))
        g1b, g2b = srsfile.point_sizes(cid, compressed)
        return {"info": (nv, nc, nnz, ni), "comms": g1(self.index_comms).reshape(6, g1b), "g": g1(powers[:1]),
                "gamma_g": g1(srs.gamma_limbs[[list(srs.gamma_indices).index(0)]]), "h": g2(np.frombuffer(h, dtype=np.uint8)),
                "beta_h": g2(np.frombuffer(beta_h, dtype=np.uint8)), "bounds": bounds, "bound_points": bound_points.reshape(len(bounds), -1),
                "supported_degree": max_degree(nc, nv, nnz), "max_degree": D}

    def save_verifier_key(self, path, compressed=True):
        """Write the `IndexVerifierKey` `Marlin::index` returns for this index as a raw ark-serialize file
        (marlin_b200/keyfile.py).  The G2 half comes from the SRS trapdoor or its source file, as `Marlin.verifier_key` takes it."""
        from . import keyfile
        keyfile.write_verifier_key(path, self.pc, self._vk_fields(compressed))

    def save(self, path, compressed=True):
        """Write the `IndexProverKey` `Marlin::index` returns for this index as a raw ark-serialize file
        (marlin_b200/keyfile.py): the verifier key, empty commitment randomness, the matrices as the index received them,
        the six index polynomials (trailing zero coefficients stripped) with their evaluations on K, and the committer key
        `PC::trim` makes from the SRS.  Field elements are converted to canonical form on the GPU."""
        from . import keyfile
        L = _lib.lib()
        srs, cid = self.srs, self.srs.curve_id
        vk = self._vk_fields(compressed)
        nv, nc, nnz, ni = vk["info"]
        nnz_c, K = ctypes.c_size_t(0), ctypes.c_size_t(0)
        mnnz = np.zeros(3, dtype=np.uint64)
        _lib.check(L.b2m_index_sizes(self.handle, ctypes.byref(nnz_c), ctypes.byref(K), _lib.ptr(mnnz)))
        K = K.value
        vectors = np.zeros((12, K, keyfile.FR_BYTES), dtype=np.uint8)
        row_ptrs = [np.zeros(nc + 1, dtype=np.uint64) for _ in range(3)]
        cols = [np.zeros(max(int(n), 1), dtype=np.uint64) for n in mnnz]
        coeffs = [np.zeros((max(int(n), 1), keyfile.FR_BYTES), dtype=np.uint8) for n in mnnz]
        arr = lambda xs: (ctypes.c_void_p * 3)(*[x.ctypes.data for x in xs])
        _lib.check(L.b2m_index_export(self.handle, _lib.ptr(vectors), arr(row_ptrs), arr(cols), arr(coeffs)))
        mats = [(row_ptrs[m], cols[m][:int(mnnz[m])], coeffs[m][:int(mnnz[m])]) for m in range(3)]
        dom = domain_bytes(cid, K)
        index = {"info": vk["info"], "matrices": mats, "coeffs": list(vectors[:6]), "evals": list(vectors[6:]), "domains": [dom] * 6}
        D = srs.max_degree
        bounds = vk["bounds"]
        md = vk["supported_degree"]
        powers = np.ascontiguousarray(srs.powers_limbs)
        g1 = lambda limbs: g1_to_bytes(srs.ctx, cid, limbs, compressed)
        gamma = lambda idx: g1(srs_gamma_powers(srs, idx))
        ck = {"powers": g1(powers[:md + 1]), "shifted": g1(powers[D - bounds[-1]:]), "gamma": gamma([0, 1, 2]), "bounds": bounds,
              "max_degree": D}
        if self.pc == _lib.PC_SONIC_KZG10:
            ck["shifted_gamma"] = {d: gamma([D - d + i for i in range(3) if D - d + i < D + 2]) for d in bounds}
        g1b, _ = srsfile.point_sizes(cid, compressed)
        for k in ("powers", "shifted", "gamma"):
            ck[k] = ck[k].reshape(-1, g1b)
        if "shifted_gamma" in ck:
            ck["shifted_gamma"] = {d: v.reshape(-1, g1b) for d, v in ck["shifted_gamma"].items()}
        keyfile.write_prover_key(path, self.pc, vk, index, ck)

    def close(self):
        if self.handle:
            _lib.lib().b2m_index_destroy(self.handle)
            self.handle = None


class VerifierKey:
    """`IndexVerifierKey` + the verifier half of the SRS (b2m_vk), built by `Marlin.verifier_key` from public data."""

    def __init__(self, ctx, handle, curve_id, pc):
        self.ctx, self.handle, self.curve_id, self.pc = ctx, handle, curve_id, pc

    def timings(self):
        """Phase split (ms) of the last verify_batch: decode, transcript, MSM tables, MSMs, pairings, bisection."""
        buf = ctypes.create_string_buffer(4096)
        _lib.check(_lib.lib().b2m_verify_timings(self.handle, buf, 4096))
        return json.loads(buf.value.decode() or "{}")

    def close(self):
        if self.handle:
            _lib.lib().b2m_vk_destroy(self.handle)
            self.handle = None


class PcVerifierKey:
    """`PC::VerifierKey` of MarlinKZG10 / SonicKZG10 (b2m_pc_vk), built by `Marlin.pc_verifier_key`."""

    def __init__(self, ctx, handle, curve_id, pc, degree_bounds):
        self.ctx, self.handle, self.curve_id, self.pc, self.degree_bounds = ctx, handle, curve_id, pc, degree_bounds

    def timings(self):
        """Phase split (ms) of the last check_combinations / batch_check: decode, terms, MSM tables, fold, MSMs, pairings."""
        buf = ctypes.create_string_buffer(4096)
        _lib.check(_lib.lib().b2m_pc_vk_timings(self.handle, buf, 4096))
        return json.loads(buf.value.decode() or "{}")

    def close(self):
        if self.handle:
            _lib.lib().b2m_pc_vk_destroy(self.handle)
            self.handle = None


class OpeningSet:
    """The inputs of one `PC::check_combinations` (or `batch_check`) call.
    commitments: {label: G1} with G1 compressed ark-serialize bytes or affine Montgomery limbs (`g1_to_bytes` converts);
    shifted: {label: G1}, MarlinKZG10's `shifted_comm` of bounded commitments; degree_bounds: {label: bound} (absent = None);
    lcs: [(label, [(coeff, commitment label or None for LCTerm::One)])] (None for `batch_check`: one LC per commitment);
    query_set: [(lc label, (point label, point))]; evaluations: {(lc label, point): value}; proofs: [(w, random_v or None)],
    one `kzg10::Proof` per point label in label order; challenge: the opening challenge xi.  Field elements are Python ints."""

    def __init__(self, commitments, query_set, evaluations, proofs, challenge, lcs=None, degree_bounds=None, shifted=None):
        self.commitments, self.query_set, self.evaluations, self.proofs = commitments, query_set, evaluations, proofs
        self.challenge, self.lcs, self.degree_bounds, self.shifted = challenge, lcs, degree_bounds or {}, shifted or {}


def _p2(n):
    s = 1
    while s < n:
        s *= 2
    return s


def index_degree_bounds(num_constraints, num_non_zero):
    """The bounds `Marlin::index` enforces, {|H| - 2, |K| - 2} sorted and deduplicated [reference src/ahp/mod.rs:96-106]"""
    return sorted({_p2(num_constraints) - 2, _p2(num_non_zero) - 2})


def g2_half(srs, bounds):
    """h, beta h and {D - d: beta^-(D - d) h} per bound d (uncompressed bytes) of an SRS: from its trapdoor, or from the file
    it was loaded from."""
    from . import srsfile
    cid = srs.curve_id
    if srs.trapdoor is not None:
        return srsfile.g2_setup(cid, fields.FR_MODULUS[cid], srs.trapdoor[0], srs.max_degree, bounds)
    if srs.g2 is not None:
        return srs.g2
    raise ValueError("this SRS has no G2 half (neither a trapdoor nor a source file)")


def g1_to_bytes(ctx, cid, limbs, compressed):
    """affine Montgomery limbs -> ark-serialize G1 bytes (GPU), flat uint8"""
    limbs = np.ascontiguousarray(limbs, dtype=np.uint64).reshape(-1, 2 * _lib.LIMBS[cid][1])
    g1, _ = srsfile.point_sizes(cid, compressed)
    out = np.zeros(len(limbs) * g1, dtype=np.uint8)
    conv = _lib.lib().b2m_g1_to_compressed if compressed else _lib.lib().b2m_g1_to_uncompressed
    _lib.check(conv(ctx.handle, cid, _lib.ptr(limbs), len(limbs), _lib.ptr(out)))
    return out


def g2_to_bytes(cid, unc, compressed):
    """uncompressed G2 bytes -> the chosen form, flat uint8"""
    unc = np.ascontiguousarray(unc, dtype=np.uint8).reshape(-1)
    if not compressed:
        return unc
    _, g2 = srsfile.point_sizes(cid, True)
    n = unc.size // (2 * g2)
    out = np.zeros(n * g2, dtype=np.uint8)
    _lib.check(_lib.lib().b2m_g2_to_compressed(cid, _lib.ptr(unc), n, _lib.ptr(out)))
    return out


def srs_gamma_powers(srs, idx):
    """powers_of_gamma_g at the given exponents, affine limbs: from the whole source file when there is one, else from the
    powers on the device"""
    if srs.ark is not None:
        keys, limbs = srs.ark["gamma_keys"], srs.ark["gamma_limbs"]
    else:
        keys, limbs = np.asarray(srs.gamma_indices, dtype=np.uint64), np.asarray(srs.gamma_limbs)
    out = []
    for i in idx:
        hit = np.flatnonzero(keys == np.uint64(i))
        if not len(hit):
            raise ValueError(f"the SRS holds no powers_of_gamma_g[{i}]")
        out.append(limbs[int(hit[0])])
    return np.stack(out)


def pairing_check(ctx, curve, g2_points, products):
    """`product_of_pairings(pairs).is_one()` for many products on the GPU (b2m_pairing_check).  curve: a C ABI curve id
    (_lib.CURVE_*).  g2_points: a list of
    uncompressed ark-serialize G2 byte strings; products: a list of products, each a list of (g1, k) pairs with g1 an array
    of 2 * limbs uint64 (affine Montgomery, zeros = infinity) and k an index into g2_points.  Returns a list of bools."""
    cid = curve
    nq = _lib.LIMBS[cid][1]
    off = np.zeros(len(products) + 1, dtype=np.uint64)
    g1, idx = [], []
    for k, pr in enumerate(products):
        for pt, q in pr:
            g1.append(np.asarray(pt, dtype=np.uint64).reshape(2 * nq))
            idx.append(q)
        off[k + 1] = len(idx)
    g1a = np.concatenate(g1) if g1 else np.zeros(2 * nq, dtype=np.uint64)
    idxa = np.asarray(idx or [0], dtype=np.uint32)
    g2a = np.frombuffer(b"".join(g2_points) or b"\0", dtype=np.uint8)
    out = np.zeros(max(1, len(products)), dtype=np.int32)
    _lib.check(_lib.lib().b2m_pairing_check(ctx.handle, cid, len(g2_points), _lib.ptr(g2a), len(products), _lib.ptr(off), _lib.ptr(g1a),
                                            _lib.ptr(idxa), _lib.ptr(out)))
    return [bool(v) for v in out[:len(products)]]


def domain_bytes(cid, size):
    """`Radix2EvaluationDomain::new(size)` as ark-serialize writes it (b2m_domain_ark)"""
    out = np.zeros(172, dtype=np.uint8)
    _lib.check(_lib.lib().b2m_domain_ark(cid, size.bit_length() - 1, _lib.ptr(out)))
    return out.tobytes()


def _proof_args(curve_ids, public_inputs, proofs):
    """b2m_verify_batch / b2m_verify_multi arguments for proof i of curve curve_ids[i]: (input pointers, input lengths, proof
    pointers, proof lengths), the verdict array, and the buffers behind the pointers (kept alive by the caller)"""
    n = len(proofs)
    ins = [np.ascontiguousarray(_lib.ints_to_limbs([fields.fr_to_mont(c, v % fields.FR_MODULUS[c]) for v in x], 4))
           for c, x in zip(curve_ids, public_inputs)]
    bufs = [np.frombuffer(bytes(p), dtype=np.uint8).copy() if len(p) else np.zeros(1, dtype=np.uint8) for p in proofs]
    in_ptrs = (ctypes.c_void_p * max(n, 1))(*[a.ctypes.data for a in ins])
    in_lens = (ctypes.c_size_t * max(n, 1))(*[len(a) for a in ins])
    pr_ptrs = (ctypes.c_void_p * max(n, 1))(*[a.ctypes.data for a in bufs])
    pr_lens = (ctypes.c_size_t * max(n, 1))(*[len(p) for p in proofs])
    return (in_ptrs, in_lens, pr_ptrs, pr_lens), (ctypes.c_int * max(n, 1))(), (ins, bufs)


def verify_many(entries, rng):
    """`Marlin::verify` for proofs under many verifier keys in one batch (b2m_verify_multi).  entries: (vk, public_input,
    proof_bytes) triples, public inputs as `Marlin.verify_batch` takes them; the keys (collected by identity) must share one
    Context and curve, their PC variants and SRSs may differ.  Returns True / False / None per entry: what
    `verify_batch(vk, ...)` gives that entry under its own key.  rng: as for `verify_batch`."""
    keys, key_of = [], []
    for vk, _, _ in entries:
        k = next((j for j, x in enumerate(keys) if x is vk), None)
        if k is None:
            k = len(keys)
            keys.append(vk)
        key_of.append(k)
    n = len(entries)
    args, verdicts, _keep = _proof_args([keys[k].curve_id for k in key_of], [e[1] for e in entries], [e[2] for e in entries])
    vks = (ctypes.c_void_p * max(len(keys), 1))(*[k.handle for k in keys])
    kof = (ctypes.c_uint32 * max(n, 1))(*key_of)
    _lib.check(_lib.lib().b2m_verify_multi(len(keys), vks, n, kof, *args, ctypes.byref(rng.c) if rng is not None else None, verdicts))
    return [{1: True, 0: False}.get(verdicts[i]) for i in range(n)]


def pc_check_arrays(cid, sets, identity, limbs_to_bytes):
    """The arrays of b2m_pc_check_combinations (after n_sets, in argument order) for OpeningSets of curve cid: commitments
    in label order, LCs in label order (identity: one per commitment, as `batch_check` forms them), points in point-label
    order, the query set deduplicated.  limbs_to_bytes: affine limbs (k, 2 * Fq limbs) -> k compressed G1 points."""
    r = fields.FR_MODULUS[cid]
    fq_bytes = 8 * _lib.LIMBS[cid][1]
    g1s, shifted = [], []
    comm_off, bounds, has_shifted = [0], [], []
    lc_off, term_off, lc_comm, coeffs = [0], [0], [], []
    point_off, points, ws, has_rv, rvs = [0], [], [], [], []
    query_off, q_lc, q_pt, evals, xis = [0], [], [], [], []
    fr = lambda v: fields.fr_to_mont(cid, v % r)  # noqa: E731
    canon = lambda v: int(v).to_bytes(32, "little")  # noqa: E731  (not reduced: a value >= r is the library's to reject)
    for s in sets:
        labels = sorted(s.commitments)
        ci = {l: i for i, l in enumerate(labels)}
        for l in labels:
            g1s.append(s.commitments[l])
            d = s.degree_bounds.get(l)
            bounds.append(-1 if d is None else int(d))
            sh = s.shifted.get(l)
            has_shifted.append(0 if sh is None else 1)
            shifted.append(bytes(fq_bytes) if sh is None else sh)
        comm_off.append(len(g1s))
        if identity:
            if s.lcs is not None:
                raise ValueError("batch_check takes no linear combinations")
            lcs = [(l, [(1, l)]) for l in labels]
        else:
            lcs = sorted(s.lcs, key=lambda lc: lc[0])
        li = {lc[0]: i for i, lc in enumerate(lcs)}
        if len(li) != len(lcs):
            raise ValueError("two linear combinations share a label")
        for _, terms in lcs:
            for c, t in terms:
                if t is not None and t not in ci:
                    raise ValueError(f"MissingPolynomial: no commitment labelled {t!r}")
                lc_comm.append(-1 if t is None else ci[t])
                coeffs.append(fr(c))
            term_off.append(len(lc_comm))
        lc_off.append(len(term_off) - 1)
        queries = sorted(set((lc, (pl, int(pt))) for lc, (pl, pt) in s.query_set))
        at = {}
        for _, (pl, pt) in queries:
            if at.setdefault(pl, pt) != pt:
                raise ValueError(f"point label {pl!r} names two points")
        pls = sorted(at)
        pi = {pl: j for j, pl in enumerate(pls)}
        if len(s.proofs) != len(pls):
            raise ValueError(f"{len(s.proofs)} opening proofs for {len(pls)} points")
        for pl, (w, rv) in zip(pls, s.proofs):
            points.append(fr(at[pl]))
            ws.append(w)
            has_rv.append(0 if rv is None else 1)
            rvs.append(canon(0 if rv is None else rv))
        point_off.append(len(points))
        for lc, (pl, pt) in queries:
            if lc not in li:
                raise ValueError(f"MissingLinearCombination: no LC labelled {lc!r}")
            if (lc, pt) not in s.evaluations:
                raise ValueError(f"MissingEvaluation for {lc!r} at point {pl!r}")
            q_lc.append(li[lc])
            q_pt.append(pi[pl])
            evals.append(canon(s.evaluations[(lc, pt)]))
        query_off.append(len(q_lc))
        xis.append(fr(s.challenge))

    def g1_blob(items):
        out = np.zeros((max(len(items), 1), fq_bytes), dtype=np.uint8)
        limbs = [i for i, it in enumerate(items) if not isinstance(it, (bytes, bytearray))]
        for i, it in enumerate(items):
            if isinstance(it, (bytes, bytearray)):
                out[i] = np.frombuffer(bytes(it), dtype=np.uint8)
        if limbs:
            out[limbs] = limbs_to_bytes(np.stack([np.asarray(items[i], dtype=np.uint64).reshape(-1) for i in limbs])).reshape(-1, fq_bytes)
        return out

    def arr(vals, dtype):
        return np.ascontiguousarray(np.asarray(vals if vals else [0], dtype=dtype))

    def fr_arr(vals):
        return np.ascontiguousarray(_lib.ints_to_limbs(vals or [0], 4))

    def byte_arr(vals):
        return np.frombuffer(b"".join(vals) or bytes(32), dtype=np.uint8).copy()

    return [arr(comm_off, np.uint64), g1_blob(g1s), arr(bounds, np.int64), arr(has_shifted, np.int32), g1_blob(shifted),
            arr(lc_off, np.uint64), arr(term_off, np.uint64), arr(lc_comm, np.int64), fr_arr(coeffs), arr(point_off, np.uint64),
            fr_arr(points), g1_blob(ws), arr(has_rv, np.int32), byte_arr(rvs), arr(query_off, np.uint64), arr(q_lc, np.uint64),
            arr(q_pt, np.uint64), byte_arr(evals), fr_arr(xis)]


def max_degree(num_constraints, num_variables, num_non_zero):
    """`AHPForR1CS::max_degree` [reference src/ahp/mod.rs:71-93]"""
    def p2(n):
        s = 1
        while s < n:
            s *= 2
        return s
    h = p2(max(num_variables, num_constraints))
    k = p2(num_non_zero)
    return max(2 * h + 1 - 2, 3 * h + 2 - 3, h, h, k - 1)


class Marlin:
    """`Marlin<F, PC, FS>` for one curve and PC scheme on one GPU."""

    def __init__(self, curve="bls12_381", pc="marlin_kzg10", device=0, ctx=None):
        self.curve_id = fields.CURVE_IDS[curve]
        self.pc = PC_IDS[pc]
        self.ctx = ctx or Context(device)

    # -- universal_setup ---------------------------------------------------------------------------
    def universal_setup(self, num_constraints, num_variables, num_non_zero, beta, g=None, gamma=7, degree_bounds=(),
                        window_bits=0, window_tables=0):
        """[reference src/lib.rs:79-96] with an explicit trapdoor: an insecure test SRS exactly like the
        reference's `universal_setup(.., test_rng)`, generated on the GPU.  `degree_bounds`: bounds whose
        shifted gamma powers SonicKZG10 will need (ignored by MarlinKZG10).  window_bits / window_tables = 0: chosen by the
        library from the key size and the context's memory budget (b2m_srs_create_layout)."""
        md = max_degree(num_constraints, num_variables, num_non_zero)
        return self.srs_from_trapdoor(md, beta, g, gamma, degree_bounds, window_bits, window_tables)

    def srs_from_trapdoor(self, md, beta, g=None, gamma=7, degree_bounds=(), window_bits=0, window_tables=0):
        L = _lib.lib()
        cid = self.curve_id
        lq = _lib.LIMBS[cid][1]
        g = g or fields.G1_GENERATOR[cid]
        r = fields.FR_MODULUS[cid]
        g_l = _lib.ints_to_limbs([fields.fq_to_mont(cid, g[0]), fields.fq_to_mont(cid, g[1])], lq).reshape(1, 2 * lq)
        beta_l = _lib.ints_to_limbs([beta % r], 4)
        powers = np.zeros((md + 1, 2 * lq), dtype=np.uint64)
        _lib.check(L.b2m_g1_powers(self.ctx.handle, cid, _lib.ptr(g_l), _lib.ptr(beta_l), md + 1, _lib.ptr(powers)))
        # gamma powers: gamma * beta^i * g = one-term MSMs of the G1 powers
        idx = [0, 1, 2]
        for d in sorted(set(degree_bounds)):
            idx += [md - d + i for i in range(3) if md - d + i <= md]
        idx = sorted(set(idx))
        # powers_of_gamma_g at the needed exponents: FixedBaseMSM(gamma_g, [beta^i]) with gamma_g = gamma * g
        gamma_g = np.zeros((1, 2 * lq), dtype=np.uint64)
        _lib.check(L.b2m_fixed_base_msm(self.ctx.handle, cid, _lib.ptr(g_l), _lib.ptr(_lib.ints_to_limbs([gamma % r], 4)), 1, _lib.ptr(gamma_g)))
        exps = _lib.ints_to_limbs([pow(beta % r, i, r) for i in idx], 4)
        gam = np.zeros((len(idx), 2 * lq), dtype=np.uint64)
        _lib.check(L.b2m_fixed_base_msm(self.ctx.handle, cid, _lib.ptr(gamma_g), _lib.ptr(exps), len(idx), _lib.ptr(gam)))
        srs = self.srs_from_points(powers, gam, idx, window_bits, window_tables)
        srs.trapdoor = (beta % r, gamma % r)
        return srs

    def load_srs(self, path, window_bits=0, window_tables=0):
        """Load an SRS file (marlin_b200/srsfile.py layout; `deserialize_unchecked` semantics: no subgroup check)."""
        from . import srsfile
        L = _lib.lib()
        d = srsfile.read_srs(path)
        if d["curve_id"] != self.curve_id:
            raise ValueError(f"{path} holds curve {d['curve_id']}, this Marlin instance is curve {self.curve_id}")
        lq = _lib.LIMBS[self.curve_id][1]
        g1 = 2 * srsfile.fq_bytes(self.curve_id)
        n = len(d["powers"]) // g1
        powers = np.zeros((n, 2 * lq), dtype=np.uint64)
        raw = np.frombuffer(d["powers"], dtype=np.uint8)
        _lib.check(L.b2m_g1_from_uncompressed(self.ctx.handle, self.curve_id, _lib.ptr(np.ascontiguousarray(raw)), n, _lib.ptr(powers)))
        idx = sorted(d["gamma"])
        graw = np.frombuffer(b"".join(d["gamma"][k] for k in idx), dtype=np.uint8)
        gam = np.zeros((len(idx), 2 * lq), dtype=np.uint64)
        _lib.check(L.b2m_g1_from_uncompressed(self.ctx.handle, self.curve_id, _lib.ptr(np.ascontiguousarray(graw)), len(idx), _lib.ptr(gam)))
        srs = self.srs_from_points(powers, gam, idx, window_bits, window_tables)
        srs.g2 = (d["h"], d["beta_h"], d["neg_powers"])
        return srs

    def load_ptau(self, path, max_degree=None, check=True, rng=None, window_bits=0, window_tables=0):
        """Load a snarkjs Powers-of-Tau file (marlin_b200/ptau.py) -- the output of a multi-party ceremony -- as a MarlinKZG10
        SRS of max degree D = max_degree (default: the whole file, 2^(power+1) - 2).  powers_of_g = tauG1[0..=D], the gamma
        powers {0, 1, 2} = alphaTauG1[0..=2] (alpha plays gamma: it is accumulated over the contributions like tau and known to
        nobody if one contributor was honest), h = tauG2[0], beta_h = tauG2[1]; nothing else is read.  Every point is decoded
        and validated on the GPU (coordinates below p, on the curve, in the prime-order subgroup) and must be finite; the first
        bad one raises B2MError (B2M_ERR_SERIALIZATION) naming it, e.g. `tauG1[1048573]: not in the prime-order subgroup`.
        check=True then decides on the GPU that the points are one chain of powers (b2m_srs_check_powers, with rng or an
        OS-seeded ZkRng()); a break raises naming the point, e.g. `tauG1[7] is not tau times tauG1[6]`.  This proves the file
        is a well-formed powers-of-tau SRS, not which ceremony made it.  SonicKZG10 is refused: the file has no
        neg_powers_of_h.  verifier_key, save and save_ark work on the result as on any loaded SRS."""
        from . import ptau
        if self.pc == _lib.PC_SONIC_KZG10:
            raise ValueError("a .ptau file holds no neg_powers_of_h: SonicKZG10 cannot use it (MarlinKZG10 can)")
        f = ptau.read_ptau(path)
        cid = self.curve_id
        if f.curve_id != cid:
            raise ValueError(f"{path} is a {_CURVE_NAMES[f.curve_id]} file, this Marlin instance is {_CURVE_NAMES[cid]}")
        D = f.max_degree if max_degree is None else int(max_degree)
        if D > f.max_degree:
            raise ValueError(f"{path}: max degree {D} needs a power-{ptau.power_for_degree(D)} file; this one is power {f.power} "
                             f"(max degree {f.max_degree})")
        if D < 1:
            raise ValueError(f"max degree {D} < 1")
        if f.counts[4] < 3:
            raise ValueError(f"{path}: alphaTauG1 holds {f.counts[4]} points, the SRS needs 3 (power >= 2)")
        L = _lib.lib()
        lq = _lib.LIMBS[cid][1]

        def bad(field, i, reason):
            raise _lib.B2MError(_lib.ERR_SERIALIZATION, f"{field}[{i}]: {reason}")

        def g1(pts, field):
            pts = np.ascontiguousarray(pts)
            out = np.zeros((len(pts), 2 * lq), dtype=np.uint64)
            bi, br = ctypes.c_size_t(0), ctypes.c_int(0)
            rc = L.b2m_g1_decode_lem(self.ctx.handle, cid, _lib.ptr(pts.reshape(-1)), len(pts), _lib.ptr(out), ctypes.byref(bi), ctypes.byref(br))
            if rc == _lib.ERR_SERIALIZATION:
                bad(field, bi.value, _lib.POINT_REASONS.get(br.value, "invalid point"))
            _lib.check(rc)
            inf = np.flatnonzero(~out.any(axis=1))
            if len(inf):
                bad(field, int(inf[0]), "the point at infinity")
            return out

        powers = g1(f.tau_g1(D + 1), "tauG1")
        gam = g1(f.alpha_tau_g1(3), "alphaTauG1")
        g2in = np.ascontiguousarray(f.tau_g2(2))
        g2 = np.zeros((2, 4 * f.n8), dtype=np.uint8)
        bi, br = ctypes.c_size_t(0), ctypes.c_int(0)
        rc = L.b2m_g2_decode_lem(self.ctx.handle, cid, _lib.ptr(g2in.reshape(-1)), 2, _lib.ptr(g2), ctypes.byref(bi), ctypes.byref(br))
        if rc == _lib.ERR_SERIALIZATION:
            bad("tauG2", bi.value, _lib.POINT_REASONS.get(br.value, "invalid point"))
        _lib.check(rc)
        for i in range(2):
            if g2[i, -1] & 0x40:
                bad("tauG2", i, "the point at infinity")
        srs = self.srs_from_points(powers, gam, [0, 1, 2], window_bits, window_tables)
        srs.g2 = (g2[0].tobytes(), g2[1].tobytes(), {})
        if check:
            names = {0: lambda i: f"tauG1[{i + 1}] is not tau times tauG1[{i}]" + (" (or tauG2[1] is not tau times tauG2[0])" if i == 0 else ""),
                     1: lambda k: f"alphaTauG1[{k + 1}] is not tau times alphaTauG1[{k}]"}
            self._check_powers(srs, g2[0], g2[1], [], None, rng, names)
        return srs

    def _check_powers(self, srs, h, beta_h, neg_keys, neg, rng, names):
        """b2m_srs_check_powers; on a break the SRS is closed and B2MError (B2M_ERR_SERIALIZATION) raised with
        names[family](index)"""
        rng = rng if rng is not None else ZkRng()
        ok, kind, idx = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_size_t(0)
        h, beta_h = np.ascontiguousarray(h, dtype=np.uint8), np.ascontiguousarray(beta_h, dtype=np.uint8)
        keys = np.ascontiguousarray(neg_keys, dtype=np.uint64)
        negb = np.ascontiguousarray(neg, dtype=np.uint8) if len(keys) else None
        try:
            _lib.check(_lib.lib().b2m_srs_check_powers(srs.handle, _lib.ptr(h), _lib.ptr(beta_h), len(keys), _lib.ptr(keys) if len(keys) else None,
                                                       _lib.ptr(negb) if len(keys) else None, ctypes.byref(rng.c), ctypes.byref(ok),
                                                       ctypes.byref(kind), ctypes.byref(idx)))
        except Exception:
            srs.close()
            raise
        if not ok.value:
            srs.close()
            raise _lib.B2MError(_lib.ERR_SERIALIZATION, names[kind.value](int(idx.value)))

    def load_ark_srs(self, path, compressed=True, degree_bounds=(), window_bits=0, window_tables=0, check_powers=False, rng=None):
        """Load a raw arkworks `kzg10::UniversalParams` file, as `UniversalParams::serialize` (compressed=True) or
        `serialize_uncompressed` wrote it, with `deserialize` semantics: every point is decoded and validated on the GPU (flags,
        coordinates below p, on the curve, in the prime-order subgroup), and the first invalid one raises B2MError
        (B2M_ERR_SERIALIZATION) naming its field and index, e.g. `powers_of_g[1048573]: not in the prime-order subgroup`
        (BTreeMap fields are indexed by key).  The device key receives the gamma powers `universal_setup(degree_bounds=...)`
        would make -- indices 0, 1, 2 and D - d + {0, 1, 2} per bound d -- while the returned SRS keeps the whole file (every
        gamma power, every G2 point, contiguous) for `verifier_key` and `save_ark`.  check_powers=True also decides on the GPU
        that the points are one chain of powers of one beta (b2m_srs_check_powers over powers_of_g, the gamma powers on the
        device and every neg_powers_of_h entry, with rng or an OS-seeded ZkRng()); a break raises B2MError naming the point,
        e.g. `powers_of_g[7] is not beta times powers_of_g[6]`."""
        from . import srsfile
        L = _lib.lib()
        cid = self.curve_id
        lq = _lib.LIMBS[cid][1]
        g1, g2 = srsfile.point_sizes(cid, compressed)
        d = srsfile.read_ark(path, cid, compressed)

        def bad(field, names, idx, reason):
            raise _lib.B2MError(_lib.ERR_SERIALIZATION, f"{field}[{names(idx)}]: {_lib.POINT_REASONS.get(reason, 'invalid point')}")

        def g1_decode(pts, field, names=int):
            pts = np.ascontiguousarray(pts)
            out = np.zeros((len(pts), 2 * lq), dtype=np.uint64)
            bi, br = ctypes.c_size_t(0), ctypes.c_int(0)
            rc = L.b2m_g1_decode_ark(self.ctx.handle, cid, _lib.ptr(pts.reshape(-1)), len(pts), int(compressed), _lib.ptr(out), ctypes.byref(bi),
                                     ctypes.byref(br))
            if rc == _lib.ERR_SERIALIZATION:
                bad(field, names, bi.value, br.value)
            _lib.check(rc)
            return out

        n = len(d["powers"])
        if n < 1:
            raise ValueError(f"{path}: powers_of_g is empty")
        D = n - 1
        powers = g1_decode(d["powers"], "powers_of_g")
        gkeys = d["gamma_keys"]
        gamma_all = g1_decode(d["gamma"], "powers_of_gamma_g", lambda i: int(gkeys[i]))
        nkeys = d["neg_keys"]
        g2_in = np.concatenate([d["h"].reshape(1, g2), d["beta_h"].reshape(1, g2), d["neg"].reshape(-1, g2)])
        g2_out = np.zeros((len(g2_in), 4 * srsfile.fq_bytes(cid)), dtype=np.uint8)
        bi, br = ctypes.c_size_t(0), ctypes.c_int(0)
        rc = L.b2m_g2_decode_ark(self.ctx.handle, cid, _lib.ptr(g2_in.reshape(-1)), len(g2_in), int(compressed), _lib.ptr(g2_out), ctypes.byref(bi),
                                 ctypes.byref(br))
        if rc == _lib.ERR_SERIALIZATION:
            i = bi.value
            field, names = (("h", None), ("beta_h", None))[i] if i < 2 else ("neg_powers_of_h", lambda j: int(nkeys[j - 2]))
            if names is None:
                raise _lib.B2MError(rc, f"{field}: {_lib.POINT_REASONS.get(br.value, 'invalid point')}")
            bad(field, names, i, br.value)
        _lib.check(rc)
        # the gamma powers the PC needs on the device
        idx = {0, 1, 2}
        for b in sorted(set(degree_bounds)):
            idx |= {D - b + i for i in range(3) if 0 <= D - b + i <= D}
        idx = sorted(idx)
        pos = np.searchsorted(gkeys, np.asarray(idx, dtype=np.uint64))
        missing = [k for k, p in zip(idx, pos) if p >= len(gkeys) or int(gkeys[p]) != k]
        if missing:
            raise ValueError(f"{path}: powers_of_gamma_g holds no entry for the indices {missing}")
        srs = self.srs_from_points(powers, gamma_all[pos], idx, window_bits, window_tables)
        h, beta_h, neg = g2_out[0], g2_out[1], np.ascontiguousarray(g2_out[2:])
        srs.g2 = (h.tobytes(), beta_h.tobytes(), srsfile.G2Points(nkeys, neg))
        srs.ark = {"gamma_keys": gkeys, "gamma_limbs": gamma_all, "h": h, "beta_h": beta_h, "neg_keys": nkeys, "neg": neg}
        if check_powers:
            names = {0: lambda i: f"powers_of_g[{i + 1}] is not beta times powers_of_g[{i}]" + (" (or beta_h is not beta times h)" if i == 0 else ""),
                     1: lambda k: f"powers_of_gamma_g[{k + 1}] is not beta times powers_of_gamma_g[{k}]",
                     2: lambda k: f"neg_powers_of_h[{k}] is not beta^-{k} h (checked against powers_of_g[{k}])",
                     3: lambda k: f"neg_powers_of_h[{k}] is not beta^-{k} h (or powers_of_gamma_g[{k}] is not beta^{k} gamma g)"}
            self._check_powers(srs, h, beta_h, nkeys, neg, rng, names)
        return srs

    def srs_from_points(self, powers_limbs, gamma_limbs, gamma_indices, window_bits=0, window_tables=0):
        """Upload an existing SRS (affine Montgomery limbs, as ark-ff stores them).  window_tables > 0 keeps that many window
        tables instead of the planned number (the proof bytes do not depend on it)."""
        L = _lib.lib()
        h = ctypes.c_void_p()
        gi = np.asarray(gamma_indices, dtype=np.uint64)
        powers_limbs = np.ascontiguousarray(powers_limbs)
        gamma_limbs = np.ascontiguousarray(gamma_limbs)
        _lib.check(L.b2m_srs_create_layout(self.ctx.handle, self.curve_id, _lib.ptr(powers_limbs), len(powers_limbs), _lib.ptr(gamma_limbs),
                                           _lib.ptr(gi), len(gi), window_bits, window_tables, ctypes.byref(h)))
        return UniversalSRS(self.ctx, self.curve_id, h, len(powers_limbs) - 1, powers_limbs, gamma_limbs, [int(i) for i in gi])

    # -- PC::trim (Level 1) ---------------------------------------------------------------------------------
    def trim(self, srs, supported_degree, supported_hiding_bound, enforced_degree_bounds=()):
        """`PC::trim(pp, supported_degree, supported_hiding_bound, enforced_degree_bounds)` [reference src/lib.rs:112-121]
        -> CommitterKey (the verifier key's G1 part is read with CommitterKey.shift_power)."""
        L = _lib.lib()
        h = ctypes.c_void_p()
        b = np.asarray(sorted(enforced_degree_bounds), dtype=np.uint64)
        _lib.check(L.b2m_trim(srs.handle, self.pc, supported_degree, supported_hiding_bound, _lib.ptr(b) if len(b) else None, len(b),
                              ctypes.byref(h)))
        return CommitterKey(srs, h, self.pc, supported_degree, supported_hiding_bound, [int(x) for x in b])

    def open_combinations(self, ck, polys, rands, shifted_rands, lcs, query_set, points, challenge_limbs):
        """`PC::open_combinations` [reference src/lib.rs:292-302].  polys: (coeff limbs, degree_bound, hiding_bound) as for
        `commit`; rands / shifted_rands as returned by `commit`; lcs: list of term lists [(coeff Montgomery limbs (4,), poly index
        or None for the constant term)], in label order; query_set: [(lc index, point index)]; points: (n_points, 4) Montgomery
        limbs in point-label order.  Returns [(w affine limbs, random_v limbs or None)] per point."""
        L = _lib.lib()
        n = len(polys)
        lq = _lib.LIMBS[self.curve_id][1]
        arrs = [np.ascontiguousarray(p[0], dtype=np.uint64) for p in polys]
        ptrs = (ctypes.c_void_p * n)(*[a.ctypes.data for a in arrs])
        lens = (ctypes.c_size_t * n)(*[len(a) for a in arrs])
        db = (ctypes.c_int64 * n)(*[-1 if p[1] is None else p[1] for p in polys])
        hid = (ctypes.c_int * n)(*[0 if p[2] is None else 1 for p in polys])
        rands = np.ascontiguousarray(rands, dtype=np.uint64)
        shifted_rands = np.ascontiguousarray(shifted_rands, dtype=np.uint64)
        offs, lp, lcf = [0], [], []
        for terms in lcs:
            for coeff, idx in terms:
                lp.append(-1 if idx is None else idx)
                lcf.append(np.asarray(coeff, dtype=np.uint64).reshape(4))
            offs.append(len(lp))
        offs_a = (ctypes.c_size_t * len(offs))(*offs)
        lp_a = (ctypes.c_int64 * len(lp))(*lp)
        lcf_a = np.ascontiguousarray(np.stack(lcf), dtype=np.uint64)
        ql = (ctypes.c_size_t * len(query_set))(*[q[0] for q in query_set])
        qp = (ctypes.c_size_t * len(query_set))(*[q[1] for q in query_set])
        pts = np.ascontiguousarray(points, dtype=np.uint64).reshape(-1, 4)
        npts = len(pts)
        w = np.zeros((npts, 2 * lq), dtype=np.uint64)
        has = (ctypes.c_int * npts)()
        rv = np.zeros((npts, 4), dtype=np.uint64)
        _lib.check(L.b2m_ck_open_combinations(ck.handle, n, ptrs, lens, db, hid, _lib.ptr(rands), _lib.ptr(shifted_rands), rands.shape[1],
                                              len(lcs), offs_a, lp_a, _lib.ptr(lcf_a), len(query_set), ql, qp, npts, _lib.ptr(pts),
                                              _lib.ptr(np.ascontiguousarray(challenge_limbs, dtype=np.uint64)), _lib.ptr(w), has, _lib.ptr(rv)))
        return [(w[i], rv[i] if has[i] else None) for i in range(npts)]

    # -- PC::commit (Level 1) ------------------------------------------------------------------------------
    def commit(self, srs, polys, zk_rng=None):
        """`PC::commit(ck, polynomials, rng)` [reference src/lib.rs:125,172,193,213].  polys: list of
        (coeff_limbs uint64[n,4] Montgomery, degree_bound or None, hiding_bound or None).
        Returns (comms, shifted_comms, rands, shifted_rands) as limb arrays; rands are 4 Fr per polynomial."""
        L = _lib.lib()
        n = len(polys)
        lq = _lib.LIMBS[self.curve_id][1]
        arrs = [np.ascontiguousarray(p[0], dtype=np.uint64) for p in polys]
        ptrs = (ctypes.c_void_p * n)(*[a.ctypes.data for a in arrs])
        lens = (ctypes.c_size_t * n)(*[len(a) for a in arrs])
        db = (ctypes.c_int64 * n)(*[-1 if p[1] is None else p[1] for p in polys])
        hb = (ctypes.c_int64 * n)(*[-1 if p[2] is None else p[2] for p in polys])
        comm = np.zeros((n, 2 * lq), dtype=np.uint64)
        shifted = np.zeros((n, 2 * lq), dtype=np.uint64)
        rand = np.zeros((n, 4, 4), dtype=np.uint64)
        srand = np.zeros((n, 4, 4), dtype=np.uint64)
        rp = ctypes.byref(zk_rng.c) if zk_rng is not None else None
        if isinstance(srs, CommitterKey):  # `PC::commit(ck, ..)` with the committer key's degree / bound checks
            _lib.check(L.b2m_ck_commit(srs.handle, n, ptrs, lens, db, hb, rp, _lib.ptr(comm), _lib.ptr(shifted), _lib.ptr(rand), _lib.ptr(srand), 4))
        else:
            _lib.check(L.b2m_pc_commit(srs.handle, self.pc, n, ptrs, lens, db, hb, rp, _lib.ptr(comm), _lib.ptr(shifted), _lib.ptr(rand),
                                       _lib.ptr(srand), 4))
        return comm, shifted, rand, srand

    def open(self, srs, polys, rands, shifted_rands, point_limbs, challenge_limbs, max_degree_bound=None):
        """`PC::open_individual_opening_challenges` at one point [U marlin_pc / sonic_pc open].  polys as in `commit`
        (coeff limbs, degree_bound, _), rands / shifted_rands as returned by `commit`; point and opening challenge are
        Montgomery Fr limbs.  Returns (w affine limbs, random_v limbs or None)."""
        L = _lib.lib()
        n = len(polys)
        lq = _lib.LIMBS[self.curve_id][1]
        arrs = [np.ascontiguousarray(p[0], dtype=np.uint64) for p in polys]
        ptrs = (ctypes.c_void_p * n)(*[a.ctypes.data for a in arrs])
        lens = (ctypes.c_size_t * n)(*[len(a) for a in arrs])
        db = (ctypes.c_int64 * n)(*[-1 if p[1] is None else p[1] for p in polys])
        rands = np.ascontiguousarray(rands, dtype=np.uint64)
        shifted_rands = np.ascontiguousarray(shifted_rands, dtype=np.uint64)
        w = np.zeros(2 * lq, dtype=np.uint64)
        rv = np.zeros(4, dtype=np.uint64)
        has = ctypes.c_int(0)
        _lib.check(L.b2m_pc_open(srs.handle, self.pc, n, ptrs, lens, db, _lib.ptr(rands), _lib.ptr(shifted_rands), rands.shape[1],
                                 -1 if max_degree_bound is None else max_degree_bound, _lib.ptr(np.ascontiguousarray(point_limbs)),
                                 _lib.ptr(np.ascontiguousarray(challenge_limbs)), _lib.ptr(w), ctypes.byref(has), _lib.ptr(rv)))
        return w, (rv if has.value else None)

    # -- index -----------------------------------------------------------------------------------------
    def index(self, srs, r1cs):
        """[reference src/lib.rs:100-148] -> IndexProverKey (device resident); .vk_bytes is `index_vk` (ToBytes)."""
        L = _lib.lib()
        h = ctypes.c_void_p()
        a, b, c = r1cs.matrices()
        _lib.check(L.b2m_index_create(srs.handle, self.pc, r1cs.num_constraints, r1cs.num_variables, r1cs.num_instance,
                                      ctypes.byref(a), ctypes.byref(b), ctypes.byref(c), ctypes.byref(h)))
        return IndexProverKey(srs, h, r1cs, self.pc)

    # -- circom circuits (marlin_b200/circom.py) ---------------------------------------------------------
    def load_r1cs(self, path):
        """The matrices of a circom `.r1cs` file as the padded, squared R1CS `Marlin::index` takes (instance and witness None;
        enough for `index`, `IndexProverKey.save` and `verifier_key`).  Wires 1 .. nPubOut + nPubIn are the public inputs, in
        snarkjs `public.json` order; wire w goes to column w (w < 1 + nPubOut + nPubIn) or past the instance padding, as
        ark-circom and the indexer place it (r1cs.Shape), and circom constraint k is row k.  The constraint section is
        decoded on the GPU, every row in normal form (columns ascending, equal wires summed, zero sums dropped).  A bad term
        raises naming it, e.g. `constraints[12].B[3]: wire 4097 >= nWires 4096`."""
        from . import circom
        from . import r1cs as gr1cs
        L = _lib.lib()
        cid = self.curve_id
        f = circom.read_r1cs(path)
        circom.check_prime(path, "section 1 (header)", f.prime, cid)
        sh = gr1cs.Shape(f.ni0, f.n_wires - f.ni0, f.m)
        rps = circom.constraint_rows(f)
        nnz = [int(r[-1]) for r in rps]
        out_rp = [np.zeros(f.m + 1, dtype=np.uint64) for _ in range(3)]
        cols = [np.zeros(max(n, 1), dtype=np.uint64) for n in nnz]
        coeffs = [np.zeros((max(n, 1), 4), dtype=np.uint64) for n in nnz]
        arr = lambda xs: (ctypes.c_void_p * 3)(*[x.ctypes.data for x in xs])  # noqa: E731
        bm, bt, br = ctypes.c_int(0), ctypes.c_size_t(0), ctypes.c_int(0)
        data = f.constraints
        rc = L.b2m_circom_decode_constraints(self.ctx.handle, cid, data.ctypes.data if len(data) else None, len(data), f.m, arr(rps), f.n_wires,
                                             f.ni0, sh.shift, arr(out_rp), arr(cols), arr(coeffs), ctypes.byref(bm), ctypes.byref(bt),
                                             ctypes.byref(br))
        if rc == _lib.ERR_SERIALIZATION:
            j, t = bm.value, bt.value
            k = int(np.searchsorted(rps[j], np.uint64(t), side="right")) - 1
            i = t - int(rps[j][k])
            at = f"constraints[{k}].{circom.MATRICES[j]}[{i}]"
            if br.value == 1:
                off = circom.term_offset(rps, k, j, i)
                wire = int.from_bytes(bytes(data[off:off + 4]), "little")
                raise _lib.B2MError(rc, f"{at}: wire {wire} >= nWires {f.n_wires}")
            raise _lib.B2MError(rc, f"{at}: coefficient not below r")
        _lib.check(rc)
        mats = []
        for j in range(3):
            n = int(out_rp[j][-1])
            row_ptr = np.concatenate([out_rp[j], np.full(sh.pad_rows, n, dtype=np.uint64)])
            if n == 0:  # the placeholder `from_rows` emits for an empty matrix
                mats.append((row_ptr, np.zeros(1, dtype=np.uint64), np.zeros((1, 4), dtype=np.uint64)))
            else:
                mats.append((row_ptr, cols[j][:n], coeffs[j][:n]))
        out = gr1cs.R1CS(cid, sh.ni, mats[0], mats[1], mats[2], None, None, num_variables=sh.size)
        out.circom = f.info()
        return out

    def load_wtns(self, r1cs, path, check=True):
        """`r1cs` (from load_r1cs) with the assignment of a circom `.wtns` file: instance = wires 0 .. nPubOut + nPubIn
        padded with zeros, witness = the remaining wires then ones for the squaring.  Values are decoded and checked below r
        on the GPU; wire 0 must be one.  check=True runs `which_is_unsatisfied` and raises naming the lowest failing
        constraint, e.g. `constraint 1234 is not satisfied`."""
        from . import circom
        from . import r1cs as gr1cs
        info = r1cs.circom
        if info is None:
            raise ValueError("load_wtns takes an R1CS from load_r1cs")
        L = _lib.lib()
        cid = self.curve_id
        f = circom.read_wtns(path)
        circom.check_prime(path, "section 1 (header)", f.prime, cid)
        if f.n_witness != info.n_wires:
            raise ValueError(f"{path}: section 1 (header): nWitness = {f.n_witness}, the circuit has nWires = {info.n_wires}")
        vals = np.zeros((f.n_witness, 4), dtype=np.uint64)
        bi = ctypes.c_size_t(0)
        rc = L.b2m_fr_decode_ark(self.ctx.handle, cid, f.values.ctypes.data, f.n_witness, _lib.ptr(vals), ctypes.byref(bi))
        if rc == _lib.ERR_SERIALIZATION:
            raise _lib.B2MError(rc, f"witness[{bi.value}]: not below r")
        _lib.check(rc)
        one = _lib.ints_to_limbs([fields.fr_to_mont(cid, 1)], 4)[0]
        if not np.array_equal(vals[0], one):
            raise ValueError(f"{path}: witness[0] is {fields.fr_from_mont(cid, _lib.limbs_to_ints(vals[0])[0])}, wire 0 is the constant one")
        ni0 = 1 + info.n_pub_out + info.n_pub_in
        sh = gr1cs.Shape(ni0, info.n_wires - ni0, info.m_constraints)
        inst = np.concatenate([vals[:ni0], np.zeros((sh.shift, 4), dtype=np.uint64)])
        wit = np.concatenate([vals[ni0:], np.tile(one, (sh.pad_witness, 1))])
        out = gr1cs.R1CS(cid, sh.ni, r1cs.a, r1cs.b, r1cs.c, inst, wit)
        out.circom = info
        if check:
            bad = self.which_is_unsatisfied(out)
            if bad is not None:
                raise ValueError(f"{path}: constraint {bad} is not satisfied")
        return out

    def which_is_unsatisfied(self, r1cs):
        """ark-relations' `which_is_unsatisfied` on the GPU (b2m_r1cs_check): the lowest row r of the padded instance with
        <A_r, z> * <B_r, z> != <C_r, z>, or None when every row holds.  Circom constraint k is row k."""
        if r1cs.witness is None:
            raise ValueError("the instance has no assignment (load_wtns gives one)")
        a, b, c = r1cs.matrices()
        inst, wit = np.ascontiguousarray(r1cs.instance), np.ascontiguousarray(r1cs.witness)
        bad = ctypes.c_size_t(0)
        _lib.check(_lib.lib().b2m_r1cs_check(self.ctx.handle, self.curve_id, r1cs.num_constraints, r1cs.num_variables, r1cs.num_instance,
                                             ctypes.byref(a), ctypes.byref(b), ctypes.byref(c), _lib.ptr(inst),
                                             _lib.ptr(wit) if len(wit) else None, ctypes.byref(bad)))
        return None if bad.value == r1cs.num_constraints else bad.value

    # -- index key files (marlin_b200/keyfile.py) --------------------------------------------------------
    def _decode_g1(self, pts, field, compressed, names=int):
        """ark-serialize G1 bytes (n, size) -> affine limbs, validated on the GPU; an invalid point raises naming field[index]"""
        L = _lib.lib()
        pts = np.ascontiguousarray(pts, dtype=np.uint8)
        n = len(pts)
        out = np.zeros((n, 2 * _lib.LIMBS[self.curve_id][1]), dtype=np.uint64)
        if n == 0:
            return out
        bi, br = ctypes.c_size_t(0), ctypes.c_int(0)
        rc = L.b2m_g1_decode_ark(self.ctx.handle, self.curve_id, _lib.ptr(pts.reshape(-1)), n, int(compressed), _lib.ptr(out), ctypes.byref(bi),
                                 ctypes.byref(br))
        if rc == _lib.ERR_SERIALIZATION:
            raise _lib.B2MError(rc, f"{field}[{names(bi.value)}]: {_lib.POINT_REASONS.get(br.value, 'invalid point')}")
        _lib.check(rc)
        return out

    def _decode_g2(self, pts, field, compressed, names=int):
        """ark-serialize G2 bytes (n, size) -> uncompressed canonical bytes (n, 4 sizeof(Fq)), validated on the GPU"""
        from . import srsfile
        L = _lib.lib()
        pts = np.ascontiguousarray(pts, dtype=np.uint8)
        n = len(pts)
        out = np.zeros((n, 4 * srsfile.fq_bytes(self.curve_id)), dtype=np.uint8)
        if n == 0:
            return out
        bi, br = ctypes.c_size_t(0), ctypes.c_int(0)
        rc = L.b2m_g2_decode_ark(self.ctx.handle, self.curve_id, _lib.ptr(pts.reshape(-1)), n, int(compressed), _lib.ptr(out), ctypes.byref(bi),
                                 ctypes.byref(br))
        if rc == _lib.ERR_SERIALIZATION:
            at = "" if names is None else f"[{names(bi.value)}]"
            raise _lib.B2MError(rc, f"{field}{at}: {_lib.POINT_REASONS.get(br.value, 'invalid point')}")
        _lib.check(rc)
        return out

    def _decode_vk(self, vk, compressed):
        """Every point of a parsed `IndexVerifierKey`, decoded and validated on the GPU"""
        f = "index_vk.verifier_key"
        out = {"comms": self._decode_g1(vk["comms"], "index_vk.index_comms", compressed),
               "g": self._decode_g1(vk["g"].reshape(1, -1), f + ".g", compressed)[0],
               "gamma_g": self._decode_g1(vk["gamma_g"].reshape(1, -1), f + ".gamma_g", compressed)[0]}
        out["h"] = self._decode_g2(vk["h"].reshape(1, -1), f + ".h", compressed, None)[0]
        out["beta_h"] = self._decode_g2(vk["beta_h"].reshape(1, -1), f + ".beta_h", compressed, None)[0]
        keys = vk["bounds"]
        if self.pc == _lib.PC_MARLIN_KZG10:
            out["bound_points"] = self._decode_g1(vk["bound_points"], f + ".degree_bounds_and_shift_powers", compressed)
        else:
            out["bound_points"] = self._decode_g2(vk["bound_points"], f + ".degree_bounds_and_neg_powers_of_h", compressed)
        return out

    def _make_vk(self, vk, pts):
        nv, nc, nnz, _ = vk["info"]
        L = _lib.lib()
        b = np.asarray(vk["bounds"], dtype=np.uint64)
        handle = ctypes.c_void_p()
        _lib.check(L.b2m_vk_create(self.ctx.handle, self.curve_id, self.pc, nc, nv, nnz, _lib.ptr(np.ascontiguousarray(pts["comms"])),
                                   _lib.ptr(np.ascontiguousarray(pts["g"])), _lib.ptr(np.ascontiguousarray(pts["gamma_g"])),
                                   _lib.ptr(np.ascontiguousarray(pts["h"])), _lib.ptr(np.ascontiguousarray(pts["beta_h"])), len(b),
                                   _lib.ptr(b) if len(b) else None, _lib.ptr(np.ascontiguousarray(pts["bound_points"])) if len(b) else None,
                                   ctypes.byref(handle)))
        return VerifierKey(self.ctx, handle, self.curve_id, self.pc)

    def load_verifier_key(self, path, compressed=True):
        """A `VerifierKey` from a raw arkworks `IndexVerifierKey` file alone (`serialize` when compressed, else
        `serialize_uncompressed`; marlin_b200/keyfile.py): no SRS and no index are needed.  Every point is decoded and validated
        on the GPU; an invalid one raises B2MError (B2M_ERR_SERIALIZATION) naming its field and index."""
        from . import keyfile
        vk = keyfile.read_verifier_key(path, self.curve_id, self.pc, compressed)
        return self._make_vk(vk, self._decode_vk(vk, compressed))

    def load_index(self, srs, path, compressed=True, check_commitments=False):
        """An `IndexProverKey` from a raw arkworks key file, on `srs`, without re-indexing: no arithmetization and no commitment
        MSM run.  Every point is decoded and validated on the GPU (b2m_g1_decode_ark / b2m_g2_decode_ark), every field element
        is checked to be below r on the GPU, and the NTT over K of each index polynomial must equal its evaluations
        (b2m_index_load).  The committer key and the verifier key's G1 part must be those `PC::trim` makes from `srs` for the
        bounds {|H| - 2, |K| - 2}.  check_commitments=True also recomputes the six index commitments.  A failure raises
        B2MError (B2M_ERR_SERIALIZATION) or ValueError naming the field and the first bad index, e.g.
        `index.joint_arith.evals_on_K.val_b[70001]: not below the field modulus`."""
        from . import keyfile
        L = _lib.lib()
        cid, marlin = self.curve_id, self.pc == _lib.PC_MARLIN_KZG10
        d = keyfile.read_prover_key(path, cid, self.pc, compressed)
        vk, idx, ck = d["vk"], d["index"], d["ck"]
        nv, nc, nnz, ni = vk["info"]
        pts = self._decode_vk(vk, compressed)
        ckn = "committer_key." + ("powers" if marlin else "powers_of_g")
        shn = "committer_key." + ("shifted_powers" if marlin else "shifted_powers_of_g")
        ck_powers = self._decode_g1(ck["powers"], ckn, compressed)
        ck_shifted = self._decode_g1(ck["shifted"], shn, compressed) if ck["shifted"] is not None else None
        ck_gamma = self._decode_g1(ck["gamma"], "committer_key.powers_of_gamma_g", compressed)
        ck_sgamma = {}
        for k, v in (ck.get("shifted_gamma") or {}).items():
            ck_sgamma[k] = self._decode_g1(v, f"committer_key.shifted_powers_of_gamma_g[{k}]", compressed)

        # the committer key and the verifier key's G1 part against the SRS they are loaded onto
        D = srs.max_degree
        bounds = index_degree_bounds(nc, nnz)
        md = max_degree(nc, nv, nnz)
        powers = np.asarray(srs.powers_limbs)

        def same(field, got, want, offset=0):
            got, want = np.asarray(got).reshape(len(got), -1), np.asarray(want).reshape(len(want), -1)
            if len(got) != len(want):
                raise ValueError(f"{path}: {field}: {len(got)} points, the SRS gives {len(want)}")
            diff = np.flatnonzero(np.any(got != want, axis=1))
            if len(diff):
                raise ValueError(f"{path}: {field}[{int(diff[0]) + offset}]: differs from the SRS")

        def equal(field, got, want):
            if got != want:
                raise ValueError(f"{path}: {field} is {got}, expected {want}")
        equal("committer_key.max_degree", ck["max_degree"], D)
        equal("committer_key.enforced_degree_bounds", ck["bounds"], bounds)
        equal("index_vk.verifier_key.max_degree", vk["max_degree"], D)
        equal("index_vk.verifier_key.supported_degree", vk["supported_degree"], md)
        equal("index_vk.verifier_key degree bounds", [int(b) for b in vk["bounds"]], bounds)
        if md > D:
            raise ValueError(f"{path}: the index needs max degree {md}, the SRS has {D}")
        same(ckn, ck_powers, powers[:md + 1])
        if ck_shifted is None:
            raise ValueError(f"{path}: {shn} is None, the index enforces degree bounds {bounds}")
        same(shn, ck_shifted, powers[D - bounds[-1]:])
        same("committer_key.powers_of_gamma_g", ck_gamma, srs_gamma_powers(srs, [0, 1, 2]))
        if not marlin:
            equal("committer_key.shifted_powers_of_gamma_g keys", sorted(ck_sgamma), bounds)
            for k in bounds:
                same(f"committer_key.shifted_powers_of_gamma_g[{k}]", ck_sgamma[k], srs_gamma_powers(srs, [D - k + i for i in range(3) if D - k + i < D + 2]))
        same("index_vk.verifier_key.g", pts["g"].reshape(1, -1), powers[:1])
        same("index_vk.verifier_key.gamma_g", pts["gamma_g"].reshape(1, -1), srs_gamma_powers(srs, [0]))
        if marlin:
            same("index_vk.verifier_key.degree_bounds_and_shift_powers", pts["bound_points"], np.stack([powers[D - b] for b in bounds]))

        # the index: sizes and domains, matrices (coefficients decoded on the GPU), then the twelve vectors
        K = _p2(nnz)
        dom = domain_bytes(cid, K)
        for i, name in enumerate(keyfile.POLY_LABELS):
            ename = keyfile.EVAL_NAMES[keyfile.EVAL_OF_POLY[i]]
            if len(idx["evals"][i]) != K:
                raise ValueError(f"{path}: index.joint_arith.evals_on_K.{ename}.evals has {len(idx['evals'][i])} elements, |K| = {K}")
            if idx["domains"][i] != dom:
                raise ValueError(f"{path}: index.joint_arith.evals_on_K.{ename}.domain is not the domain of size {K}")
            if len(idx["coeffs"][i]) > K:
                raise ValueError(f"{path}: index.joint_arith.{name}.polynomial has {len(idx['coeffs'][i])} coefficients, |K| = {K}")
        mats, keep = [], []
        for m, (row_ptr, col, coeff) in zip(keyfile.MATRICES, idx["matrices"]):
            if len(row_ptr) != nc + 1:
                raise ValueError(f"{path}: index.{m} has {len(row_ptr) - 1} rows, num_constraints is {nc}")
            ne = len(col)
            limbs = np.zeros((max(ne, 1), 4), dtype=np.uint64)
            bi = ctypes.c_size_t(0)
            rc = L.b2m_fr_decode_ark(self.ctx.handle, cid, _lib.ptr(np.ascontiguousarray(coeff)), ne, _lib.ptr(limbs), ctypes.byref(bi))
            if rc == _lib.ERR_SERIALIZATION:
                r = int(np.searchsorted(row_ptr, np.uint64(bi.value), side="right")) - 1
                raise _lib.B2MError(rc, f"index.{m}[{r}][{bi.value - int(row_ptr[r])}].0: not below the field modulus")
            _lib.check(rc)
            col = np.ascontiguousarray(col, dtype=np.uint64) if ne else np.zeros(1, dtype=np.uint64)
            row_ptr = np.ascontiguousarray(row_ptr, dtype=np.uint64)
            keep += [row_ptr, col, limbs]
            mt = _lib.Matrix()
            mt.row_ptr, mt.col, mt.coeff = row_ptr.ctypes.data, col.ctypes.data, limbs.ctypes.data
            mats.append(mt)
        vecs = [np.ascontiguousarray(v) for v in idx["coeffs"] + idx["evals"]]
        vptr = (ctypes.c_void_p * 12)(*[v.ctypes.data if len(v) else None for v in vecs])
        vlen = (ctypes.c_size_t * 12)(*[len(v) for v in vecs])
        h = ctypes.c_void_p()
        bv, bi, br = ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_int(0)
        rc = L.b2m_index_load(srs.handle, self.pc, nc, nv, ni, nnz, ctypes.byref(mats[0]), ctypes.byref(mats[1]), ctypes.byref(mats[2]), vptr, vlen,
                              _lib.ptr(np.ascontiguousarray(pts["comms"])), int(check_commitments), ctypes.byref(bv), ctypes.byref(bi),
                              ctypes.byref(br), ctypes.byref(h))
        if rc == _lib.ERR_SERIALIZATION and br.value:
            v, i = bv.value, bi.value
            label = keyfile.POLY_LABELS[v % 6]
            ev = f"index.joint_arith.evals_on_K.{keyfile.EVAL_NAMES[keyfile.EVAL_OF_POLY[v % 6]]}"
            field = f"index.joint_arith.{label}.polynomial" if v < 6 else ev
            msg = {1: f"{field}[{i}]: not below the field modulus",
                   2: f"{ev}[{i}]: not the FFT over K of index.joint_arith.{label}.polynomial",
                   3: f"index_vk.index_comms[{v}]: not the commitment to index.joint_arith.{label}"}[br.value]
            raise _lib.B2MError(rc, msg)
        _lib.check(rc)
        pk = IndexProverKey(srs, h, types.SimpleNamespace(num_constraints=nc, num_variables=nv, num_instance=ni), self.pc)
        neg = {}
        if not marlin:
            neg = {D - int(b): pts["bound_points"][k].tobytes() for k, b in enumerate(vk["bounds"])}
        pk.file_g2 = (pts["h"].tobytes(), pts["beta_h"].tobytes(), neg)
        return pk

    # -- prove -----------------------------------------------------------------------------------------
    def prove(self, index_pk, r1cs, zk_rng):
        """[reference src/lib.rs:151-311] -> `CanonicalSerialize` bytes of `Proof<F, PC>`.
        r1cs = None proves the instance previously copied to the GPU with `stage`."""
        L = _lib.lib()
        buf = (ctypes.c_uint8 * 2048)()
        n = ctypes.c_size_t(0)
        if r1cs is None:
            _lib.check(L.b2m_prove(index_pk.handle, None, 0, None, 0, ctypes.byref(zk_rng.c), buf, 2048, ctypes.byref(n)))
        else:
            inst = np.ascontiguousarray(r1cs.instance)
            wit = np.ascontiguousarray(r1cs.witness)
            _lib.check(L.b2m_prove(index_pk.handle, _lib.ptr(inst), len(inst), _lib.ptr(wit), len(wit), ctypes.byref(zk_rng.c), buf,
                                   2048, ctypes.byref(n)))
        return bytes(buf[:n.value])

    # -- verify ----------------------------------------------------------------------------------------
    def verifier_key(self, index_pk, srs):
        """The verifier key of an index: index_info, the six index commitments, g and gamma g, and the verifier's shift
        material for the bounds |H| - 2 and |K| - 2 -- MarlinKZG10: powers_of_g[D - d]; SonicKZG10: beta^-(D - d) h -- with
        h, beta h from the SRS's trapdoor or from the file it was loaded from (as `UniversalSRS.save` takes them)."""
        L = _lib.lib()
        cid = self.curve_id
        nv, nc, nnz = struct.unpack_from("<QQQ", index_pk.vk_bytes, 0)
        bounds = index_degree_bounds(nc, nnz)
        D = srs.max_degree
        h, beta_h, neg = g2_half(srs, bounds)
        powers = np.ascontiguousarray(srs.powers_limbs)
        if self.pc == _lib.PC_MARLIN_KZG10:
            bound_points = np.ascontiguousarray(np.stack([powers[D - d] for d in bounds]))
        else:
            missing = [d for d in bounds if D - d not in neg]
            if missing:
                raise ValueError(f"the SRS holds no neg_powers_of_h for the degree bounds {missing}")
            bound_points = np.frombuffer(b"".join(neg[D - d] for d in bounds), dtype=np.uint8).copy()
        gamma_g = np.ascontiguousarray(srs.gamma_limbs[list(srs.gamma_indices).index(0)])
        hb = np.frombuffer(h, dtype=np.uint8).copy()
        bhb = np.frombuffer(beta_h, dtype=np.uint8).copy()
        b = np.asarray(bounds, dtype=np.uint64)
        handle = ctypes.c_void_p()
        _lib.check(L.b2m_vk_create(self.ctx.handle, cid, self.pc, nc, nv, nnz, _lib.ptr(np.ascontiguousarray(index_pk.index_comms)),
                                   _lib.ptr(np.ascontiguousarray(powers[0])), _lib.ptr(gamma_g), _lib.ptr(hb), _lib.ptr(bhb), len(b),
                                   _lib.ptr(b), _lib.ptr(bound_points), ctypes.byref(handle)))
        return VerifierKey(self.ctx, handle, cid, self.pc)

    def verify_batch(self, vk, public_inputs, proofs, rng):
        """`Marlin::verify` [reference src/lib.rs:315-433] for many proofs under one key.  public_inputs[i]: the field
        elements (Python ints) of proof i's public input, without the leading one; rng: the ZkRng / CallbackRng the batch
        randomisers are drawn from (unpredictable to the prover).  Returns True (accepted) / False (rejected) / None
        (malformed bytes) per proof."""
        n = len(proofs)
        if len(public_inputs) != n:
            raise ValueError("one public input per proof")
        args, verdicts, _keep = _proof_args([self.curve_id] * n, public_inputs, proofs)
        _lib.check(_lib.lib().b2m_verify_batch(vk.handle, n, *args, ctypes.byref(rng.c) if rng is not None else None, verdicts))
        return [{1: True, 0: False}.get(verdicts[i]) for i in range(n)]

    def verify(self, vk, public_input, proof_bytes, rng):
        """`Marlin::verify` of one proof -> bool (malformed bytes are False)."""
        return self.verify_batch(vk, [public_input], [proof_bytes], rng)[0] is True

    # -- PC::check_combinations (Level 1) --------------------------------------------------------------
    def pc_verifier_key(self, srs, enforced_degree_bounds=()):
        """`PC::VerifierKey` after `PC::trim`: g, gamma g, h, beta h and per enforced bound d MarlinKZG10's powers_of_g[D - d] or
        SonicKZG10's beta^-(D - d) h, with the G2 half from the SRS's trapdoor or its source file (as `verifier_key`)."""
        cid = self.curve_id
        bounds = sorted(set(int(d) for d in enforced_degree_bounds))
        D = srs.max_degree
        h, beta_h, neg = g2_half(srs, bounds)
        if self.pc == _lib.PC_MARLIN_KZG10:
            powers = np.ascontiguousarray(srs.powers_limbs)
            bound_points = np.ascontiguousarray(np.stack([powers[D - d] for d in bounds])) if bounds else None
        else:
            missing = [d for d in bounds if D - d not in neg]
            if missing:
                raise ValueError(f"the SRS holds no neg_powers_of_h for the degree bounds {missing}")
            bound_points = np.frombuffer(b"".join(neg[D - d] for d in bounds), dtype=np.uint8).copy() if bounds else None
        g = np.ascontiguousarray(srs.powers_limbs[0])
        gamma_g = np.ascontiguousarray(srs.gamma_limbs[list(srs.gamma_indices).index(0)])
        b = np.asarray(bounds, dtype=np.uint64)
        handle = ctypes.c_void_p()
        _lib.check(_lib.lib().b2m_pc_vk_create(self.ctx.handle, cid, self.pc, D, _lib.ptr(g), _lib.ptr(gamma_g),
                                                _lib.ptr(np.frombuffer(h, dtype=np.uint8).copy()),
                                                _lib.ptr(np.frombuffer(beta_h, dtype=np.uint8).copy()), len(b), _lib.ptr(b) if bounds else None,
                                                _lib.ptr(bound_points), ctypes.byref(handle)))
        return PcVerifierKey(self.ctx, handle, cid, self.pc, bounds)

    def check_combinations(self, vk, sets, rng):
        """`PC::check_combinations` for many independent OpeningSets in one GPU batch (b2m_pc_check_combinations).  rng: the
        ZkRng / CallbackRng the batch randomisers are drawn from (unpredictable to the prover).  Returns True (accepted) / False
        (rejected) / None (malformed: a point that does not decode, an evaluation or random_v not below r, a bounded MarlinKZG10
        commitment without its shifted commitment) per set, as `verify_batch`."""
        return self._pc_check(vk, sets, rng, identity=False)

    def batch_check(self, vk, sets, rng):
        """`PC::batch_check` for many OpeningSets: check_combinations with one LC per commitment, coefficient one, labelled as
        the commitment (upstream orders both by label, so the challenges are the same).  Each set's `lcs` must be None."""
        return self._pc_check(vk, sets, rng, identity=True)

    def check(self, vk, opening_set, rng):
        """`PC::check` of one OpeningSet at a single point: `batch_check` of that set -> True / False / None."""
        if len({q[1][0] for q in opening_set.query_set}) != 1:
            raise ValueError("check opens at a single point")
        return self.batch_check(vk, [opening_set], rng)[0]

    def _pc_check(self, vk, sets, rng, identity):
        arrays = pc_check_arrays(vk.curve_id, sets, identity, lambda limbs: g1_to_bytes(self.ctx, vk.curve_id, limbs, True))
        n = len(sets)
        verdicts = np.zeros(max(n, 1), dtype=np.int32)
        _lib.check(_lib.lib().b2m_pc_check_combinations(vk.handle, n, *[_lib.ptr(a) for a in arrays],
                                                         ctypes.byref(rng.c) if rng is not None else None, _lib.ptr(verdicts)))
        return [{1: True, 0: False}.get(int(verdicts[i])) for i in range(n)]

    def stage(self, index_pk, r1cs):
        """Copy (x, w) into HBM ahead of time (device-resident timing in bench.py)."""
        inst = np.ascontiguousarray(r1cs.instance)
        wit = np.ascontiguousarray(r1cs.witness)
        _lib.check(_lib.lib().b2m_index_stage(index_pk.handle, _lib.ptr(inst), len(inst), _lib.ptr(wit), len(wit)))
