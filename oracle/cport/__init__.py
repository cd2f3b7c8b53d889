"""ctypes wrapper of oracle/cport/libcport.so -- the C (OpenMP) restatement of the reference's CPU
algorithms (ark-ec Pippenger MSM, ark-poly radix-2 FFT).  TEST INFRASTRUCTURE: tests/ use it as a
fast checker; bench.py times it as the CPU baseline ("kind": "port")."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PATH = os.path.join(_HERE, "libcport.so")
_lib = None
CURVE_ID = {"bls12_381": 0, "bn254": 1}


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            subprocess.check_call(["make", "-C", _HERE])
        L = ctypes.CDLL(_PATH)
        vp, sz, ci = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
        L.cport_msm.argtypes = [ci, vp, vp, sz, vp, ci]
        L.cport_fft.argtypes = [ci, vp, ctypes.c_uint, ci, ci]
        L.cport_coset_fft.argtypes = [ci, vp, ctypes.c_uint, ci, ci]
        L.cport_gen_bases.argtypes = [ci, vp, sz, vp]
        L.cport_max_threads.restype = ci
        L.cport_set_skip_index_commit.argtypes = [ci]
        L.cport_set_skip_index_commit.restype = None
        u8p = ctypes.c_void_p
        L.cport_index_create.argtypes = [ci, ci, ci, vp, sz, vp, vp, sz, sz, sz, sz] + [vp] * 9 + [ctypes.POINTER(ctypes.c_void_p)]
        L.cport_index_free.argtypes = [vp]
        L.cport_index_free.restype = None
        L.cport_index_vk_bytes.argtypes = [vp, u8p, sz]
        L.cport_index_vk_bytes.restype = sz
        L.cport_prove.argtypes = [vp, vp, sz, vp, sz, ci, u8p, ctypes.POINTER(ctypes.c_uint64), u8p, sz, ctypes.POINTER(sz),
                                  ctypes.POINTER(ctypes.c_double)]
        _lib = L
    return _lib


def usable_cpus():
    """Threads the baseline may really use: the affinity mask capped by the cgroup CPU quota (a container that
    sees 128 cores but owns 8 would otherwise be timed while oversubscribed 16x)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if quota != "max":
            n = max(1, min(n, int(int(quota) / int(period))))
    except Exception:
        try:
            quota = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            period = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if quota > 0:
                n = max(1, min(n, quota // period))
        except Exception:
            pass
    return max(1, n)


_best_threads = None


def best_threads():
    """Thread count that actually runs fastest on this host (probes 2^16-point FFTs): guards the baseline
    against containers that expose more cores than they may use."""
    global _best_threads
    if _best_threads is None:
        import time
        os.environ.setdefault("OMP_WAIT_POLICY", "passive")
        cap = min(usable_cpus(), lib().cport_max_threads())
        rng = np.random.default_rng(0)
        data = rng.integers(0, 1 << 62, size=(1 << 16, 4), dtype=np.uint64)
        best, best_t = 1, None
        t = cap
        cands = []
        while t >= 1:
            cands.append(t)
            t //= 2
        for t in cands:
            dt = None
            for _ in range(3):  # first run warms the OpenMP pool for this team size
                buf = data.copy()
                t0 = time.perf_counter()
                fft("bls12_381", buf, threads=t)
                d = time.perf_counter() - t0
                dt = d if dt is None else min(dt, d)
            if best_t is None or dt < 0.95 * best_t:  # prefer more threads unless fewer are clearly faster
                best, best_t = t, dt
        _best_threads = best
    return _best_threads


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def msm(curve_name, bases_limbs, scalars_limbs, threads=0):
    """bases: (n, 2*LQ) uint64 Montgomery affine; scalars: (n, 4) uint64 canonical -> (2*LQ,) uint64 affine."""
    bases_limbs = np.ascontiguousarray(bases_limbs, dtype=np.uint64)
    scalars_limbs = np.ascontiguousarray(scalars_limbs, dtype=np.uint64)
    out = np.zeros(bases_limbs.shape[1], dtype=np.uint64)
    lib().cport_msm(CURVE_ID[curve_name], _ptr(bases_limbs), _ptr(scalars_limbs), len(scalars_limbs), _ptr(out), threads)
    return out


def fft(curve_name, data_limbs, inverse=False, threads=0):
    """in-place radix-2 FFT of (2^k, 4) uint64 Montgomery Fr limbs."""
    n = len(data_limbs)
    log_n = n.bit_length() - 1
    assert 1 << log_n == n and data_limbs.flags["C_CONTIGUOUS"]
    lib().cport_fft(CURVE_ID[curve_name], _ptr(data_limbs), log_n, 1 if inverse else 0, threads)
    return data_limbs


def coset_fft(curve_name, data_limbs, inverse=False, threads=0):
    """in-place coset FFT (ark-poly `coset_fft` / `coset_ifft`, offset = the field's multiplicative generator) of (2^k, 4)
    uint64 Montgomery Fr limbs."""
    n = len(data_limbs)
    log_n = n.bit_length() - 1
    assert 1 << log_n == n and data_limbs.flags["C_CONTIGUOUS"] and data_limbs.dtype == np.uint64
    lib().cport_coset_fft(CURVE_ID[curve_name], _ptr(data_limbs), log_n, 1 if inverse else 0, threads)
    return data_limbs


class CpuProver:
    """The C++ restatement of `Marlin::index` + `Marlin::prove` (prover.cpp) behind the same inputs as the
    product's C ABI: SRS points and CSR matrices as limb arrays, assignments as Montgomery limbs."""

    def __init__(self, curve_name, pc, powers_limbs, gamma_limbs, gamma_indices, num_constraints, num_variables, num_instance, a, b, c,
                 threads=0):
        L = lib()
        self.h = ctypes.c_void_p()
        self.keep = [np.ascontiguousarray(x, dtype=np.uint64) for x in (powers_limbs, gamma_limbs, np.asarray(gamma_indices, dtype=np.uint64))]
        mats = []
        for m in (a, b, c):
            mats += [np.ascontiguousarray(x, dtype=np.uint64) for x in m]
        self.keep += mats
        nthreads = threads or min(usable_cpus(), L.cport_max_threads())
        rc = L.cport_index_create(CURVE_ID[curve_name], 1 if pc == "sonic_kzg10" else 0, nthreads, _ptr(self.keep[0]), len(self.keep[0]),
                                  _ptr(self.keep[1]), _ptr(self.keep[2]), len(self.keep[2]), num_constraints, num_variables, num_instance,
                                  *[_ptr(x) for x in mats], ctypes.byref(self.h))
        if rc:
            raise RuntimeError(f"cport_index_create failed with code {rc}")
        n = L.cport_index_vk_bytes(self.h, None, 0)
        buf = (ctypes.c_uint8 * n)()
        L.cport_index_vk_bytes(self.h, buf, n)
        self.vk_bytes = bytes(buf)
        self.threads = nthreads

    def prove(self, instance_limbs, witness_limbs, seed, rounds=12, word_pos=0):
        """-> (proof bytes, new word_pos, seconds)"""
        L = lib()
        inst = np.ascontiguousarray(instance_limbs, dtype=np.uint64)
        wit = np.ascontiguousarray(witness_limbs, dtype=np.uint64)
        key = (ctypes.c_uint8 * 32)(*bytes(seed))
        pos = ctypes.c_uint64(word_pos)
        out = (ctypes.c_uint8 * 2048)()
        n = ctypes.c_size_t(0)
        secs = ctypes.c_double(0)
        rc = L.cport_prove(self.h, _ptr(inst), len(inst), _ptr(wit), len(wit), rounds, key, ctypes.byref(pos), out, 2048, ctypes.byref(n),
                           ctypes.byref(secs))
        if rc:
            raise RuntimeError(f"cport_prove failed with code {rc}")
        return bytes(out[:n.value]), int(pos.value), secs.value

    def close(self):
        if self.h:
            lib().cport_index_free(self.h)
            self.h = None


def cpu_model():
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name"):
                return line.split(":", 1)[1].strip()
    except Exception:
        pass
    return "unknown"


def prover_baseline(curve_name, pc, log_n, threads=0, repeats=1, time_budget_s=None, skip_index_commit=True):
    """CPU baseline for bench.py: the C++ restatement of the reference prover (prover.cpp) timed on `Marlin::prove` of the
    reference bench's DummyCircuit with 2^log_n constraints (index and SRS excluded, like benches/bench.rs:79-107).
    Runs up to `repeats` proves, stopping early once `time_budget_s` (set-up included) would be exceeded; at least one.
    The SRS used for timing is a set of distinct curve points ((i + 1) * G), not powers of a trapdoor, and (by default) the
    six index commitments -- set-up work outside the timed region -- are skipped: the work of `prove` is identical, the
    proof is not meant to verify.  The OpenMP team size is set explicitly (usable_cpus()), so a launcher's
    OMP_NUM_THREADS=1 (torchrun) cannot turn the baseline single-threaded."""
    import time
    from marlin_b200 import _lib as plib, fields, r1cs as gr1cs  # host-side marshalling helpers only (no GPU code runs)
    t_start = time.time()
    L = lib()
    L.cport_set_skip_index_commit(1 if skip_index_commit else 0)
    cid = CURVE_ID[curve_name]
    n = 1 << log_n
    D = 4 * n - 1
    lq = plib.LIMBS[cid][1]
    g = fields.G1_GENERATOR[cid]
    g_l = plib.ints_to_limbs([fields.fq_to_mont(cid, g[0]), fields.fq_to_mont(cid, g[1])], lq).reshape(1, 2 * lq)
    powers = np.zeros((D + 1, 2 * lq), dtype=np.uint64)
    L.cport_gen_bases(cid, _ptr(g_l), D + 1, _ptr(powers))
    gidx = sorted({0, 1, 2} | {D - d + i for d in (n - 2, 4 * n - 2) for i in range(3) if D - d + i <= D})
    gam = np.ascontiguousarray(powers[gidx])
    circ = gr1cs.dummy_circuit(cid, 0x1234567890abcdef, 0xfedcba0987654321, 10, n)
    nthreads = threads or min(usable_cpus(), L.cport_max_threads())
    try:
        cp = CpuProver(curve_name, pc, powers, gam, gidx, circ.num_constraints, circ.num_variables, circ.num_instance, circ.a, circ.b, circ.c,
                       nthreads)
    finally:
        L.cport_set_skip_index_commit(0)
    setup_s = time.time() - t_start
    try:
        secs = []
        pos = 0
        for _ in range(max(1, repeats)):
            if secs and time_budget_s is not None and (time.time() - t_start) + max(secs) > time_budget_s:
                break
            _, pos, s = cp.prove(circ.instance, circ.witness, bytes(range(32)), 12, pos)
            secs.append(s)
        mean = sum(secs) / len(secs)
        return {"value": n / mean, "unit": "constraints/s", "cores": cp.threads, "kind": "port", "cpu": cpu_model(),
                "sample": (f"C++/OpenMP restatement of the reference prover (oracle/cport/prover.cpp: ark-ec Pippenger with one task per "
                           f"window, radix-2 FFTs, the reference's round structure): {len(secs)} full Marlin::prove ({pc}, {curve_name}) of "
                           f"DummyCircuit 2^{log_n}, mean {mean:.2f} s on {cp.threads} threads; set-up (SRS points, index) {setup_s:.0f} s "
                           f"outside the timed region"),
                "seconds": mean, "seconds_per_step": secs, "steps_run": len(secs), "log_n": log_n, "setup_s": setup_s}
    finally:
        cp.close()
