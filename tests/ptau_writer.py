"""Test helper: snarkjs Powers-of-Tau (.ptau) files from the Python oracle, for chosen tau, alpha, beta, at small powers.

`sections(...)` returns the file as a list of [id, bytearray] (sections 1-7, optionally the prepared Lagrange sections
12-15) and `pack(...)` frames them, so a test can corrupt a point, a size, an id or a header field before writing.  Points are
in snarkjs's "LEM" form: every Fq (Fq2: c0 then c1) little-endian Montgomery with R = 2^(64 * limbs), infinity all-zero
[U snarkjs].  Not product code: the product only reads such files (marlin_b200/ptau.py)."""
import struct

import numpy as np

from oracle import ec

import ark_srs_oracle as ao


def _limbs64(curve):
    return curve.fq.nbytes // 8


def fq_lem(curve, v):
    n8 = curve.fq.nbytes
    return (v * (1 << (64 * _limbs64(curve))) % curve.fq.p).to_bytes(n8, "little")


def g1_lem(curve, P):
    if P is None:
        return bytes(2 * curve.fq.nbytes)
    return fq_lem(curve, P[0]) + fq_lem(curve, P[1])


def g2_lem(curve, Q):
    if Q is None:
        return bytes(4 * curve.fq.nbytes)
    return b"".join(fq_lem(curve, v) for v in (Q[0][0], Q[0][1], Q[1][0], Q[1][1]))


def header(curve, power, ceremony_power=None, q=None, n8=None):
    n8 = curve.fq.nbytes if n8 is None else n8
    q = curve.fq.p if q is None else q
    return struct.pack("<I", n8) + q.to_bytes(n8, "little") + struct.pack("<II", power, power if ceremony_power is None else ceremony_power)


def powers(curve, n, tau, base, add, smul):
    """[base, tau base, tau^2 base, ...] (n points)"""
    out, P = [], base
    for _ in range(n):
        out.append(P)
        P = smul(tau, P)
    return out


def sections(curve, power, tau, alpha, beta, prepared=False):
    """[[id, bytearray], ...] of a .ptau file whose secrets are (tau, alpha, beta), G and H the standard generators"""
    r = curve.fr.p
    g2 = ao.G2(curve)
    g1mul = lambda k, P: ec.scalar_mul(curve, k % r, P)  # noqa: E731
    g2mul = lambda k, Q: g2.smul(k % r, Q)  # noqa: E731
    n1, n2 = 2 ** (power + 1) - 1, 2 ** power
    tau_g1 = powers(curve, n1, tau, curve.g, None, g1mul)
    tau_g2 = powers(curve, n2, tau, g2.gen, None, g2mul)
    alpha_g1 = [g1mul(alpha, P) for P in tau_g1[:n2]]
    beta_g1 = [g1mul(beta, P) for P in tau_g1[:n2]]
    out = [[1, bytearray(header(curve, power))],
           [2, bytearray(b"".join(g1_lem(curve, P) for P in tau_g1))],
           [3, bytearray(b"".join(g2_lem(curve, Q) for Q in tau_g2))],
           [4, bytearray(b"".join(g1_lem(curve, P) for P in alpha_g1))],
           [5, bytearray(b"".join(g1_lem(curve, P) for P in beta_g1))],
           [6, bytearray(g2_lem(curve, g2mul(beta, g2.gen)))],
           [7, bytearray(struct.pack("<I", 0))]]  # no contribution records
    if prepared:  # the Lagrange sections' contents are never read: any bytes of a plausible size do
        out += [[12, bytearray(b"\x11" * (2 * curve.fq.nbytes * 4))], [13, bytearray(b"\x22" * (4 * curve.fq.nbytes * 4))],
                [14, bytearray(b"\x33" * (2 * curve.fq.nbytes * 4))], [15, bytearray(b"\x44" * (2 * curve.fq.nbytes * 4))]]
    return out


def pack(secs, magic=b"ptau", version=1, sizes=None):
    """frame the sections; sizes: {position in secs: declared size} to write a size that disagrees with the data"""
    sizes = sizes or {}
    out = [magic, struct.pack("<II", version, len(secs))]
    for k, (sid, data) in enumerate(secs):
        out += [struct.pack("<IQ", sid, sizes.get(k, len(data))), bytes(data)]
    return b"".join(out)


def set_point(secs, sid, i, blob):
    """overwrite point i of section sid"""
    data = next(d for s, d in secs if s == sid)
    pb = len(blob)
    data[i * pb:(i + 1) * pb] = blob


def write(path, secs, **kw):
    with open(path, "wb") as f:
        f.write(pack(secs, **kw))
    return path


def write_gpu_prefix(ctx, cid, path, power, D, tau, alpha):
    """a power-`power` file (curve id cid) whose tauG1[0..=D] (G the generator) and alphaTauG1[0..2] are computed on the GPU
    and tauG2[0..1] on the host; every other byte is a file hole, so files of the sizes users run stay cheap to write"""
    from marlin_b200 import _lib, fields, srsfile
    L = _lib.lib()
    lq = _lib.LIMBS[cid][1]
    n8 = 8 * lq
    q = fields.FQ_MODULUS[cid]
    gx, gy = fields.G1_GENERATOR[cid]
    g_l = _lib.ints_to_limbs([fields.fq_to_mont(cid, gx), fields.fq_to_mont(cid, gy)], lq).reshape(1, 2 * lq)
    tau_pts = np.zeros((D + 1, 2 * lq), dtype=np.uint64)
    _lib.check(L.b2m_g1_powers(ctx.handle, cid, _lib.ptr(g_l), _lib.ptr(_lib.ints_to_limbs([tau], 4)), D + 1, _lib.ptr(tau_pts)))
    alpha_pts = np.zeros((3, 2 * lq), dtype=np.uint64)
    a_l = _lib.ints_to_limbs([alpha * pow(tau, i, fields.FR_MODULUS[cid]) % fields.FR_MODULUS[cid] for i in range(3)], 4)
    _lib.check(L.b2m_fixed_base_msm(ctx.handle, cid, _lib.ptr(g_l), _lib.ptr(a_l), 3, _lib.ptr(alpha_pts)))
    h, beta_h, _ = srsfile.g2_setup(cid, fields.FR_MODULUS[cid], tau, D, ())
    g2 = b""
    for blob in (h, beta_h):
        for k in range(4):
            g2 += fields.fq_to_mont(cid, int.from_bytes(blob[k * n8:(k + 1) * n8], "little")).to_bytes(n8, "little")
    hdr = struct.pack("<I", n8) + q.to_bytes(n8, "little") + struct.pack("<II", power, power)
    sizes = [(1, len(hdr)), (2, (2 ** (power + 1) - 1) * 2 * n8), (3, 2 ** power * 4 * n8), (4, 2 ** power * 2 * n8),
             (5, 2 ** power * 2 * n8), (6, 4 * n8), (7, 4)]
    with open(path, "wb") as f:
        f.write(b"ptau" + struct.pack("<II", 1, len(sizes)))
        for sid, size in sizes:
            f.write(struct.pack("<IQ", sid, size))
            at = f.tell()
            data = {1: hdr, 2: tau_pts.tobytes(), 3: g2, 4: alpha_pts.tobytes()}.get(sid)
            if data is not None:
                f.write(data)
            f.seek(at + size)
        f.truncate()
