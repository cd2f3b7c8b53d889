"""Field moduli the host-side marshalling needs (same constants as csrc/gen_params.py)."""
from . import _lib

FR_MODULUS = {
    _lib.CURVE_BLS12_381: 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001,
    _lib.CURVE_BN254: 21888242871839275222246405745257275088548364400416034343698204186575808495617,
    _lib.CURVE_BLS12_377: 0x12ab655e9a2ca55660b44d1e5c37b00159aa76fed00000010a11800000000001,
}
FQ_MODULUS = {
    _lib.CURVE_BLS12_381: 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab,
    _lib.CURVE_BN254: 21888242871839275222246405745257275088696311157297823662689037894645226208583,
    _lib.CURVE_BLS12_377: 0x01ae3a4617c510eac63b05c06ca1493b1a22d9f300f5138f1ef3622fba094800170b5d44300000008508c00000000001,
}
# standard G1 generators (x, y)
G1_GENERATOR = {
    _lib.CURVE_BLS12_381: (
        0x17f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb,
        0x08b3f481e3aaa0f1a09e30ed741d8ae4fcf5e095d5d00af600db18cb2c04b3edd03cc744a2888ae40caa232946c5e7e1),
    _lib.CURVE_BN254: (1, 2),
    _lib.CURVE_BLS12_377: (
        0x008848defe740a67c8fc6225bf87ff5485951e2caa9d41bb188282c8bd37cb5cd5481512ffcd394eeab9b16eb21be9ef,
        0x01914a69c5102eff1f674f5d30afeec4bd7fb348ca3e52d96d182ad44fb82305c2fe3d3634a9591afd82de55559c8ea6),
}
CURVE_IDS = {"bls12_381": _lib.CURVE_BLS12_381, "bn254": _lib.CURVE_BN254, "bls12_377": _lib.CURVE_BLS12_377}


def fr_to_mont(curve_id, v):
    p = FR_MODULUS[curve_id]
    return (v % p) * (1 << 256) % p


def fr_from_mont(curve_id, v):
    p = FR_MODULUS[curve_id]
    return v * pow(1 << 256, -1, p) % p


def fq_to_mont(curve_id, v):
    p = FQ_MODULUS[curve_id]
    n = _lib.LIMBS[curve_id][1]
    return (v % p) * (1 << (64 * n)) % p


def fq_from_mont(curve_id, v):
    p = FQ_MODULUS[curve_id]
    n = _lib.LIMBS[curve_id][1]
    return v * pow(1 << (64 * n), -1, p) % p
