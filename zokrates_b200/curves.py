"""Curve / field constants the host side needs (names as `zokrates_field::Field::name()`,
/root/reference/zokrates_field/src/bn128.rs:1-13, bls12_381.rs:1-13, bls12_377.rs:1-13; moduli SURVEY.md App. C)."""
from __future__ import annotations

import hashlib
from dataclasses import dataclass


@dataclass(frozen=True)
class Curve:
    name: str
    id: int                 # ZKB_CURVE_* in include/zkb.h
    r: int                  # scalar field modulus
    p: int                  # base field modulus
    fr_bytes: int
    fq_bytes: int
    repr_shave_bits: int    # ark FpParameters::REPR_SHAVE_BITS of Fr (Fr::rand masking)
    two_adicity: int
    fr_generator: int

    @property
    def field_id(self) -> bytes:
        """`Field::id()`: first 4 bytes of sha256 of the modulus' little-endian bytes
        (zokrates_field/src/lib.rs:283-293) — the curve tag in the `out` program header."""
        return hashlib.sha256(self.r.to_bytes(self.fr_bytes, "little")).digest()[:4]


BN128 = Curve("bn128", 0, 21888242871839275222246405745257275088548364400416034343698204186575808495617,
              21888242871839275222246405745257275088696311157297823662689037894645226208583, 32, 32, 2, 28, 5)
BLS12_381 = Curve("bls12_381", 1, 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001,
                  0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab,
                  32, 48, 1, 32, 7)
BLS12_377 = Curve("bls12_377", 2, 0x12ab655e9a2ca55660b44d1e5c37b00159aa76fed00000010a11800000000001,
                  0x01ae3a4617c510eac63b05c06ca1493b1a22d9f300f5138f1ef3622fba094800170b5d44300000008508c00000000001,
                  32, 48, 3, 47, 22)
CURVES = {"bn128": BN128, "bls12_381": BLS12_381, "bls12_377": BLS12_377}


def curve(name_or_curve) -> Curve:
    if isinstance(name_or_curve, Curve):
        return name_or_curve
    return CURVES[name_or_curve]
