"""CPU tier: the separated Montgomery arithmetic (fp.cuh mul_wide / sqr_wide / redc / mul_sub), the lazily
reduced Fq2 (fp2.cuh mul_v / sqr_v / mul_sub_v) and the XYZZ additions built on them (ec.cuh madd / add),
compiled as plain C++ from tests/host_emu/emu_wide.cpp and checked against Python integers and oracle/ff.py."""
import ctypes
import os
import random
import subprocess

import pytest

from oracle.ff import BLS12_381, BN254, g1_group, g2_group

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "zokrates_b200", "csrc")

# (field id in emu_wide.cpp, modulus, 32-bit limbs)
FIELDS = [(0, BN254.r, 8, "bn254_fr"), (1, BN254.p, 8, "bn254_fq"), (2, BLS12_381.r, 8, "bls12_381_fr"),
          (3, BLS12_381.p, 12, "bls12_381_fq")]
CURVES = [(0, BN254, 8), (1, BLS12_381, 12)]
U32P = ctypes.POINTER(ctypes.c_uint32)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu_wide") / "libemu_wide.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-DZKB_EMU", "-shared", "-fPIC", "-I", os.path.join(ROOT, "include"),
                    "-I", CSRC, os.path.join(ROOT, "tests", "host_emu", "emu_wide.cpp"), "-o", out], check=True)
    dll = ctypes.CDLL(out)
    dll.emu_wide_fp.argtypes = [ctypes.c_int, ctypes.c_int] + [U32P] * 5
    dll.emu_wide_fp2.argtypes = [ctypes.c_int, ctypes.c_int] + [U32P] * 5
    dll.emu_wide_ec.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int] + [U32P] * 3
    return dll


def limbs(x, n):
    return (ctypes.c_uint32 * n)(*[(x >> (32 * i)) & 0xFFFFFFFF for i in range(n)])


def value(buf, lo, n):
    return sum(buf[lo + i] << (32 * i) for i in range(n))


class Fp:
    """Calls into the harness for one field; all values are plain integers (Montgomery images where it matters)."""

    def __init__(self, dll, fid, p, n):
        self.dll, self.fid, self.p, self.n = dll, fid, p, n
        self.R = 1 << (32 * n)
        self.Rinv = pow(self.R, -1, p)
        self.lazy = 4 * p < self.R

    def _op(self, op, a, b=0, c=0, d=0, out=None):
        n = self.n
        o = (ctypes.c_uint32 * (2 * n))()
        self.dll.emu_wide_fp(self.fid, op, limbs(a, 2 * n), limbs(b, n), limbs(c, n), limbs(d, n), o)
        return value(o, 0, out or n)

    def mul_wide(self, a, b):
        return self._op(0, a, b, out=2 * self.n)

    def sqr_wide(self, a):
        return self._op(1, a, out=2 * self.n)

    def redc(self, t):
        return self._op(2, t)

    def sqr(self, a):
        return self._op(3, a)

    def mul_sub(self, a, b, c, d):
        return self._op(4, a, b, c, d)


@pytest.fixture(scope="module", params=FIELDS, ids=lambda f: f[3])
def fp(request, lib):
    fid, p, n, _ = request.param
    return Fp(lib, fid, p, n)


def test_wide_products_edges(fp):
    p, R = fp.p, fp.R
    # reduced operands, the unreduced sums the lazy callers feed (< 2p), and the whole limb range
    edges = [0, 1, 2, p - 1, p, p + 1, 2 * p - 1, R - 1, R >> 1]
    for a in edges:
        assert fp.sqr_wide(a) == a * a, a
        for b in edges:
            assert fp.mul_wide(a, b) == a * b, (a, b)


def test_redc_edges(fp):
    p, R = fp.p, fp.R
    ts = [0, 1, p - 1, p, (p - 1) ** 2, p * R - 1, p * R - R, (p - 1) * R, (p - 1) * R + R - 1]
    if fp.lazy:  # the largest operands the lazy formulas build: two products (< 2p^2) and four (< 4p^2)
        ts += [2 * (p - 1) ** 2, (2 * p - 1) * (p - 1), 4 * (p - 1) ** 2, (2 * p - 1) ** 2]
    for t in ts:
        assert t < p * R
        r = fp.redc(t)
        assert r == t * fp.Rinv % p, t  # fully reduced: equality with the canonical residue


def test_random(fp):
    p, R, rnd = fp.p, fp.R, random.Random(20261015 + fp.fid)
    for _ in range(10000):
        a, b, c, d = (rnd.randrange(p) for _ in range(4))
        ua, ub = rnd.randrange(2 * p), rnd.randrange(2 * p)
        assert fp.mul_wide(ua, ub) == ua * ub
        assert fp.sqr_wide(ua) == ua * ua
        t = rnd.randrange(p * R)
        assert fp.redc(t) == t * fp.Rinv % p
        assert fp.sqr(a) == a * a * fp.Rinv % p
        if fp.lazy:
            assert fp.mul_sub(a, b, c, d) == (a * b - c * d) * fp.Rinv % p
    if fp.lazy:
        for a, b in ((0, 0), (p - 1, p - 1), (0, p - 1), (1, 0)):
            assert fp.mul_sub(p - 1, p - 1, a, b) == ((p - 1) ** 2 - a * b) * fp.Rinv % p
            assert fp.mul_sub(a, b, p - 1, p - 1) == (a * b - (p - 1) ** 2) * fp.Rinv % p


# ------------------------------------------------------------------------------------------------- Fq2
@pytest.fixture(scope="module", params=CURVES, ids=lambda c: c[1].name)
def curve(request, lib):
    return request.param


def fq2_call(dll, cid, n, op, *args):
    o = (ctypes.c_uint32 * (2 * n))()
    bufs = [limbs(x[0] | (x[1] << (32 * n)), 2 * n) for x in args]
    bufs += [limbs(0, 2 * n)] * (4 - len(bufs))
    dll.emu_wide_fp2(cid, op, *bufs, o)
    return (value(o, 0, n), value(o, n, n))


def test_fq2(curve, lib):
    cid, c, n = curve
    p = c.p
    Ri = pow(1 << (32 * n), -1, p)

    def mul(a, b):
        return ((a[0] * b[0] - a[1] * b[1]) * Ri % p, (a[0] * b[1] + a[1] * b[0]) * Ri % p)

    def sub(a, b):
        return ((a[0] - b[0]) % p, (a[1] - b[1]) % p)

    rnd = random.Random(7 + cid)
    edge = [(0, 0), (1, 0), (0, 1), (p - 1, p - 1), (p - 1, 0), (0, p - 1), (1, p - 1)]
    cases = [(a, b, e, f) for a in edge for b in edge for e, f in ((edge[3], edge[3]), ((0, 0), (0, 0)))]
    cases += [tuple((rnd.randrange(p), rnd.randrange(p)) for _ in range(4)) for _ in range(10000)]
    for a, b, e, f in cases:
        assert fq2_call(lib, cid, n, 0, a, b) == mul(a, b)
        assert fq2_call(lib, cid, n, 1, a) == mul(a, a)
        m1, m2 = mul(a, b), mul(e, f)
        assert fq2_call(lib, cid, n, 2, a, b, e, f) == sub(m1, m2)


# ------------------------------------------------------------------------------------------------- points
def ec_call(dll, cid, group, op, acc, q, n):
    k = n * group  # limbs per coordinate

    def pack(coords):
        out = []
        for x in coords:
            if group == 1:
                out += [(x >> (32 * i)) & 0xFFFFFFFF for i in range(n)]
            else:
                for part in x:
                    out += [(part >> (32 * i)) & 0xFFFFFFFF for i in range(n)]
        return (ctypes.c_uint32 * (4 * k))(*(out + [0] * (4 * k - len(out))))

    o = (ctypes.c_uint32 * (4 * k))()
    dll.emu_wide_ec(cid, group, op, pack(acc), pack(q), o)
    res = []
    for j in range(4):
        if group == 1:
            res.append(value(o, j * k, n))
        else:
            res.append((value(o, j * k, n), value(o, j * k + n, n)))
    return res


def group_tests(lib, cid, c, n, group):
    G = g1_group(c) if group == 1 else g2_group(c)
    F = G.F
    R = 1 << (32 * n)
    gen = c.g1 if group == 1 else c.g2
    rnd = random.Random(100 * cid + group)

    def mont(x):
        return x * R % c.p if group == 1 else (x[0] * R % c.p, x[1] * R % c.p)

    def unmont(x):
        Ri = pow(R, -1, c.p)
        return x * Ri % c.p if group == 1 else (x[0] * Ri % c.p, x[1] * Ri % c.p)

    def to_xyzz(P, z):  # affine -> XYZZ with ZZ = z^2, ZZZ = z^3 (Montgomery images)
        if P is None:
            return [F.zero] * 4
        zz, zzz = F.sqr(z), F.mul(F.sqr(z), z)
        return [mont(F.mul(P[0], zz)), mont(F.mul(P[1], zzz)), mont(zz), mont(zzz)]

    def from_xyzz(r):
        x, y, zz, zzz = (unmont(v) for v in r)
        if F.is_zero(zz):
            return None
        return (F.mul(x, F.inv(zz)), F.mul(y, F.inv(zzz)))

    def rand_z():
        return rnd.randrange(1, c.p) if group == 1 else (rnd.randrange(c.p), rnd.randrange(1, c.p))

    pts = [G.mul(gen, rnd.randrange(1, c.r)) for _ in range(6)]
    cases = []
    for P in pts:
        for Q in pts[:3]:
            cases.append((P, Q))          # generic
        cases.append((P, P))              # doubling branch
        cases.append((P, G.neg(P)))       # inverse branch -> identity
        cases.append((None, P))           # identity accumulator
        cases.append((P, None))           # point at infinity
    for P, Q in cases:
        want = G.add(P, Q)
        acc = to_xyzz(P, rand_z())
        q_aff = [F.zero, F.zero] if Q is None else [mont(Q[0]), mont(Q[1])]
        assert from_xyzz(ec_call(lib, cid, group, 0, acc, q_aff, n)) == want, ("madd", P, Q)
        assert from_xyzz(ec_call(lib, cid, group, 1, acc, to_xyzz(Q, rand_z()), n)) == want, ("add", P, Q)


def test_g1_additions(curve, lib):
    cid, c, n = curve
    group_tests(lib, cid, c, n, 1)


def test_g2_additions(curve, lib):
    cid, c, n = curve
    group_tests(lib, cid, c, n, 2)
