"""The separated Montgomery arithmetic (fp.cuh mul_wide / sqr_wide / redc / mul_sub), the lazily reduced Fq2 (fp2.cuh
mul_v / sqr_v / mul_sub_v) and the XYZZ additions built on them (ec.cuh madd / add), checked against Python integers
and oracle/ff.py.  Every test runs twice: on the host (CPU tier: tests/host_emu/emu_wide.cpp compiled as plain C++,
the carry emulation of hd.cuh) and on the device (-m gpu: tests/host_emu/dev_wide.cu on sm_90a, the inline-PTX carry
chains of hd.cuh, one thread per case so the doubling / inverse / identity branches mix inside a warp)."""
import ctypes
import os
import random
import subprocess

import pytest

from oracle.ff import BLS12_381, BN254, g1_group, g2_group

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "zokrates_b200", "csrc")

# (field id in wide_ops.cuh, modulus, 32-bit limbs)
FIELDS = [(0, BN254.r, 8, "bn254_fr"), (1, BN254.p, 8, "bn254_fq"), (2, BLS12_381.r, 8, "bls12_381_fr"),
          (3, BLS12_381.p, 12, "bls12_381_fq")]
CURVES = [(0, BN254, 8), (1, BLS12_381, 12)]
U32P = ctypes.POINTER(ctypes.c_uint32)


class Harness:
    """The op wrappers of tests/host_emu/wide_ops.cuh, batched: `host` is emu_wide.cpp built with g++ (the carry
    emulation of hd.cuh), `device` is dev_wide.cu built for sm_90a by __graft_entry__.build() (inline-PTX carries, one
    kernel launch per call, one thread per case)."""

    def __init__(self, dll, prefix, checked):
        self.fns = [getattr(dll, prefix + op) for op in ("fp", "fp2", "ec")]
        for f in self.fns[:2]:
            f.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_size_t] + [U32P] * 5
        self.fns[2].argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_size_t] + [U32P] * 3
        for f in self.fns:
            f.restype = ctypes.c_int if checked else None

    def _call(self, k, *args):
        rc = self.fns[k](*args)
        assert not rc, f"CUDA error {rc}"

    def fp(self, fid, op, n, a, b, c, d, out_limbs):
        """Case i: a[i] as 2N limbs, b / c / d as N; returns the first `out_limbs` limbs of each result as integers."""
        o = (ctypes.c_uint32 * (2 * n * len(a)))()
        self._call(0, fid, op, len(a), limbs(a, 2 * n), limbs(b, n), limbs(c, n), limbs(d, n), o)
        return [value(o, 2 * n * i, out_limbs) for i in range(len(a))]

    def fp2(self, cid, op, n, *args):
        """args: up to four lists of (c0, c1) pairs; returns the (c0, c1) results."""
        cnt = len(args[0])
        packed = [limbs([x[0] | (x[1] << (32 * n)) for x in arg], 2 * n) for arg in args]
        packed += [limbs([0] * cnt, 2 * n)] * (4 - len(packed))
        o = (ctypes.c_uint32 * (2 * n * cnt))()
        self._call(1, cid, op, cnt, *packed, o)
        return [(value(o, 2 * n * i, n), value(o, 2 * n * i + n, n)) for i in range(cnt)]

    def ec(self, cid, group, op, a, b, words):
        """a, b: per case the flat limb lists of 4 coordinates (`words` limbs each case); returns the flat result limbs."""
        cnt = len(a)
        ab = [(ctypes.c_uint32 * (words * cnt))(*[w for x in v for w in x]) for v in (a, b)]
        o = (ctypes.c_uint32 * (words * cnt))()
        self._call(2, cid, group, op, cnt, ab[0], ab[1], o)
        return [o[words * i:words * (i + 1)] for i in range(cnt)]


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu_wide") / "libemu_wide.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-DZKB_EMU", "-shared", "-fPIC", "-I", os.path.join(ROOT, "include"),
                    "-I", CSRC, os.path.join(ROOT, "tests", "host_emu", "emu_wide.cpp"), "-o", out], check=True)
    return Harness(ctypes.CDLL(out), "emu_wide_", False)


@pytest.fixture(scope="module")
def device_lib():
    import __graft_entry__ as g
    assert os.path.exists(g.DEV_WIDE_LIB), "tests/host_emu/libdev_wide.so missing: run __graft_entry__.build()"
    return Harness(ctypes.CDLL(g.DEV_WIDE_LIB), "dev_wide_", True)


def both_sides(params, ids):
    """Every parameter on the host (id as given) and on the device (id + "-device", marked gpu)."""
    return ([pytest.param((p, "host"), id=i) for p, i in zip(params, ids)] +
            [pytest.param((p, "device"), id=i + "-device", marks=pytest.mark.gpu) for p, i in zip(params, ids)])


def harness(request, side):
    return request.getfixturevalue(side + "_lib")


def limbs(xs, n):
    """Integers -> one flat uint32 buffer, `n` little-endian limbs each."""
    return (ctypes.c_uint32 * (n * len(xs)))(*[(x >> (32 * i)) & 0xFFFFFFFF for x in xs for i in range(n)])


def value(buf, lo, n):
    return sum(buf[lo + i] << (32 * i) for i in range(n))


class Fp:
    """Calls into the harness for one field; all values are plain integers (Montgomery images where it matters), and
    every method takes and returns lists (one batch per call)."""

    def __init__(self, h, fid, p, n):
        self.h, self.fid, self.p, self.n = h, fid, p, n
        self.R = 1 << (32 * n)
        self.Rinv = pow(self.R, -1, p)
        self.lazy = 4 * p < self.R

    def _op(self, op, a, b=None, c=None, d=None, out=None):
        zero = [0] * len(a)
        return self.h.fp(self.fid, op, self.n, a, b or zero, c or zero, d or zero, out or self.n)

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


@pytest.fixture(scope="module", params=both_sides(FIELDS, [f[3] for f in FIELDS]))
def fp(request):
    (fid, p, n, _), side = request.param
    return Fp(harness(request, side), fid, p, n)


def test_wide_products_edges(fp):
    p, R = fp.p, fp.R
    # reduced operands, the unreduced sums the lazy callers feed (< 2p), and the whole limb range
    edges = [0, 1, 2, p - 1, p, p + 1, 2 * p - 1, R - 1, R >> 1]
    assert fp.sqr_wide(edges) == [a * a for a in edges]
    pairs = [(a, b) for a in edges for b in edges]
    got = fp.mul_wide([a for a, _ in pairs], [b for _, b in pairs])
    for (a, b), g in zip(pairs, got):
        assert g == a * b, (a, b)


def test_redc_edges(fp):
    p, R = fp.p, fp.R
    ts = [0, 1, p - 1, p, (p - 1) ** 2, p * R - 1, p * R - R, (p - 1) * R, (p - 1) * R + R - 1]
    if fp.lazy:  # the largest operands the lazy formulas build: two products (< 2p^2) and four (< 4p^2)
        ts += [2 * (p - 1) ** 2, (2 * p - 1) * (p - 1), 4 * (p - 1) ** 2, (2 * p - 1) ** 2]
    assert all(t < p * R for t in ts)
    for t, r in zip(ts, fp.redc(ts)):
        assert r == t * fp.Rinv % p, t  # fully reduced: equality with the canonical residue


def test_random(fp):
    p, R, rnd = fp.p, fp.R, random.Random(20261015 + fp.fid)
    K = 10000
    a, b, c, d = ([rnd.randrange(p) for _ in range(K)] for _ in range(4))
    ua, ub = [rnd.randrange(2 * p) for _ in range(K)], [rnd.randrange(2 * p) for _ in range(K)]
    t = [rnd.randrange(p * R) for _ in range(K)]
    assert fp.mul_wide(ua, ub) == [x * y for x, y in zip(ua, ub)]
    assert fp.sqr_wide(ua) == [x * x for x in ua]
    assert fp.redc(t) == [x * fp.Rinv % p for x in t]
    assert fp.sqr(a) == [x * x * fp.Rinv % p for x in a]
    if fp.lazy:
        assert fp.mul_sub(a, b, c, d) == [(w * x - y * z) * fp.Rinv % p for w, x, y, z in zip(a, b, c, d)]
        e = [(0, 0), (p - 1, p - 1), (0, p - 1), (1, 0)]
        top = [p - 1] * len(e)
        ea, eb = [x for x, _ in e], [y for _, y in e]
        assert fp.mul_sub(top, top, ea, eb) == [((p - 1) ** 2 - x * y) * fp.Rinv % p for x, y in e]
        assert fp.mul_sub(ea, eb, top, top) == [(x * y - (p - 1) ** 2) * fp.Rinv % p for x, y in e]


# ------------------------------------------------------------------------------------------------- Fq2
@pytest.fixture(scope="module", params=both_sides(CURVES, [c[1].name for c in CURVES]))
def curve(request):
    """(curve id, curve, limbs, harness)"""
    (cid, c, n), side = request.param
    return cid, c, n, harness(request, side)


def test_fq2(curve):
    cid, c, n, lib = curve
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
    A, B, E, Fs = (list(x) for x in zip(*cases))
    assert lib.fp2(cid, 0, n, A, B) == [mul(a, b) for a, b in zip(A, B)]
    assert lib.fp2(cid, 1, n, A) == [mul(a, a) for a in A]
    assert lib.fp2(cid, 2, n, A, B, E, Fs) == [sub(mul(a, b), mul(e, f)) for a, b, e, f in cases]


# ------------------------------------------------------------------------------------------------- points
def ec_call(lib, cid, group, op, accs, qs, n):
    """One batch: accs / qs are per case 4 coordinates (q: affine x, y padded to 4); returns the XYZZ results."""
    k = n * group  # limbs per coordinate

    def pack(coords):
        out = []
        for x in coords:
            for part in ((x,) if group == 1 else x):
                out += [(part >> (32 * i)) & 0xFFFFFFFF for i in range(n)]
        return out + [0] * (4 * k - len(out))

    res = []
    for o in lib.ec(cid, group, op, [pack(a) for a in accs], [pack(q) for q in qs], 4 * k):
        if group == 1:
            res.append([value(o, j * k, n) for j in range(4)])
        else:
            res.append([(value(o, j * k, n), value(o, j * k + n, n)) for j in range(4)])
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
    # one batch per op: on the device the branches mix inside a warp
    accs = [to_xyzz(P, rand_z()) for P, _ in cases]
    q_aff = [[F.zero, F.zero] if Q is None else [mont(Q[0]), mont(Q[1])] for _, Q in cases]
    q_xyzz = [to_xyzz(Q, rand_z()) for _, Q in cases]
    got_madd = ec_call(lib, cid, group, 0, accs, q_aff, n)
    got_add = ec_call(lib, cid, group, 1, accs, q_xyzz, n)
    for (P, Q), gm, ga in zip(cases, got_madd, got_add):
        want = G.add(P, Q)
        assert from_xyzz(gm) == want, ("madd", P, Q)
        assert from_xyzz(ga) == want, ("add", P, Q)


def test_g1_additions(curve):
    cid, c, n, lib = curve
    group_tests(lib, cid, c, n, 1)


def test_g2_additions(curve):
    cid, c, n, lib = curve
    group_tests(lib, cid, c, n, 2)
