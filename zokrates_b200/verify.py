"""Host-side Groth16 verification — `Backend::<T, G16>::verify` of the drop-in boundary.

The reference verifies on the CPU (`zokrates_ark/src/groth16.rs:55-86`: rebuild the ark `VerifyingKey` from the hex
fields, `prepare_verifying_key`, `verify_proof`, i.e. e(A, B) = e(alpha, beta) · e(Σ x_i·γ_abc_i, gamma) · e(C, delta)); it is
milliseconds of work and SURVEY.md §8 row a13 keeps it off the GPU.  In the Rust shim `B200::verify` simply delegates to `Ark`.
This module is the Python mirror's equivalent: a small, tower-free pairing over big integers (BN254, BLS12-381 and BLS12-377),
written for clarity, not speed (a verification takes a few seconds) — Fq12 is Fq[w] / (w^12 − 2a·w^6 + a² − β) with the Fq2
unit u = w^6 − a, u² = β (ξ = a + u the sextic non-residue: β = −1 and a = 9 for BN254, β = −1 and a = 1 for BLS12-381,
β = −5 and a = 0 for BLS12-377), G2 points are mapped through the twist into E(Fq12), and the Miller loop uses plain affine
line functions.  Independent of `oracle/` (which the product never imports).
"""
from __future__ import annotations

from typing import List, Optional, Tuple

from .curves import curve as _curve
from .proof import G1Affine, G2Affine, Proof, VerificationKey

_PARAMS = {   # b of G1, beta (u^2), a (xi = a + u), twist type, |ate loop count|, extra Frobenius lines (BN only)
    "bn128": dict(b=3, beta=-1, a=9, mtwist=False, loop=29793968203157093288, bn=True),
    "bls12_381": dict(b=4, beta=-1, a=1, mtwist=True, loop=15132376222941642752, bn=False),
    "bls12_377": dict(b=1, beta=-5, a=0, mtwist=False, loop=0x8508c00000000001, bn=False),
}


class _Fq12:
    """Arithmetic in Fq[w] / (w^12 + c6 w^6 + c0); elements are 12-tuples of ints."""

    def __init__(self, p: int, a: int, beta: int = -1):
        self.p, self.c6, self.c0 = p, (-2 * a) % p, (a * a - beta) % p
        self.one = (1,) + (0,) * 11
        self.zero = (0,) * 12

    def add(self, x, y):
        p = self.p
        return tuple((u + v) % p for u, v in zip(x, y))

    def sub(self, x, y):
        p = self.p
        return tuple((u - v) % p for u, v in zip(x, y))

    def neg(self, x):
        p = self.p
        return tuple((-u) % p for u in x)

    def mul(self, x, y):
        p = self.p
        t = [0] * 23
        for i, u in enumerate(x):
            if u:
                for j, v in enumerate(y):
                    t[i + j] += u * v
        for k in range(22, 11, -1):              # w^k = -c6 w^(k-6) - c0 w^(k-12)
            v = t[k] % p
            if v:
                t[k - 6] -= v * self.c6
                t[k - 12] -= v * self.c0
        return tuple(v % p for v in t[:12])

    def scalar(self, x, k: int):
        p = self.p
        return tuple(u * k % p for u in x)

    def inv(self, x):
        """Extended Euclid on polynomials over Fq (degree <= 12)."""
        p = self.p
        lm, hm = [1] + [0] * 12, [0] * 13
        low = list(x) + [0]
        high = [self.c0, 0, 0, 0, 0, 0, self.c6, 0, 0, 0, 0, 0, 1]

        def deg(v):
            d = len(v) - 1
            while d and v[d] == 0:
                d -= 1
            return d

        while deg(low):
            dl, dh = deg(low), deg(high)
            r = [0] * 13                          # r = high // low
            tmp = list(high)
            inv_lead = pow(low[dl], -1, p)
            for i in range(dh - dl, -1, -1):
                q = tmp[dl + i] * inv_lead % p
                r[i] = q
                if q:
                    for c in range(dl + 1):
                        tmp[c + i] = (tmp[c + i] - q * low[c]) % p
            nm, new = list(hm), list(high)
            for i in range(13):
                if lm[i] or low[i]:
                    for j in range(13 - i):
                        if r[j]:
                            nm[i + j] -= lm[i] * r[j]
                            new[i + j] -= low[i] * r[j]
            nm = [v % p for v in nm]
            new = [v % p for v in new]
            lm, low, hm, high = nm, new, lm, low
        if low[0] == 0:
            raise ZeroDivisionError("inverse of zero in Fq12")
        k = pow(low[0], -1, p)
        return tuple(v * k % p for v in lm[:12])

    def pow(self, x, e: int):
        r, b = self.one, x
        while e:
            if e & 1:
                r = self.mul(r, b)
            b = self.mul(b, b)
            e >>= 1
        return r


def _embed_fq(v: int):
    return (v,) + (0,) * 11


class _Pairing:
    def __init__(self, name: str):
        self.c = _curve(name)
        self.P = _PARAMS[name]
        self.p = self.c.p
        self.F = _Fq12(self.p, self.P["a"], self.P["beta"])
        w = [0] * 12
        w[1] = 1
        self.w = tuple(w)
        self.w2 = self.F.mul(self.w, self.w)
        self.w3 = self.F.mul(self.w2, self.w)

    # -- points
    def on_g1(self, pt) -> bool:
        if pt is None:
            return True
        x, y = pt
        return (y * y - x * x * x - self.P["b"]) % self.p == 0

    def twist(self, q):
        """(x, y) in Fq2 x Fq2 on the twist -> point of E(Fq12): x·w^2, y·w^3 (D twist) or x / w^2, y / w^3 (M twist)."""
        F, a, p = self.F, self.P["a"], self.p
        (x0, x1), (y0, y1) = q
        xs = [0] * 12; ys = [0] * 12
        xs[0], xs[6] = (x0 - a * x1) % p, x1 % p
        ys[0], ys[6] = (y0 - a * y1) % p, y1 % p
        if self.P["mtwist"]:
            return F.mul(tuple(xs), F.inv(self.w2)), F.mul(tuple(ys), F.inv(self.w3))
        return F.mul(tuple(xs), self.w2), F.mul(tuple(ys), self.w3)

    def on_curve12(self, pt) -> bool:
        F = self.F
        x, y = pt
        return F.sub(F.mul(y, y), F.mul(F.mul(x, x), x)) == _embed_fq(self.P["b"])

    def _dbl(self, R):
        F = self.F
        x, y = R
        m = F.mul(F.scalar(F.mul(x, x), 3), F.inv(F.scalar(y, 2)))
        nx = F.sub(F.mul(m, m), F.scalar(x, 2))
        return m, (nx, F.sub(F.mul(m, F.sub(x, nx)), y))

    def _add(self, R, Q):
        F = self.F
        (x1, y1), (x2, y2) = R, Q
        if x1 == x2:
            if y1 == y2:
                return self._dbl(R)
            # vertical line: R + Q is the point at infinity.  Cannot happen for points of the prime-order subgroup; an
            # on-curve point of small order / outside the subgroup can get here (no subgroup check is made, as in the
            # reference) — such a proof is simply not valid
            raise DegeneratePoint("Miller loop reached the point at infinity (G2 point outside the prime-order subgroup)")
        m = F.mul(F.sub(y2, y1), F.inv(F.sub(x2, x1)))
        nx = F.sub(F.sub(F.mul(m, m), x1), x2)
        return m, (nx, F.sub(F.mul(m, F.sub(x1, nx)), y1))

    def _line(self, m, R, Pt):
        """slope-m line through R evaluated at the G1 point Pt = (xt, yt) embedded in Fq12."""
        F = self.F
        xt, yt = Pt
        return F.sub(F.mul(m, F.sub(xt, R[0])), F.sub(yt, R[1]))

    def miller(self, Q12, P1):
        F = self.F
        Pt = (_embed_fq(P1[0]), _embed_fq(P1[1]))
        R, f = Q12, F.one
        loop = self.P["loop"]
        for bit in bin(loop)[3:]:
            m, R2 = self._dbl(R)
            f = F.mul(F.mul(f, f), self._line(m, R, Pt))
            R = R2
            if bit == "1":
                m, R2 = self._add(R, Q12)
                f = F.mul(f, self._line(m, R, Pt))
                R = R2
        if self.P["bn"]:
            p = self.p
            Q1 = (F.pow(Q12[0], p), F.pow(Q12[1], p))
            nQ2 = (F.pow(Q1[0], p), F.neg(F.pow(Q1[1], p)))
            m, R2 = self._add(R, Q1)
            f = F.mul(f, self._line(m, R, Pt))
            R = R2
            m, _ = self._add(R, nQ2)
            f = F.mul(f, self._line(m, R, Pt))
        return f

    def product_is_one(self, pairs) -> bool:
        """Π e(P_i, Q_i) == 1 for G1 points P_i (or None) and twist points Q_i (or None); one final exponentiation."""
        F = self.F
        f = F.one
        for P1, Q in pairs:
            if P1 is None or Q is None:
                continue
            f = F.mul(f, self.miller(self.twist(Q), P1))
        return F.pow(f, (self.p ** 12 - 1) // self.c.r) == F.one

    # -- G1 affine arithmetic for the public-input combination
    def g1_add(self, A, B):
        p = self.p
        if A is None:
            return B
        if B is None:
            return A
        (x1, y1), (x2, y2) = A, B
        if x1 == x2:
            if (y1 + y2) % p == 0:
                return None
            m = 3 * x1 * x1 * pow(2 * y1, -1, p) % p
        else:
            m = (y2 - y1) * pow(x2 - x1, -1, p) % p
        x3 = (m * m - x1 - x2) % p
        return x3, (m * (x1 - x3) - y1) % p

    def g1_mul(self, A, k: int):
        R = None
        while k:
            if k & 1:
                R = self.g1_add(R, A)
            A = self.g1_add(A, A)
            k >>= 1
        return R


_cache = {}


def _pairing(name: str) -> _Pairing:
    if name not in _cache:
        _cache[name] = _Pairing(name)
    return _cache[name]


def _g1(pt: G1Affine, p: int) -> Optional[Tuple[int, int]]:
    x, y = int(pt.x, 16), int(pt.y, 16)
    if x >= p or y >= p:
        raise ValueError("G1 coordinate not reduced")
    return None if x == 0 and y == 0 else (x, y)


def _g2(pt: G2Affine, p: int):
    v = [int(s, 16) for s in (pt.x[0], pt.x[1], pt.y[0], pt.y[1])]
    if any(c >= p for c in v):
        raise ValueError("G2 coordinate not reduced")
    return None if not any(v) else ((v[0], v[1]), (v[2], v[3]))


class DegeneratePoint(ValueError):
    """A G2 input drove the Miller loop into the point at infinity: not a point of the prime-order subgroup."""


def verify_proof(vk: VerificationKey, proof: Proof) -> bool:
    """True iff the proof satisfies the Groth16 equation under `vk` for its public inputs.  Malformed input raises, as
    the reference panics (`verify_proof(..).unwrap()`, zokrates_ark/src/groth16.rs:85): wrong number of public inputs,
    unreduced coordinates, points off the curve."""
    if vk.curve != proof.curve:
        raise ValueError("proof and verification key are for different curves")
    pr = _pairing(vk.curve)
    c = pr.c
    inputs = proof.input_values()
    if len(inputs) + 1 != len(vk.gamma_abc):
        raise ValueError("MalformedVerifyingKey: %d public inputs for %d gamma_abc points" % (len(inputs), len(vk.gamma_abc)))
    if any(x >= c.r for x in inputs):
        raise ValueError("public input not reduced")
    A, C = _g1(proof.proof.a, c.p), _g1(proof.proof.c, c.p)
    B = _g2(proof.proof.b, c.p)
    alpha = _g1(vk.alpha, c.p)
    beta, gamma, delta = _g2(vk.beta, c.p), _g2(vk.gamma, c.p), _g2(vk.delta, c.p)
    abc = [_g1(g, c.p) for g in vk.gamma_abc]
    for pt in [A, C, alpha] + abc:
        if not pr.on_g1(pt):
            raise ValueError("G1 point is not on the curve")
    for q in (B, beta, gamma, delta):
        if q is not None and not pr.on_curve12(pr.twist(q)):
            raise ValueError("G2 point is not on the curve")
    acc = abc[0]
    for x, g in zip(inputs, abc[1:]):
        acc = pr.g1_add(acc, pr.g1_mul(g, x))
    negA = None if A is None else (A[0], (-A[1]) % c.p)
    try:
        return pr.product_is_one([(negA, B), (alpha, beta), (acc, gamma), (C, delta)])
    except DegeneratePoint:
        return False                                  # the reference's verify returns false here, it does not crash


def verify_proof_gm17(vk, proof: Proof) -> bool:
    """`impl Backend<T, GM17> for Ark`::verify (zokrates_ark/src/gm17.rs:77-117 -> ark-gm17 `verify_proof`), on the host:
        e(A + G^alpha, B + H^beta) = e(G^alpha, H^beta) e(psi, H^gamma) e(C, H),   e(A, H^gamma) = e(G^gamma, B),
    psi = query_0 + sum x_i query_i.  Malformed input raises, as the reference panics."""
    if vk.curve != proof.curve:
        raise ValueError("proof and verification key are for different curves")
    pr = _pairing(vk.curve)
    c = pr.c
    inputs = proof.input_values()
    if len(inputs) + 1 != len(vk.query):
        raise ValueError("MalformedVerifyingKey: %d public inputs for %d query points" % (len(inputs), len(vk.query)))
    if any(x >= c.r for x in inputs):
        raise ValueError("public input not reduced")
    A, C = _g1(proof.proof.a, c.p), _g1(proof.proof.c, c.p)
    B = _g2(proof.proof.b, c.p)
    g_alpha, g_gamma = _g1(vk.g_alpha, c.p), _g1(vk.g_gamma, c.p)
    h, h_beta, h_gamma = _g2(vk.h, c.p), _g2(vk.h_beta, c.p), _g2(vk.h_gamma, c.p)
    query = [_g1(g, c.p) for g in vk.query]
    for pt in [A, C, g_alpha, g_gamma] + query:
        if not pr.on_g1(pt):
            raise ValueError("G1 point is not on the curve")
    for q in (B, h, h_beta, h_gamma):
        if q is not None and not pr.on_curve12(pr.twist(q)):
            raise ValueError("G2 point is not on the curve")
    psi = query[0]
    for x, g in zip(inputs, query[1:]):
        psi = pr.g1_add(psi, pr.g1_mul(g, x))
    neg = lambda P: None if P is None else (P[0], (-P[1]) % c.p)     # noqa: E731
    # e(A, B + H^beta) e(G^alpha, B) = e(psi, H^gamma) e(C, H)   (the e(G^alpha, H^beta) terms cancel: no G2 addition needed)
    try:
        first = pr.product_is_one([(A, B), (A, h_beta), (g_alpha, B), (neg(psi), h_gamma), (neg(C), h)])
        second = pr.product_is_one([(A, h_gamma), (neg(g_gamma), B)])
    except DegeneratePoint:
        return False
    return first and second
