"""BLS12-377 for the tests (test infrastructure only): curve parameters in oracle/ff.py's `CurveParams` form, its
Fq2 = Fq[u]/(u^2 + 5), the G1 / G2 groups, and the Groth16 / GM17 setups and trapdoor predictions.

oracle/ff.py's Fq2 and pairing are written for u^2 = -1, so its `g2_group`, `b2` and pairing do not apply to this curve.
Everything here that is not group arithmetic comes from the oracle unchanged: the QAP / SAP evaluation at tau, the witness
maps, the domains (Fr only), `fr_rand` and the ark serialisation.  Pairing checks use the product's
`zokrates_b200.verify`, which is pinned for this curve by four proofs made by ark (tests/golden/ark_gm17_bls12_377.json).
"""
from oracle import ark, gm17
from oracle.ff import CurveParams, FqOps, Group, inv_mod

P = 0x01ae3a4617c510eac63b05c06ca1493b1a22d9f300f5138f1ef3622fba094800170b5d44300000008508c00000000001
R = 0x12ab655e9a2ca55660b44d1e5c37b00159aa76fed00000010a11800000000001
X = 0x8508c00000000001
BETA = -5


class Fq2Ops:
    """Fq[u]/(u^2 - beta), beta = -5 (ark-bls12-377 Fq2Parameters::NONRESIDUE)."""

    zero = (0, 0)
    one = (1, 0)

    def __init__(self, p=P, beta=BETA):
        self.p, self.beta = p, beta

    def add(self, a, b):
        return ((a[0] + b[0]) % self.p, (a[1] + b[1]) % self.p)

    def sub(self, a, b):
        return ((a[0] - b[0]) % self.p, (a[1] - b[1]) % self.p)

    def neg(self, a):
        return ((-a[0]) % self.p, (-a[1]) % self.p)

    def mul(self, a, b):
        p = self.p
        return ((a[0] * b[0] + self.beta * a[1] * b[1]) % p, (a[0] * b[1] + a[1] * b[0]) % p)

    def sqr(self, a):
        return self.mul(a, a)

    def inv(self, a):
        p = self.p
        d = inv_mod((a[0] * a[0] - self.beta * a[1] * a[1]) % p, p)
        return (a[0] * d % p, (-a[1]) * d % p)

    def is_zero(self, a):
        return a[0] % self.p == 0 and a[1] % self.p == 0

    def from_int(self, k):
        return (k % self.p, 0)


F2 = Fq2Ops()
B2 = F2.inv((0, 1))            # D-twist: y^2 = x^3 + 1/u

BLS12_377 = CurveParams(
    name="bls12_377", r=R, p=P, fr_bytes=32, fq_bytes=48, two_adicity=47, fr_generator=22,
    b1=1, xi=(0, 1), twist='D',
    g1=(0x008848defe740a67c8fc6225bf87ff5485951e2caa9d41bb188282c8bd37cb5cd5481512ffcd394eeab9b16eb21be9ef,
        0x01914a69c5102eff1f674f5d30afeec4bd7fb348ca3e52d96d182ad44fb82305c2fe3d3634a9591afd82de55559c8ea6),
    g2=((0x018480be71c785fec89630a2a3841d01c565f071203e50317ea501f557db6b9b71889f52bb53540274e3e48f7c005196,
         0x00ea6040e700403170dc5a51b1b140d5532777ee6651cecbe7223ece0799c9de5cf89984bff76fe6b26bfefa6ea16afe),
        (0x00690d665d446f7bd960736bcbb2efb4de03ed7274b49a58e458c282f832d204f2cf88886d8c7c2ef094094409fd4ddf,
         0x00f8169fd28355189e549da3151a70aa61ef11ac3d591bf12463b01acee304c24279b83f5e52270bd9a1cdd185eb8f93)),
    ate_loop=X, repr_shave_bits=3, bn_like=False,
)
C = BLS12_377
G1 = Group(FqOps(P), 1, R)
G2 = Group(F2, B2, R)


# ------------------------------------------------------------------------------------------------ Groth16
def setup(r1cs, td):
    """ark-groth16 generate_parameters with an explicit trapdoor (oracle/ark.py `setup` with this curve's groups)."""
    r = C.r
    d, a, b, cc, zt = ark.qap_at_tau(C, r1cs, td.tau)
    ni = r1cs.num_instance
    g1 = G1.mul(C.g1, td.g1_k)
    g2 = G2.mul(C.g2, td.g2_k)
    ginv, dinv = inv_mod(td.gamma, r), inv_mod(td.delta, r)
    abc = [(td.beta * a[i] + td.alpha * b[i] + cc[i]) % r for i in range(r1cs.num_variables)]
    h_scalars, tp = [], 1
    for _ in range(d.n - 1):
        h_scalars.append(zt * dinv % r * tp % r)
        tp = tp * td.tau % r
    return ark.ProvingKey(
        alpha_g1=G1.mul(g1, td.alpha), beta_g2=G2.mul(g2, td.beta), gamma_g2=G2.mul(g2, td.gamma),
        delta_g2=G2.mul(g2, td.delta),
        gamma_abc_g1=[G1.mul(g1, abc[i] * ginv % r) for i in range(ni)],
        beta_g1=G1.mul(g1, td.beta), delta_g1=G1.mul(g1, td.delta),
        a_query=[G1.mul(g1, x) for x in a], b_g1_query=[G1.mul(g1, x) for x in b], b_g2_query=[G2.mul(g2, x) for x in b],
        h_query=[G1.mul(g1, x) for x in h_scalars],
        l_query=[G1.mul(g1, abc[i] * dinv % r) for i in range(ni, r1cs.num_variables)])


def expected_proof(r1cs, td, z, r, s):
    """(A, B, C) from the trapdoor: Fr arithmetic and one scalar multiplication each (oracle/ark.py's prediction)."""
    q = C.r
    d, a, b, cc, zt = ark.qap_at_tau(C, r1cs, td.tau)
    az = sum(x * y for x, y in zip(a, z)) % q
    bz = sum(x * y for x, y in zip(b, z)) % q
    cz = sum(x * y for x, y in zip(cc, z)) % q
    dinv = inv_mod(td.delta, q)
    a_dlog = (td.alpha + az + r * td.delta) % q
    b_dlog = (td.beta + bz + s * td.delta) % q
    ni = r1cs.num_instance
    l_dlog = sum((td.beta * a[i] + td.alpha * b[i] + cc[i]) * z[i] for i in range(ni, len(z))) % q * dinv % q
    h_dlog = (az * bz - cz) % q * dinv % q
    c_dlog = (l_dlog + h_dlog + s * a_dlog + r * b_dlog - r * s % q * td.delta) % q
    g1 = G1.mul(C.g1, td.g1_k)
    g2 = G2.mul(C.g2, td.g2_k)
    return G1.mul(g1, a_dlog), G2.mul(g2, b_dlog), G1.mul(g1, c_dlog)


# ------------------------------------------------------------------------------------------------ GM17
def gm17_setup(r1cs, td):
    """ark-gm17 generate_parameters with an explicit trapdoor (oracle/gm17.py `setup` with this curve's groups)."""
    q = C.r
    d, a, cc, zt = gm17.sap_at_tau(C, r1cs, td.tau)
    ni, nv = r1cs.num_instance, len(a)
    g, h = G1.mul(C.g1, td.g1_k), G2.mul(C.g2, td.g2_k)
    ab = (td.alpha + td.beta) % q
    g2z = td.gamma * td.gamma % q * zt % q
    tp, powers = 1, []
    for _ in range(d.n + 1):
        powers.append(g2z * tp % q)
        tp = tp * td.tau % q
    return gm17.Gm17ProvingKey(
        h_g2=h, g_alpha_g1=G1.mul(g, td.alpha), h_beta_g2=G2.mul(h, td.beta), g_gamma_g1=G1.mul(g, td.gamma),
        h_gamma_g2=G2.mul(h, td.gamma),
        query=[G1.mul(g, (td.gamma * cc[i] + ab * a[i]) % q) for i in range(ni)],
        a_query=[G1.mul(g, a[i] * td.gamma % q) for i in range(nv)],
        b_query=[G2.mul(h, a[i] * td.gamma % q) for i in range(nv)],
        c_query_1=[G1.mul(g, (td.gamma * td.gamma % q * cc[i] + ab * td.gamma % q * a[i]) % q) for i in range(ni, nv)],
        c_query_2=[G1.mul(g, 2 * g2z * a[i] % q) for i in range(nv)],
        g_gamma_z=G1.mul(g, td.gamma * zt % q), h_gamma_z=G2.mul(h, td.gamma * zt % q),
        g_ab_gamma_z=G1.mul(g, ab * td.gamma % q * zt % q), g_gamma2_z2=G1.mul(g, g2z * zt % q),
        g_gamma2_z_t=[G1.mul(g, s) for s in powers])


def gm17_expected_proof(r1cs, td, z, d1, d2, r):
    """(A, B, C) from the trapdoor (oracle/gm17.py's prediction with this curve's groups)."""
    q = C.r
    d, a, cc, zt = gm17.sap_at_tau(C, r1cs, td.tau)
    full = gm17.sap_assignment(C, r1cs, z)
    ni = r1cs.num_instance
    a0 = sum(x * y for x, y in zip(a, full)) % q
    c0 = sum(x * y for x, y in zip(cc, full)) % q
    at = (a0 + d1 * zt) % q
    ct = (c0 + d2 * zt) % q
    ht = (at * at - ct) % q * inv_mod(zt, q) % q
    ga, ab = td.gamma, (td.alpha + td.beta) % q
    a_dlog = ga * (at + r * zt) % q
    aux = sum((ga * ga % q * cc[i] + ab * ga % q * a[i]) * full[i] for i in range(ni, len(full))) % q
    c_dlog = (aux + d1 * ab % q * ga % q * zt + d2 * ga % q * ga % q * zt
              + r * r % q * ga % q * ga % q * zt % q * zt + r * ab % q * ga % q * zt
              + ga * ga % q * zt % q * (ht + 2 * r * at)) % q
    g, h = G1.mul(C.g1, td.g1_k), G2.mul(C.g2, td.g2_k)
    return G1.mul(g, a_dlog), G2.mul(h, a_dlog), G1.mul(g, c_dlog)


def expected_proof_csr(r1, td, z, r, s):
    """`expected_proof` for a product R1CS (CSR matrices) and assignment (uint64[m, 4]), without building per-column
    QAP vectors: a(tau)·z = sum_j L_j(tau) (A z)_j + sum_(i < ni) L_(N+i) z_i, and the same for b and c; the l term uses the
    instance columns only.  Returns the proof bytes."""
    from zokrates_b200._lib import fr_from_array
    q, N, ni = C.r, r1.num_constraints, r1.num_instance
    zz = fr_from_array(z)
    d = ark.Domain(C, N + ni)
    n, t = d.n, td.tau
    # L_j(t) = Z(t)/n * w^j / (t - w^j), j < N + ni, one batched inversion
    ws, w = [], 1
    for _ in range(N + ni):
        ws.append(w)
        w = w * d.omega % q
    dens = [(t - x) % q for x in ws]
    pref, acc = [], 1
    for x in dens:
        pref.append(acc)
        acc = acc * x % q
    inv = inv_mod(acc, q)
    invs = [0] * len(dens)
    for j in range(len(dens) - 1, -1, -1):
        invs[j] = inv * pref[j] % q
        inv = inv * dens[j] % q
    k = (pow(t, n, q) - 1) * inv_mod(n, q) % q
    L = [k * x % q * y % q for x, y in zip(ws, invs)]
    tot, inst = [], []
    for mi, (rowptr, col, val) in enumerate(r1.matrices()):
        vals = fr_from_array(val)
        rowptr, col = rowptr.tolist(), col.tolist()
        t_all, t_inst = 0, [0] * ni
        for j in range(N):
            lo, hi = rowptr[j], rowptr[j + 1]
            acc = 0
            for e in range(lo, hi):
                acc += vals[e] * zz[col[e]]
                if col[e] < ni:
                    t_inst[col[e]] += L[j] * vals[e]
            t_all += L[j] * (acc % q)
        if mi == 0:
            for i in range(ni):
                t_all += L[N + i] * zz[i]
                t_inst[i] += L[N + i]
        tot.append(t_all % q)
        inst.append([x % q for x in t_inst])
    az, bz, cz = tot
    aux = [(tot[m] - sum(inst[m][i] * zz[i] for i in range(ni))) % q for m in range(3)]
    dinv = inv_mod(td.delta, q)
    a_dlog = (td.alpha + az + r * td.delta) % q
    b_dlog = (td.beta + bz + s * td.delta) % q
    l_dlog = (td.beta * aux[0] + td.alpha * aux[1] + aux[2]) % q * dinv % q
    h_dlog = (az * bz - cz) % q * dinv % q
    c_dlog = (l_dlog + h_dlog + s * a_dlog + r * b_dlog - r * s % q * td.delta) % q
    g1 = G1.mul(C.g1, td.g1_k)
    g2 = G2.mul(C.g2, td.g2_k)
    return ark.ser_g1(C, G1.mul(g1, a_dlog)) + ark.ser_g2(C, G2.mul(g2, b_dlog)) + ark.ser_g1(C, G1.mul(g1, c_dlog))


def to_oracle(r1):
    """A product R1CS (CSR) as oracle/ark.py's row lists."""
    from zokrates_b200._lib import fr_from_array
    mats = []
    for rowptr, col, val in r1.matrices():
        vals, rowptr, col = fr_from_array(val), rowptr.tolist(), col.tolist()
        mats.append([[(col[e], vals[e]) for e in range(rowptr[j], rowptr[j + 1])] for j in range(r1.num_constraints)])
    return ark.R1CS(r1.num_instance, r1.num_witness, *mats)


# ------------------------------------------------------------------------------------------------ NTT (C)
_NTT = None


def _ntt_lib():
    """tests/bls12_377_ntt.c, built once per process into a temporary directory."""
    global _NTT
    if _NTT is None:
        import ctypes
        import os
        import subprocess
        import tempfile
        src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "bls12_377_ntt.c")
        out = os.path.join(tempfile.mkdtemp(prefix="ntt377_"), "libntt377.so")
        subprocess.run(["gcc", "-O2", "-fopenmp", "-shared", "-fPIC", src, "-o", out], check=True)
        _NTT = ctypes.CDLL(out)
        _NTT.ref_ntt377.argtypes = [ctypes.c_void_p, ctypes.c_uint32] + [ctypes.c_void_p] * 4
        _NTT.ref_ntt377.restype = None
    return _NTT


def ref_ntt(x, log_n, inverse=False, coset=False):
    """ark's fft / ifft / coset_fft / coset_ifft of uint64[2^log_n, 4] (canonical limbs) on this curve's Fr, in C; the
    domain constants come from Python integers (w = 22^((r - 1) / 2^log_n))."""
    import numpy as np
    from zokrates_b200._lib import fr_array
    n = 1 << log_n
    w = pow(C.fr_generator, (R - 1) >> log_n, R)
    g = C.fr_generator
    consts = fr_array([pow(w, -1, R) if inverse else w, pow(n, -1, R) if inverse else 1, g, pow(g, -1, R)])
    a = np.ascontiguousarray(x, dtype=np.uint64).copy()
    assert a.shape == (n, 4)
    ptr = [consts[i:i + 1].ctypes.data for i in range(4)]
    pre = ptr[2] if coset and not inverse else None
    post = ptr[3] if coset and inverse else None
    _ntt_lib().ref_ntt377(a.ctypes.data, log_n, ptr[0], ptr[1], pre, post)
    return a
