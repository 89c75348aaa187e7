"""BLS12-377: the curve constants, four GM17 proofs made by ark on this curve, the Fq2 = Fq[u]/(u^2 + 5) arithmetic and the
point additions over it, and Groth16 / GM17 setup, proving and verification through the host emulation.

The op tests run on the host (tests/host_emu/emu_wide_bls12_377.cpp, the carry emulation of hd.cuh) and, marked gpu, on the
device (tests/host_emu/dev_wide_bls12_377.cu, the inline-PTX carries), as tests/test_field_wide.py does for the other two
curves.  Expected values come from Python integers and tests/bls12_377_ref.py."""
import ctypes
import io
import json
import os
import random
import re
import subprocess

import pytest

from oracle import ark, gm17
from tests import bls12_377_ref as B
from tests.test_field_wide import Harness, ec_call
from tests.util import proof_bytes
from zokrates_b200 import backend, ir, rng as prng, synthetic, zir
from zokrates_b200._lib import Context, fr_from_array
from zokrates_b200.curves import BLS12_377, CURVES
from zokrates_b200.proof import G1Affine, G2Affine, Gm17VerificationKey, Proof, ProofPoints, gm17_vk_from_pk_bytes
from zokrates_b200.verify import verify_proof, verify_proof_gm17

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "zokrates_b200", "csrc")
P, R, X = B.P, B.R, B.X
CID = 2


# ------------------------------------------------------------------------------------------------- constants
def test_curve_relations():
    assert R == X ** 4 - X ** 2 + 1 and R.bit_length() == 253
    assert (X - 1) ** 2 * R % 3 == 0 and P == (X - 1) ** 2 * R // 3 + X and P.bit_length() == 377
    assert (R - 1) % (1 << 47) == 0 and ((R - 1) >> 47) % 2 == 1
    assert (P - 1) % (1 << 46) == 0 and ((P - 1) >> 46) % 2 == 1
    root = pow(22, (R - 1) >> 47, R)
    assert pow(root, 1 << 46, R) == R - 1                     # order exactly 2^47
    assert pow(P - 5, (P - 1) // 2, P) == P - 1                # -5 is a non-residue: Fq[u]/(u^2 + 5) is a field
    assert (1 << 384) // P == 152 and (1 << 256) * 10 // R == 137   # headroom R/p ~ 152, R/r ~ 13.7
    c = BLS12_377
    assert (c.id, c.r, c.p, c.fr_bytes, c.fq_bytes, c.repr_shave_bits, c.two_adicity, c.fr_generator) == \
        (2, R, P, 32, 48, 3, 47, 22)
    assert CURVES["bls12_377"] is c and (1 << 256) >> c.repr_shave_bits > R > (1 << 256) >> (c.repr_shave_bits + 1)


def test_generators():
    g1, g2 = B.C.g1, B.C.g2
    assert B.G1.is_on_curve(g1) and B.G1.mul(g1, R) is None and B.G1.mul(g1, R - 1) == B.G1.neg(g1)
    assert B.G2.is_on_curve(g2) and B.G2.mul(g2, R) is None and B.G2.mul(g2, R - 1) == B.G2.neg(g2)
    assert B.F2.mul(B.B2, (0, 1)) == (1, 0)                   # D-twist: b2 = 1 / u, and w^6 = u


def test_field_id():
    assert BLS12_377.field_id.hex() == "c2955ab5" == zir.CURVE_IDS["bls12_377"].hex()
    assert [CURVES[n].field_id.hex() for n in ("bn128", "bls12_381")] == ["b4f7b5bd", "40d8c1f9"]
    src = open(os.path.join(CSRC, "prog.cuh")).read()
    table = re.search(r"CURVE_ID\[3\]\[4\] = \{(.*?)\};", src, re.S).group(1)
    rows = [bytes(int(v, 16) for v in re.findall(r"0x([0-9a-f]{2})", row)) for row in re.findall(r"\{([^{}]*)\}", table)]
    assert rows == [CURVES[n].field_id for n in ("bn128", "bls12_381", "bls12_377")]
    assert re.search(r"#define ZKB_CURVE_BLS12_377 2\b", open(os.path.join(ROOT, "include", "zkb.h")).read())


def _struct(name):
    src = open(os.path.join(CSRC, "field_params.cuh")).read()
    body = re.search(r"struct %s \{(.*?)\n\};" % name, src, re.S).group(1)
    out = {k: int(v) for k, v in re.findall(r"int (\w+) = (-?\d+);", body)}
    for fn, arr in re.findall(r"uint32_t (\w+)\(int i\) \{ constexpr uint32_t t\[\d+\] = \{([^}]*)\}", body):
        out[fn] = sum(int(v, 16) << (32 * i) for i, v in enumerate(re.findall(r"0x([0-9a-f]{8})u", arr)))
    return out


def test_field_params_limbs():
    for name, m, adic, gen in (("Bls377Fr", R, 47, 22), ("Bls377Fq", P, 46, 15)):
        s, n = _struct(name), (m.bit_length() + 31) // 32
        Rm = 1 << (32 * n)
        assert (s["N"], s["BITS"], s["TWO_ADICITY"]) == (n, m.bit_length(), adic)
        assert (s["mod"], s["r1"], s["r2"], s["gen"], s["pm2"]) == (m, Rm % m, Rm * Rm % m, gen * Rm % m, m - 2)
        assert s["root"] == pow(gen, (m - 1) >> adic, m) * Rm % m
    assert _struct("Bls377Fq")["FP2_NONRESIDUE"] == -5 and "FP2_NONRESIDUE" not in _struct("Bls381Fq")
    g = _struct("Bls377Gen")
    Rq = 1 << 384
    (x0, x1), (y0, y1) = B.C.g2
    assert [g[k] for k in ("g1x", "g1y", "g2x0", "g2x1", "g2y0", "g2y1")] == \
        [v * Rq % P for v in (B.C.g1[0], B.C.g1[1], x0, x1, y0, y1)]


# ------------------------------------------------------------------------------------------------- ark fixture
def _fixture():
    with open(os.path.join(ROOT, "tests", "golden", "ark_gm17_bls12_377.json")) as f:
        return json.load(f)["proofs"]


def _proof_vk(e, inputs=None, swap=False):
    p, v = e["proof"], e["vk"]
    sw = (lambda t: t[::-1]) if swap else (lambda t: t)
    g2 = lambda x: G2Affine(tuple(sw(x[0])), tuple(sw(x[1])))       # noqa: E731
    pr = Proof(ProofPoints(G1Affine(*p["a"]), g2(p["b"]), G1Affine(*p["c"])), inputs or e["inputs"], "bls12_377", "gm17")
    vk = Gm17VerificationKey(g2(v["h"]), G1Affine(*v["g_alpha"]), g2(v["h_beta"]), G1Affine(*v["g_gamma"]), g2(v["h_gamma"]),
                             [G1Affine(*q) for q in v["query"]], "bls12_377")
    return pr, vk


def _swapped_rejected(pr, vk):
    try:
        return not verify_proof_gm17(vk, pr)
    except ValueError as e:                # a swapped point is off the twist: the verifier refuses it, as ark panics
        return "not on the curve" in str(e)


@pytest.mark.parametrize("k", range(4), ids=["stdlib_gm17_3", "snark_verify_1", "snark_verify_2", "snark_verify_5"])
def test_ark_gm17_proofs(k):
    """Proofs made by `zokrates setup / generate-proof -b ark -s gm17` on BLS12-377 verify; a changed public input and
    swapped G2 coordinates (the JSON order is (c0, c1)) do not.  Pins the curve, the twist, u^2 = -5 and the verifier."""
    e = _fixture()[k]
    assert len(e["inputs"]) == [3, 1, 2, 5][k]
    pr, vk = _proof_vk(e)
    for pt in [pr.proof.a, pr.proof.c, vk.g_alpha, vk.g_gamma] + vk.query:
        assert B.G1.is_on_curve((int(pt.x, 16), int(pt.y, 16)))
    for q in (pr.proof.b, vk.h, vk.h_beta, vk.h_gamma):
        assert B.G2.is_on_curve(((int(q.x[0], 16), int(q.x[1], 16)), (int(q.y[0], 16), int(q.y[1], 16))))
    assert verify_proof_gm17(vk, pr)
    bad = list(e["inputs"])
    bad[0] = "0x%064x" % ((int(bad[0], 16) + 1) % R)
    bad_pr, bad_vk = _proof_vk(e, inputs=bad)
    assert verify_proof_gm17(bad_vk, bad_pr) is False          # a plain rejection: no error may stand in for it
    assert _swapped_rejected(*_proof_vk(e, swap=True))


# ------------------------------------------------------------------------------------------------- Fq2 and points
@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu_wide_377") / "libemu_wide_bls12_377.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-DZKB_EMU", "-shared", "-fPIC", "-I", os.path.join(ROOT, "include"),
                    "-I", CSRC, os.path.join(ROOT, "tests", "host_emu", "emu_wide_bls12_377.cpp"), "-o", out], check=True)
    return Harness(ctypes.CDLL(out), "emu_wide_", False)


@pytest.fixture(scope="module")
def device_lib():
    import __graft_entry__ as g
    assert os.path.exists(g.DEV_WIDE_377_LIB), "tests/host_emu/libdev_wide_bls12_377.so missing: run __graft_entry__.build()"
    return Harness(ctypes.CDLL(g.DEV_WIDE_377_LIB), "dev_wide_", True)


@pytest.fixture(scope="module", params=[pytest.param("host", id="host"),
                                        pytest.param("device", id="device", marks=pytest.mark.gpu)])
def lib(request):
    return request.getfixturevalue(request.param + "_lib")


def test_fp_lazy_ops(lib):
    """mul_wide / sqr_wide / redc / mul_sub of both fields at the edges and on random operands."""
    for fid, p, n in ((0, R, 8), (1, P, 12)):
        Rm = 1 << (32 * n)
        Ri = pow(Rm, -1, p)
        rnd = random.Random(377 + fid)
        K = 2000
        ua = [0, 1, p - 1, p, 2 * p - 1] + [rnd.randrange(2 * p) for _ in range(K)]
        ub = [p - 1, 2 * p - 1, 1, 0, 2 * p - 1] + [rnd.randrange(2 * p) for _ in range(K)]
        z = [0] * len(ua)
        assert lib.fp(fid, 0, n, ua, ub, z, z, 2 * n) == [x * y for x, y in zip(ua, ub)]
        assert lib.fp(fid, 1, n, ua, z, z, z, 2 * n) == [x * x for x in ua]
        t = [0, p * Rm - 1, 12 * (p - 1) ** 2] + [rnd.randrange(p * Rm) for _ in range(K)]
        z = [0] * len(t)
        assert lib.fp(fid, 2, n, t, z, z, z, n) == [x * Ri % p for x in t]
        a, b, c, d = ([p - 1] + [rnd.randrange(p) for _ in range(K)] for _ in range(4))
        assert lib.fp(fid, 4, n, a, b, c, d, n) == [(w * x - y * v) * Ri % p for w, x, y, v in zip(a, b, c, d)]


def test_fq2(lib):
    """mul_v / sqr_v / mul_sub_v of Fq[u]/(u^2 + 5) at the edge table and on 10 000 random cases."""
    n, F = 12, B.F2
    Ri = pow(1 << 384, -1, P)

    def mont_mul(a, b):
        c = F.mul(a, b)
        return (c[0] * Ri % P, c[1] * Ri % P)

    rnd = random.Random(3775)
    edge = [(0, 0), (1, 0), (0, 1), (P - 1, P - 1), (P - 1, 0), (0, P - 1), (1, P - 1)]
    cases = [(a, b, e, f) for a in edge for b in edge for e, f in ((edge[3], edge[3]), ((0, 0), (0, 0)), (edge[5], edge[5]))]
    cases += [tuple((rnd.randrange(P), rnd.randrange(P)) for _ in range(4)) for _ in range(10000)]
    A, Bs, E, Fs = (list(x) for x in zip(*cases))
    assert lib.fp2(CID, 0, n, A, Bs) == [mont_mul(a, b) for a, b in zip(A, Bs)]
    assert lib.fp2(CID, 1, n, A) == [mont_mul(a, a) for a in A]
    assert lib.fp2(CID, 2, n, A, Bs, E, Fs) == [F.sub(mont_mul(a, b), mont_mul(e, f)) for a, b, e, f in cases]
    # inv (norm c0^2 + 5 c1^2): Montgomery image in, Montgomery image out, inv(0) = 0; edges with c0 = 0 and c1 = 0
    Rm = 1 << 384

    def mont_inv(a):
        if a == (0, 0):
            return (0, 0)
        x = F.inv((a[0] * Ri % P, a[1] * Ri % P))
        return (x[0] * Rm % P, x[1] * Rm % P)

    inv_cases = edge + [(0, rnd.randrange(1, P)) for _ in range(50)] + [(rnd.randrange(1, P), 0) for _ in range(50)]
    inv_cases += [(rnd.randrange(P), rnd.randrange(P)) for _ in range(10000)]
    assert lib.fp2(CID, 3, n, inv_cases) == [mont_inv(a) for a in inv_cases]


def test_fq2_host_tail(host_lib):
    """The prover's serial host tail (fp64.cuh: Fp2T over Fp64, every product reduced): mul_v, sqr_v, inv for u^2 = -5."""
    n, F = 12, B.F2
    Rm = 1 << 384
    Ri = pow(Rm, -1, P)

    def mont_mul(a, b):
        c = F.mul(a, b)
        return (c[0] * Ri % P, c[1] * Ri % P)

    def mont_inv(a):
        if a == (0, 0):
            return (0, 0)
        x = F.inv((a[0] * Ri % P, a[1] * Ri % P))
        return (x[0] * Rm % P, x[1] * Rm % P)

    rnd = random.Random(3776)
    edge = [(0, 0), (1, 0), (0, 1), (P - 1, P - 1), (P - 1, 0), (0, P - 1), (1, P - 1)]
    A = edge * len(edge) + [(rnd.randrange(P), rnd.randrange(P)) for _ in range(5000)]
    Bs = [b for b in edge for _ in edge] + [(rnd.randrange(P), rnd.randrange(P)) for _ in range(5000)]
    assert host_lib.fp2(CID, 4, n, A, Bs) == [mont_mul(a, b) for a, b in zip(A, Bs)]
    assert host_lib.fp2(CID, 5, n, A) == [mont_mul(a, a) for a in A]
    assert host_lib.fp2(CID, 6, n, A) == [mont_inv(a) for a in A]


def _group_cases(lib, group):
    G = B.G1 if group == 1 else B.G2
    F = G.F
    Rm = 1 << 384
    Ri = pow(Rm, -1, P)
    gen = B.C.g1 if group == 1 else B.C.g2
    rnd = random.Random(37700 + group)

    def mont(x):
        return x * Rm % P if group == 1 else (x[0] * Rm % P, x[1] * Rm % P)

    def unmont(x):
        return x * Ri % P if group == 1 else (x[0] * Ri % P, x[1] * Ri % P)

    def to_xyzz(pt, z):
        if pt is None:
            return [F.zero] * 4
        zz, zzz = F.sqr(z), F.mul(F.sqr(z), z)
        return [mont(F.mul(pt[0], zz)), mont(F.mul(pt[1], zzz)), mont(zz), mont(zzz)]

    def from_xyzz(r):
        x, y, zz, zzz = (unmont(v) for v in r)
        if F.is_zero(zz):
            return None
        return (F.mul(x, F.inv(zz)), F.mul(y, F.inv(zzz)))

    def rand_z():
        return rnd.randrange(1, P) if group == 1 else (rnd.randrange(P), rnd.randrange(1, P))

    pts = [G.mul(gen, rnd.randrange(1, R)) for _ in range(6)]
    cases = []
    for pt in pts:
        cases += [(pt, q) for q in pts[:3]] + [(pt, pt), (pt, G.neg(pt)), (None, pt), (pt, None)]
    accs = [to_xyzz(p_, rand_z()) for p_, _ in cases]
    q_aff = [[F.zero, F.zero] if q is None else [mont(q[0]), mont(q[1])] for _, q in cases]
    q_xyzz = [to_xyzz(q, rand_z()) for _, q in cases]
    got_madd = ec_call(lib, CID, group, 0, accs, q_aff, 12)
    got_add = ec_call(lib, CID, group, 1, accs, q_xyzz, 12)
    for (p_, q), gm, ga in zip(cases, got_madd, got_add):
        want = G.add(p_, q)
        assert from_xyzz(gm) == want, ("madd", p_, q)
        assert from_xyzz(ga) == want, ("add", p_, q)


def test_g1_additions(lib):
    """XYZZ madd / add: generic, doubling, inverse (identity result), identity accumulator, point at infinity."""
    _group_cases(lib, 1)


def test_g2_additions(lib):
    _group_cases(lib, 2)


# ------------------------------------------------------------------------------------------------- host emulation
def _field_42_prog():
    """zokrates_ark/src/groth16.rs `verify_bls12_377_field`: one constraint _0 * ~one == ~out_0, public input 42."""
    V = ir.Variable
    return ir.Prog([ir.Parameter.public(V.new(0))], 1, [ir.constraint(V.new(0), ir.LinComb.one(), V.public(0))], "bls12_377")


def test_verify_bls12_377_field_groth16(emu_lib):
    prog = _field_42_prog()
    witness = ir.Interpreter().execute(prog, [42])
    td = [11, 22, 33, 44, 55555, 3, 7]
    kp = backend.B200.setup(prog, td, lib=emu_lib)
    proof = backend.B200.generate_proof(prog, witness, io.BytesIO(kp.pk), prng.get_rng_from_entropy("f42"), lib=emu_lib)
    assert proof.curve == "bls12_377" and proof.input_values() == [42, 42]
    assert verify_proof(kp.vk, proof)
    bad = Proof.from_raw(BLS12_377, proof.to_raw(), [42, 43])
    assert not verify_proof(kp.vk, bad)
    # key bytes and proof against the test reference
    from zokrates_b200 import r1cs as pr1cs
    r1 = pr1cs.synthesize(prog)
    o = B.to_oracle(r1)
    assert kp.pk == ark.pk_serialize(B.C, B.setup(o, ark.Trapdoor(*td)))
    orng = ark.rng_from_entropy("f42")
    r, s = ark.fr_rand(B.C, orng), ark.fr_rand(B.C, orng)
    assert proof.to_raw() == proof_bytes(B.C, B.expected_proof(o, ark.Trapdoor(*td), fr_from_array(r1.assignment(witness)), r, s))


def test_verify_bls12_377_field_gm17(emu_lib):
    prog = _field_42_prog()
    witness = ir.Interpreter().execute(prog, [42])
    td = gm17.Gm17Trapdoor(3, 5, 7, 1234567, 11, 13)
    pk = backend.B200.setup_gm17(prog, [td.alpha, td.beta, td.gamma, td.tau, td.g1_k, td.g2_k], lib=emu_lib)
    from zokrates_b200 import r1cs as pr1cs
    r1 = pr1cs.synthesize(prog)
    o = B.to_oracle(r1)
    assert pk == gm17.pk_serialize(B.C, B.gm17_setup(o, td))
    proof = backend.B200.generate_proof_gm17(prog, witness, io.BytesIO(pk), prng.get_rng_from_entropy("g42"), lib=emu_lib)
    orng = ark.rng_from_entropy("g42")
    d1, d2, r = ark.fr_rand(B.C, orng), ark.fr_rand(B.C, orng), ark.fr_rand(B.C, orng)
    z = fr_from_array(r1.assignment(witness))
    assert proof.to_raw() == proof_bytes(B.C, B.gm17_expected_proof(o, td, z, d1, d2, r))
    vk = gm17_vk_from_pk_bytes(BLS12_377, pk)
    assert verify_proof_gm17(vk, proof)
    assert not verify_proof_gm17(vk, Proof.from_raw(BLS12_377, proof.to_raw(), [42, 41], scheme="gm17"))


def test_synthetic_2p10_emulated(emu_lib):
    """A 2^10-domain circuit through the host emulation: the proof equals the python prover's bytes over the emulated key
    and the trapdoor prediction; the witness map equals the oracle's."""
    ctx = Context(CID, 0, emu_lib)
    r1, z = synthetic.make("bls12_377", 1000)
    h = ctx.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())
    td = [3, 5, 7, 11, 1234567, 17, 19]
    pk = ctx.setup(h, td)
    proof = ctx.prove(ctx.pk_load(pk), h, z, 1234, 5678)
    o, zz = B.to_oracle(r1), fr_from_array(z)
    exp = B.expected_proof_csr(r1, ark.Trapdoor(*td), z, 1234, 5678)
    assert proof == exp
    assert fr_from_array(ctx.witness_map(h, z, r1.domain_size)) == ark.witness_map(B.C, o, zz)
    assert proof == proof_bytes(B.C, B.expected_proof(o, ark.Trapdoor(*td), zz, 1234, 5678))
    ctx.close()


def test_curve_id_accepted_and_sizes(emu_lib):
    assert emu_lib.curve_sizes(CID)[:3] == [32, 48, 384]
    ctx = Context(CID, 0, emu_lib)
    assert (ctx.fr_bytes, ctx.fq_bytes, ctx.proof_bytes) == (32, 48, 384)
    ctx.close()
