"""GM17 (SURVEY.md §8 row f3) above the NTT tile threshold, up to the 2^21 SAP domain of the benchmark circuit, against
independent answers:

  * `zko_gm17_trapdoor_expected` (oracle/zkoracle.c): the proof predicted from the setup trapdoor with Fr arithmetic alone
    (closed-form Lagrange coefficients over the SAP domain, per-row sums, three generator multiplications — no NTT, no MSM,
    no key).  It and `zko_gm17_sap_at_tau` are checked byte for byte against oracle/gm17.py here first.
  * BLS12-377 (no C oracle): tests/bls12_377_ref.py's prediction, the same restatement with that curve's groups.
  * A crafted proving key whose points are known multiples of the generator (tests/test_gpu_exceptional.py's pool), so the
    expected proof follows from the discrete logs and gm17.witness_map's h coefficients; its tail sums are P + P and P + (-P).
  * The pairing equations of zokrates_b200.verify.verify_proof_gm17 under the key's own verifying key.

The SAP of an N-constraint circuit with ni instance variables has 2N + 2(ni - 1) + 1 rows, so a circuit of 2^k - 2
constraints and ni = 2 fills a domain of 2^(k+1) but one row, and 2^(k-2) - 1 constraints leave almost half of a 2^k domain
as padding.  The CPU tier runs the kernel sources through the host emulation (domains 2^11 - 2^13); `-m gpu` runs the
product library on the device (2^14 - 2^21).  Nothing here reads the reference project."""
import random

import numpy as np
import pytest

from oracle import gm17
from oracle.ff import BLS12_381, BN254
from tests import bls12_377_ref as B
from tests.test_gpu_exceptional import K, Pool, adversarial_z
from tests.util import csr_from_rows, proof_bytes
from zokrates_b200 import synthetic
from zokrates_b200._lib import (OPT_BATCH_AFFINE, OPT_BATCH_AFFINE_MIN_LOG, OPT_BITSUM_RADIX, OPT_NTT_KERNEL, Context,
                                ZkbError, fr_array, fr_from_array)
from zokrates_b200.curves import curve as pcurve
from zokrates_b200.proof import Proof, gm17_vk_from_pk_bytes
from zokrates_b200.r1cs import R1CS
from zokrates_b200.verify import verify_proof_gm17

OPT_CHUNK_TARGET = 13                              # include/zkb.h ZKB_OPT_CHUNK_TARGET
CURVES = [(0, BN254), (1, BLS12_381)]
TD6 = [3, 5, 7, 1234567, 11, 13]                   # alpha, beta, gamma, tau, g1_k, g2_k
TD7 = [3, 5, 7, 11, 1234567, 17, 19]               # a Groth16 trapdoor for the interleaving checks
R, S = 1234567, 7654321
ZKB_E_ARG = 1


# ---- circuits, assignments and masks ---------------------------------------------------------------------------------
def sap_log(r1):
    rows = 2 * r1.num_constraints + 2 * (r1.num_instance - 1) + 1
    return (rows - 1).bit_length()


def relabel(r1, ni):
    """The same matrices with the first ni variables public (the SAP gains 2(ni - 1) rows and ni - 1 variables)."""
    return R1CS(r1.curve, r1.num_constraints, ni, r1.num_variables - ni, r1.a, r1.b, r1.c)


def adversarial_circuit(c, n_cons, ni, seed):
    """Inputs (the public ones first) cycle through 0, 1, r - 1, one repeated value and uniform values, so y_j = 1, 0, 4, ...;
    rows cycle through squares and (u + v)(v + u) (A z = B z, so x_i = 0), products with the coefficient r - 1, and copies
    (B = 1, repeated values).  Returns the product R1CS and its satisfying assignment."""
    r = c.r
    rnd = random.Random(seed)
    rep = rnd.randrange(r)
    m0 = ni + 6
    z = [1] + [[0, 1, r - 1, rep, None][(j - 1) % 5] for j in range(1, m0)]
    z = [rnd.randrange(r) if v is None else v for v in z]
    rows = ([], [], [])
    for i in range(n_cons):
        w = m0 + i
        u, v = rnd.randrange(w), rnd.randrange(w)
        a, b = [([(u, 1)], [(u, 1)]), ([(u, 1), (v, 1)], [(v, 1), (u, 1)]), ([(u, r - 1)], [(v, 1)]), ([(u, 1)], [(0, 1)])][i % 4]
        z.append(sum(k * z[j] for j, k in a) * sum(k * z[j] for j, k in b) % r)
        rows[0].append(a); rows[1].append(b); rows[2].append([(w, 1)])
    r1 = R1CS(c.name, n_cons, ni, m0 + n_cons - ni, *(csr_from_rows(m, r) for m in rows))
    return r1, fr_array(z)


def circuit(ctx, c, kind, log_n, dist):
    """kind: "least" (rows = n - 1), "most" (rows = n/2 + 1), "ni1" (ni = 1), "ni1025" (ni = 1025: the extra rows alone need
    more than 2^11 points) at a SAP domain of 2^log_n; dist "uniform", "bits" or "adversarial"."""
    n_cons = {"least": (1 << (log_n - 1)) - 2, "most": (1 << (log_n - 2)) - 1, "ni1": (1 << (log_n - 1)) - 2,
              "ni1025": (1 << (log_n - 2)) - 2}[kind]
    ni = {"ni1": 1, "ni1025": 1025}.get(kind, 2)
    if dist == "adversarial":
        r1, z = adversarial_circuit(c, n_cons, ni, seed=log_n)
    else:
        r1, z = synthetic.make_layered(ctx, c.name, n_cons, distribution=dist)
        r1 = relabel(r1, ni)
    assert sap_log(r1) == log_n, (kind, log_n, sap_log(r1))
    return r1, z


def mask_cases(c, seed):
    """(d1, d2, r): all zero; d1 = 0; d2 = 0; r = -d1 (the terms scaled by r + d1 vanish); random."""
    rnd = random.Random(seed)
    d1, d2, r = (rnd.randrange(1, c.r) for _ in range(3))
    return {"zero": (0, 0, 0), "d1=0": (0, d2, r), "d2=0": (d1, 0, r), "r=-d1": (d1, d2, c.r - d1), "random": (d1, d2, r)}


def load(ctx, r1):
    return ctx.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())


def predict(oracle_c, cid, c, r1, z, masks):
    return oracle_c.gm17_trapdoor_expected(cid, r1, TD6, z, *masks, c.fq_bytes)


def verifies(c, pk, raw, r1, z):
    pc = pcurve(c.name)
    pub = fr_from_array(z[1:r1.num_instance]) if r1.num_instance > 1 else []
    return verify_proof_gm17(gm17_vk_from_pk_bytes(pc, pk), Proof.from_raw(pc, raw, pub, scheme="gm17"))


def setup_and_prove(ctx, r1, z, want, masks):
    """Device setup, then one proof per mask case, each equal to want(masks).  Returns (key bytes, r1cs handle, pk handle)."""
    rh = load(ctx, r1)
    pk = ctx.gm17_setup(rh, TD6)
    pkh = ctx.gm17_pk_load(pk)
    for name, m in masks.items():
        assert ctx.gm17_prove(pkh, rh, z, *m) == want(m), name
    return pk, rh, pkh


# ---- the crafted key -------------------------------------------------------------------------------------------------
GGZ, GAB = 21, 22                                  # dlogs of g_gamma_z / h_gamma_z and g_ab_gamma_z


class CraftedGm17:
    """A GM17 proving key (ark's serialize_unchecked layout) for r1 whose every section is tiled from the pool by numpy index
    (runs of one point, (P, -P) pairs, runs of infinity), and the proof expected from the discrete logs with the SAP assignment
    and h coefficients of gm17.witness_map.  `tail` steers the last addition of each proof element: "double" makes it P + P,
    "cancel" P + (-P), so A, B and C are the point at infinity; None leaves it generic.  The key loads because
    zkb_gm17_pk_load checks lengths only."""

    def __init__(self, pool, r1, z, masks, tail, seed):
        c = pool.c
        q = c.r
        d1, d2, r = masks
        ni, m, N = r1.num_instance, r1.num_variables, r1.num_constraints
        nv = m + N + ni - 1
        n = 1 << sap_log(r1)
        full, h = gm17.witness_map(c, B.to_oracle(r1), fr_from_array(z), d1, d2)
        s, hs = fr_array(full), fr_array(h)
        rng = np.random.default_rng(seed)
        t = np.arange(nv)
        pair = (t // 2) % 8 + 8 * (t % 2)
        ia = np.where(t < nv // 4, pair, np.where((t // 64) % 3 == 0, K, (t // 64) % K))
        ib = np.where((t // 1000) % 4 == 1, K, (t // 16) % K)
        i1 = np.where(t[:nv - ni] % 5 == 0, pair[:nv - ni], (t[:nv - ni] // 128) % (K + 1))
        i2 = rng.integers(0, K + 1, nv)
        th = np.arange(n + 1)
        ih = np.where((th // 512) % 2 == 0, (th // 32) % K, rng.integers(0, K + 1, n + 1))
        dl = pool.dlog_sum
        x_a = ((r + d1) * GGZ + dl(ia[1:], s[1:])) % q
        x_b = ((r + d1) * GGZ + dl(ib[1:], s[1:])) % q
        k2 = (r * r + 2 * r * d1) % q
        s_h = dl(ih, hs)
        c_rest = (dl(i1, s[ni:]) + (r + d1) * GAB + r * (pool.dlog[i2[0]] + dl(i2[1:], s[1:])) + d2 * pool.dlog[ih[0]]) % q
        if tail is None:
            a0, b0, g2z2 = pool.dlog[ia[0]], pool.dlog[ib[0]], 23
        else:
            sign = 1 if tail == "double" else -1
            assert k2 and s_h and x_a and x_b
            a0, b0 = sign * x_a % q, sign * x_b % q
            g2z2 = (sign * s_h - c_rest) * pow(k2, -1, q) % q
        P = pool.point
        vec = lambda k: int(k).to_bytes(8, "little")            # noqa: E731
        self.pk = b"".join([P(2, 1), P(1, 3), P(2, 5), P(1, 7), P(2, 7), vec(ni), pool.points(1, np.arange(ni) % K),
                            vec(nv), P(1, a0), pool.points(1, ia[1:]), vec(nv), P(2, b0), pool.points(2, ib[1:]),
                            vec(nv - ni), pool.points(1, i1), vec(nv), pool.points(1, i2), P(1, GGZ), P(2, GGZ), P(1, GAB),
                            P(1, g2z2), vec(n + 1), pool.points(1, ih)])
        self.expected = P(1, x_a + a0) + P(2, x_b + b0) + P(1, c_rest + k2 * g2z2 + s_h)
        if tail == "cancel":
            assert self.expected == ark_infinity(c)


def ark_infinity(c):
    from oracle import ark
    return ark.ser_g1(c, None) + ark.ser_g2(c, None) + ark.ser_g1(c, None)


def check_crafted(ctx, c, r1, seed):
    """The crafted key under random masks with a generic tail, P + P and P + (-P) tails, and all-zero masks."""
    pool = Pool(c, seed)
    z = adversarial_z(c, r1.num_variables, seed)
    rh = load(ctx, r1)
    masks = mask_cases(c, seed)
    for tail, m in ((None, masks["random"]), ("double", masks["random"]), ("cancel", masks["d2=0"]), (None, masks["zero"])):
        cr = CraftedGm17(pool, r1, z, m, tail, seed)
        pkh = ctx.gm17_pk_load(cr.pk)
        assert ctx.gm17_prove(pkh, rh, z, *m) == cr.expected, tail
        ctx.gm17_pk_free(pkh)
    ctx.r1cs_free(rh)


# ---- CPU tier: the C oracle against oracle/gm17.py -------------------------------------------------------------------
def _prog_case(c, cname, shape, seed):
    from oracle import ark, ir as oir
    from tests.util import rand_prog_pair
    oprog, _, inputs = rand_prog_pair(c, *shape, seed=seed, curve_name=cname)
    r1o, z = ark.synthesize(oprog, oir.execute(c, oprog, inputs))
    r1 = R1CS(c.name, r1o.num_constraints, r1o.num_instance, r1o.num_witness, *(csr_from_rows(m, c.r) for m in (r1o.a, r1o.b, r1o.c)))
    return r1, fr_array(z)


ORACLE_CASES = [(cid, c, shape) for cid, c in CURVES for shape in ((5, 1, 2), (1, 1, 1), (7, 2, 1), (4, 1, 1), (40, 2, 3), (300, 2, 3))]
ORACLE_CASES += [(cid, c, kind) for cid, c in CURVES for kind in ("synthetic-2^11", "ni1025")]


@pytest.mark.parametrize("cid,c,shape", ORACLE_CASES, ids=[f"{c.name}-{s}" for _, c, s in ORACLE_CASES])
def test_c_oracle_vs_python(oracle_c, cid, c, shape):
    """zko_gm17_sap_at_tau and zko_gm17_trapdoor_expected equal oracle/gm17.py byte for byte: the random programs of
    tests/test_gm17.py, a synthetic circuit with a 2^11 SAP domain, and one with 1025 instance variables (2^12), under every
    mask case.  A tau inside the domain is refused."""
    if isinstance(shape, tuple):
        r1, z = _prog_case(c, c.name, shape, seed=2)
    elif shape == "ni1025":
        r1, z = adversarial_circuit(c, 1022, 1025, seed=3)
    else:
        r1, z = synthetic.make(c.name, (1 << 10) - 2)
    r1o, zi = B.to_oracle(r1), fr_from_array(z)
    td = gm17.Gm17Trapdoor(*TD6)
    d, a, cc, zt = gm17.sap_at_tau(c, r1o, td.tau)
    ga, gc, gzt = oracle_c.gm17_sap_at_tau(cid, r1, td.tau)
    assert fr_from_array(ga) == a and fr_from_array(gc) == cc and gzt == zt
    for name, m in mask_cases(c, len(zi)).items():
        assert predict(oracle_c, cid, c, r1, z, m) == proof_bytes(c, gm17.trapdoor_expected_proof(c, r1o, td, zi, *m)), name
    with pytest.raises(RuntimeError, match="rc=3"):
        oracle_c.gm17_trapdoor_expected(cid, r1, TD6[:3] + [d.omega] + TD6[4:], z, 1, 2, 3, c.fq_bytes)


# ---- CPU tier: the host emulation ------------------------------------------------------------------------------------
EMU_SHAPES = [(0, BN254, "least", 11, "adversarial"), (0, BN254, "most", 12, "bits"), (0, BN254, "least", 13, "uniform"),
              (0, BN254, "ni1", 12, "uniform"), (0, BN254, "ni1025", 12, "bits"),
              (1, BLS12_381, "least", 11, "uniform"), (1, BLS12_381, "most", 13, "adversarial")]


@pytest.mark.parametrize("cid,c,kind,log_n,dist", EMU_SHAPES, ids=[f"{c.name}-{k}-2^{g}-{d}" for _, c, k, g, d in EMU_SHAPES])
def test_emu_setup_and_prove(emu_lib, oracle_c, cid, c, kind, log_n, dist):
    """Emulated device setup and proofs above the tile threshold: every mask case gives the trapdoor-predicted bytes, and the
    random-mask proof passes both pairing equations under the key's own verifying key."""
    ctx = Context(cid, 0, emu_lib)
    r1, z = circuit(ctx, c, kind, log_n, dist)
    masks = mask_cases(c, log_n)
    pk, rh, pkh = setup_and_prove(ctx, r1, z, lambda m: predict(oracle_c, cid, c, r1, z, m), masks)
    assert verifies(c, pk, ctx.gm17_prove(pkh, rh, z, *masks["random"]), r1, z)
    ctx.close()


def test_emu_bls12_377(emu_lib):
    """BLS12-377 at a 2^11 SAP domain (adversarial assignment, 3 public inputs) against tests/bls12_377_ref.py's prediction."""
    ctx = Context(2, 0, emu_lib)
    r1, z = adversarial_circuit(B.C, (1 << 10) - 4, 3, seed=7)
    assert sap_log(r1) == 11
    r1o, zi, td = B.to_oracle(r1), fr_from_array(z), gm17.Gm17Trapdoor(*TD6)
    masks = mask_cases(B.C, 377)
    del masks["d1=0"], masks["d2=0"]
    pk, rh, pkh = setup_and_prove(ctx, r1, z, lambda m: proof_bytes(B.C, B.gm17_expected_proof(r1o, td, zi, *m)), masks)
    assert verifies(B.C, pk, ctx.gm17_prove(pkh, rh, z, *masks["random"]), r1, z)
    ctx.close()


@pytest.fixture(scope="module")
def emu_bn(emu_lib):
    """A BN254 context with a 2^11-domain circuit, its GM17 key loaded and a Groth16 key for the same circuit."""
    ctx = Context(0, 0, emu_lib)
    r1, z = circuit(ctx, BN254, "least", 11, "uniform")
    rh = load(ctx, r1)
    pk = ctx.gm17_setup(rh, TD6)
    yield ctx, r1, z, rh, pk, ctx.gm17_pk_load(pk), ctx.pk_load(ctx.setup(rh, TD7))
    ctx.close()


def test_emu_resident_assignment(emu_bn, oracle_c):
    """gm17_prove with z = NULL reads the assignment set by zkb_r1cs_set_assignment; without one the call is refused."""
    ctx, r1, z, rh, pk, pkh, _ = emu_bn
    fresh = load(ctx, r1)
    with pytest.raises(ZkbError, match="no resident assignment") as e:
        ctx.gm17_prove(pkh, fresh, None, 1, 2, 3)
    assert e.value.code == ZKB_E_ARG
    ctx.set_assignment(fresh, z)
    for m in mask_cases(BN254, 5).values():
        assert ctx.gm17_prove(pkh, fresh, None, *m) == ctx.gm17_prove(pkh, rh, z, *m) == predict(oracle_c, 0, BN254, r1, z, m)
    ctx.r1cs_free(fresh)


def test_emu_refusals(emu_bn, oracle_c):
    """ZKB_E_ARG for: a key of a circuit with the same SAP variable count but another domain, a key whose ni differs, an
    unknown handle, and a proof requested while a Groth16 proof is in flight (whose ticket still collects to its own bytes)."""
    ctx, r1, z, rh, pk, pkh, g16 = emu_bn
    N2 = 300                                               # the first 300 rows, the variable count padded to the same nv
    cut = [(rp[:N2 + 1], col[:int(rp[N2])], val[:int(rp[N2])]) for rp, col, val in r1.matrices()]
    small = R1CS(r1.curve, N2, r1.num_instance, r1.num_witness + r1.num_constraints - N2, *cut)
    assert sap_log(small) < sap_log(r1)
    sh = load(ctx, small)
    zs = np.zeros((small.num_variables, 4), np.uint64)
    with pytest.raises(ZkbError, match="domain size") as e:
        ctx.gm17_prove(pkh, sh, zs, 1, 2, 3)
    assert e.value.code == ZKB_E_ARG
    other = load(ctx, relabel(r1, 3))
    with pytest.raises(ZkbError, match="variable counts") as e:
        ctx.gm17_prove(pkh, other, z, 1, 2, 3)
    assert e.value.code == ZKB_E_ARG
    with pytest.raises(ZkbError, match="unknown gm17 pk handle") as e:
        ctx.gm17_prove(pkh + 1000, rh, z, 1, 2, 3)
    assert e.value.code == ZKB_E_ARG
    ticket = ctx.prove_submit(g16, rh, z, R, S)
    with pytest.raises(ZkbError, match="in flight") as e:
        ctx.gm17_prove(pkh, rh, z, 1, 2, 3)
    assert e.value.code == ZKB_E_ARG
    assert ctx.prove_collect(ticket) == oracle_c.trapdoor_expected(0, r1, TD7, z, R, S, BN254.fq_bytes)
    assert ctx.gm17_prove(pkh, rh, z, 1, 2, 3) == predict(oracle_c, 0, BN254, r1, z, (1, 2, 3))
    ctx.r1cs_free(sh)
    ctx.r1cs_free(other)


def key_sections(c, pk):
    """The sections of a GM17 key in ark's serialize_unchecked order: (name, group, bytes) per element or vector."""
    g1b, g2b = 2 * c.fq_bytes, 4 * c.fq_bytes
    layout = [("h_g2", 2, 0), ("g_alpha_g1", 1, 0), ("h_beta_g2", 2, 0), ("g_gamma_g1", 1, 0), ("h_gamma_g2", 2, 0),
              ("query", 1, 1), ("a_query", 1, 1), ("b_query", 2, 1), ("c_query_1", 1, 1), ("c_query_2", 1, 1),
              ("g_gamma_z", 1, 0), ("h_gamma_z", 2, 0), ("g_ab_gamma_z", 1, 0), ("g_gamma2_z2", 1, 0), ("g_gamma2_z_t", 1, 1)]
    out, off = {}, 0
    for name, g, is_vec in layout:
        cnt = 1
        if is_vec:
            cnt = int.from_bytes(pk[off:off + 8], "little")
            off += 8
        size = cnt * (g1b if g == 1 else g2b)
        out[name] = (g, pk[off:off + size])
        off += size
    assert off == len(pk)
    return out


def interleave(ctx, oracle_c, cid, c, r1, z, rh, g16, gm17_pk):
    """Groth16 proof, GM17 setup, GM17 proof, a standalone G1 MSM and a Groth16 proof again on one context: the two schemes
    share the misc MSM plan, its window buffer and the setup scratch."""
    g16_want = oracle_c.trapdoor_expected(cid, r1, TD7, z, R, S, c.fq_bytes)
    assert ctx.prove(g16, rh, z, R, S) == g16_want
    assert ctx.gm17_setup(rh, TD6) == gm17_pk
    pkh = ctx.gm17_pk_load(gm17_pk)
    m = mask_cases(c, 9)["random"]
    assert ctx.gm17_prove(pkh, rh, z, *m) == predict(oracle_c, cid, c, r1, z, m)
    ctx.gm17_pk_free(pkh)
    pts = key_sections(c, gm17_pk)["c_query_2"][1]
    sc = fr_array([random.Random(cid).randrange(c.r) for _ in range(len(pts) // (2 * c.fq_bytes))])
    assert ctx.msm(1, pts, sc) == oracle_c.msm(cid, 1, pts, sc, c.fq_bytes)
    assert ctx.prove(g16, rh, z, R, S) == g16_want


def test_emu_interleaved_with_groth16(emu_bn, oracle_c):
    ctx, r1, z, rh, pk, pkh, g16 = emu_bn
    interleave(ctx, oracle_c, 0, BN254, r1, z, rh, g16, pk)


@pytest.mark.parametrize("cid,c", CURVES, ids=[c.name for _, c in CURVES])
def test_emu_crafted_key(emu_lib, cid, c):
    """The crafted key of a 2^11-domain circuit with the adversarial assignment of tests/test_gpu_exceptional.py."""
    ctx = Context(cid, 0, emu_lib)
    r1, _ = synthetic.make_layered(ctx, c.name, (1 << 10) - 2)
    check_crafted(ctx, c, r1, seed=11 + cid)
    ctx.close()


# ---- GPU tier --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_bench_circuit_2_21(gpu_lib, oracle_c):
    """The benchmark circuit (2^20 - 2 constraints) under GM17: a 2^21 SAP domain.  Device setup and proof equal the trapdoor
    prediction, with the assignment passed and resident; the proof passes both pairing equations and fails with another
    public input."""
    ctx = Context(0, 0, gpu_lib)
    try:
        r1, z = synthetic.make_layered(ctx, "bn128", (1 << 20) - 2)
        assert sap_log(r1) == 21
        rh = load(ctx, r1)
        pk = ctx.gm17_setup(rh, TD6)
        pkh = ctx.gm17_pk_load(pk)
        m = mask_cases(BN254, 21)["random"]
        want = predict(oracle_c, 0, BN254, r1, z, m)
        assert ctx.gm17_prove(pkh, rh, z, *m) == want
        ctx.set_assignment(rh, z)
        assert ctx.gm17_prove(pkh, rh, None, *m) == want
        assert verifies(BN254, pk, want, r1, z)
        bad = z.copy()
        bad[1, 0] ^= np.uint64(1)
        assert not verifies(BN254, pk, want, r1, bad)
    finally:
        ctx.close()


def check_whole_key(ctx, oracle_c, cid, c, r1, pk):
    """Every key section against the trapdoor: for each vector, sum w_i P_i (the C oracle's MSM) equals (sum w_i e_i) g for
    random Fr weights w, with e_i from zko_gm17_sap_at_tau as in gm17.setup; the single points directly."""
    from oracle.ff import g1_group, g2_group
    from oracle import ark
    q = c.r
    alpha, beta, gamma, tau, g1k, g2k = TD6
    ua, wc, zt = oracle_c.gm17_sap_at_tau(cid, r1, tau)
    a, cc = fr_from_array(ua), fr_from_array(wc)
    ni, nv, n = r1.num_instance, len(a), 1 << sap_log(r1)
    ab, g2z = (alpha + beta) % q, gamma * gamma * zt % q
    G = {1: g1_group(c), 2: g2_group(c)}
    gen = {1: G[1].mul(c.g1, g1k), 2: G[2].mul(c.g2, g2k)}
    ser = {1: ark.ser_g1, 2: ark.ser_g2}

    def point(g, k):
        k %= q
        return ser[g](c, G[g].mul(gen[g], k) if k else None)
    powers, tp = [], g2z
    for _ in range(n + 1):
        powers.append(tp)
        tp = tp * tau % q
    want = {"h_g2": 1, "g_alpha_g1": alpha, "h_beta_g2": beta, "g_gamma_g1": gamma, "h_gamma_g2": gamma,
            "query": [(gamma * cc[i] + ab * a[i]) % q for i in range(ni)],
            "a_query": [gamma * x % q for x in a], "b_query": [gamma * x % q for x in a],
            "c_query_1": [(gamma * gamma * cc[i] + ab * gamma * a[i]) % q for i in range(ni, nv)],
            "c_query_2": [2 * g2z * x % q for x in a], "g_gamma_z": gamma * zt, "h_gamma_z": gamma * zt,
            "g_ab_gamma_z": ab * gamma * zt, "g_gamma2_z2": g2z * zt, "g_gamma2_z_t": powers}
    rnd = random.Random(len(pk))
    for name, (g, data) in key_sections(c, pk).items():
        e = want[name]
        if not isinstance(e, list):
            assert data == point(g, e), name
            continue
        w = [rnd.randrange(q) for _ in e]
        assert len(data) == len(e) * (2 if g == 1 else 4) * c.fq_bytes, name
        assert oracle_c.msm(cid, g, data, fr_array(w), c.fq_bytes) == point(g, sum(x * y for x, y in zip(w, e))), name


KEY_CASES = [(cid, c, k) for cid, c in CURVES for k in (16, 18)]


@pytest.mark.gpu
@pytest.mark.parametrize("cid,c,log_n", KEY_CASES, ids=[f"{c.name}-2^{k}" for _, c, k in KEY_CASES])
def test_whole_key_and_masks(gpu_lib, oracle_c, cid, c, log_n):
    """Device setup at SAP domains 2^16 and 2^18 (rows = n - 1) checked section by section, then proofs under the zero, d1 = 0,
    d2 = 0 and r = -d1 masks against the trapdoor prediction."""
    ctx = Context(cid, 0, gpu_lib)
    try:
        r1, z = circuit(ctx, c, "least", log_n, "uniform")
        rh = load(ctx, r1)
        pk = ctx.gm17_setup(rh, TD6)
        check_whole_key(ctx, oracle_c, cid, c, r1, pk)
        pkh = ctx.gm17_pk_load(pk)
        for name, m in mask_cases(c, log_n).items():
            assert ctx.gm17_prove(pkh, rh, z, *m) == predict(oracle_c, cid, c, r1, z, m), name
    finally:
        ctx.close()


GRID = [{OPT_BATCH_AFFINE: ba, OPT_BATCH_AFFINE_MIN_LOG: 0, OPT_BITSUM_RADIX: rad, OPT_CHUNK_TARGET: ct, OPT_NTT_KERNEL: nk}
        for ba in (0, 3) for rad in (2, 8) for ct in (600000, 1000) for nk in (1, 2)]
DEFAULTS = {OPT_BATCH_AFFINE: 0, OPT_BATCH_AFFINE_MIN_LOG: 16, OPT_BITSUM_RADIX: 2, OPT_CHUNK_TARGET: 600000, OPT_NTT_KERNEL: 2}


@pytest.mark.gpu
def test_knob_grid(gpu_lib, oracle_c):
    """One 2^16-domain circuit (adversarial assignment, 3 public inputs): every combination of batch-affine rounds {0, 3},
    bit-sum radix {2, 8}, chunk target {600000, 1000} and NTT tile kernel {1, 2} gives the predicted bytes."""
    ctx = Context(0, 0, gpu_lib)
    try:
        r1, z = adversarial_circuit(BN254, (1 << 15) - 4, 3, seed=16)
        assert sap_log(r1) == 16
        rh = load(ctx, r1)
        pkh = ctx.gm17_pk_load(ctx.gm17_setup(rh, TD6))
        m = mask_cases(BN254, 16)["random"]
        want = predict(oracle_c, 0, BN254, r1, z, m)
        for cfg in GRID:
            for opt, v in cfg.items():
                ctx.set_option(opt, v)
            assert ctx.gm17_prove(pkh, rh, z, *m) == want, cfg
    finally:
        for opt, v in DEFAULTS.items():
            ctx.set_option(opt, v)
        ctx.close()


@pytest.mark.gpu
def test_bls12_377_2_14(gpu_lib):
    """BLS12-377 at a 2^14 SAP domain (bits distribution) against tests/bls12_377_ref.py's prediction, and verified."""
    ctx = Context(2, 0, gpu_lib)
    try:
        r1, z = circuit(ctx, B.C, "least", 14, "bits")
        r1o, zi, td = B.to_oracle(r1), fr_from_array(z), gm17.Gm17Trapdoor(*TD6)
        masks = mask_cases(B.C, 14)
        masks = {k: masks[k] for k in ("zero", "r=-d1", "random")}
        pk, rh, pkh = setup_and_prove(ctx, r1, z, lambda m: proof_bytes(B.C, B.gm17_expected_proof(r1o, td, zi, *m)), masks)
        assert verifies(B.C, pk, ctx.gm17_prove(pkh, rh, z, *masks["random"]), r1, z)
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cid,c", CURVES, ids=[c.name for _, c in CURVES])
def test_crafted_key_2_16(gpu_lib, cid, c):
    ctx = Context(cid, 0, gpu_lib)
    try:
        r1, _ = synthetic.make_layered(ctx, c.name, (1 << 15) - 2)
        assert sap_log(r1) == 16
        check_crafted(ctx, c, r1, seed=21 + cid)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_setup_with_groth16_in_flight(gpu_lib, oracle_c):
    """GM17 setup does not check for in-flight work: run it while a Groth16 proof is submitted on the same context.  The key
    equals a quiet context's, the Groth16 ticket collects to its predicted bytes, and the rest of the interleaving holds."""
    ctx = Context(0, 0, gpu_lib)
    try:
        r1, z = circuit(ctx, BN254, "least", 16, "uniform")
        rh = load(ctx, r1)
        quiet = ctx.gm17_setup(rh, TD6)
        g16 = ctx.pk_load(ctx.setup(rh, TD7))
        ticket = ctx.prove_submit(g16, rh, z, R, S)
        assert ctx.gm17_setup(rh, TD6) == quiet
        assert ctx.prove_collect(ticket) == oracle_c.trapdoor_expected(0, r1, TD7, z, R, S, BN254.fq_bytes)
        interleave(ctx, oracle_c, 0, BN254, r1, z, rh, g16, quiet)
    finally:
        ctx.close()
