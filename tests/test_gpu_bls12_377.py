"""BLS12-377 on the GPU (libzkb200.so, curve id 2): NTTs, standalone G1 / G2 MSMs, the device setup, Groth16 proofs at
2^16 and 2^20 - 2 constraints, GM17, and the program -> witness -> proof path.  The device half of the Fq2 and point-addition
cases is in tests/test_bls12_377.py (its `-device` ids).

Expected values come from Python integers and tests/bls12_377_ref.py: the oracle's Fr-only code (domains, QAP / SAP at tau,
witness maps) with this curve's groups, and trapdoor predictions, which need no NTT, no MSM and no key.  MSM inputs are
drawn from a pool of k·G (random discrete logs, their negatives and infinity), so any expected sum is one scalar
multiplication and the doubling / inverse / identity branches of the Fq2 additions run on the device.  One proof per size
passes the pairing check of zokrates_b200.verify, which the ark GM17 fixture pins for this curve."""
import io

import numpy as np
import pytest

from oracle import ark, gm17
from tests import bls12_377_ref as B
from tests.util import proof_bytes, rand_prog_pair
from zokrates_b200 import backend, ir, proof as pproof, rng as prng, synthetic, zir
from zokrates_b200._lib import (OPT_NTT_KERNEL, OPT_TABLES, Context, ZkbError, fr_array, fr_from_array)
from zokrates_b200.curves import BLS12_377
from zokrates_b200.verify import verify_proof, verify_proof_gm17

pytestmark = pytest.mark.gpu
CID = 2
TD = [3, 5, 7, 11, 1234567, 17, 19]
R_, S_ = 1234567, 7654321


@pytest.fixture(scope="module")
def ctx(gpu_lib):
    c = Context(CID, 0, gpu_lib)
    yield c
    c.close()


def _rand_fr(rs, n):
    sc = rs.randint(0, 1 << 62, size=(n, 4)).astype(np.uint64)
    sc[:, 3] &= np.uint64((1 << 60) - 1)              # < 2^252 < r
    return sc


# ------------------------------------------------------------------------------------------------- NTT
def test_ntt_python_domain(ctx):
    """2^10, all four variants, against oracle/ark.py's Domain with this curve's Fr (the C restatement below is checked
    against the same Domain in tests/test_bls12_377.py)."""
    x = _rand_fr(np.random.RandomState(10), 1 << 10)
    xi = fr_from_array(x)
    d = ark.Domain(B.C, 1 << 10)
    assert fr_from_array(ctx.ntt(x)) == d.fft(xi)
    assert fr_from_array(ctx.ntt(x, inverse=True)) == d.ifft(xi)
    assert fr_from_array(ctx.ntt(x, coset=True)) == d.coset_fft(xi)
    assert fr_from_array(ctx.ntt(x, inverse=True, coset=True)) == d.coset_ifft(xi)


@pytest.mark.parametrize("log_n", list(range(10, 24)))
def test_ntt_four_variants(ctx, log_n):
    """zkb_ntt at 2^10 - 2^23, all four variants, with both tile kernels, against tests/bls12_377_ntt.c."""
    x = _rand_fr(np.random.RandomState(log_n), 1 << log_n)
    try:
        for inverse, coset in ((False, False), (True, False), (False, True), (True, True)):
            want = B.ref_ntt(x, log_n, inverse, coset)
            for kernel in (1, 2):
                ctx.set_option(OPT_NTT_KERNEL, kernel)
                assert np.array_equal(ctx.ntt(x, inverse=inverse, coset=coset), want), (inverse, coset, kernel)
    finally:
        ctx.set_option(OPT_NTT_KERNEL, 2)


def test_ntt_domain_cap(ctx):
    """Fr has 2-adicity 47, but the engine's domains stop at 2^28, as on the other curves."""
    buf = np.zeros((1, 4), dtype=np.uint64)          # the domain is checked before any data is read
    with pytest.raises(ZkbError, match="domain too large"):
        ctx.lib.check(ctx.lib.dll.zkb_ntt(ctx.h, buf.ctypes.data, 29, 0, 0))
    assert fr_from_array(ctx.ntt(np.zeros((1 << 10, 4), dtype=np.uint64))) == [0] * 1024   # the context still works


# ------------------------------------------------------------------------------------------------- MSM
class Pool:
    """k_j·G for 8 random k, their negatives, and infinity (index 16)."""

    def __init__(self, group, seed):
        rs = np.random.RandomState(seed)
        self.G = B.G1 if group == 1 else B.G2
        gen = B.C.g1 if group == 1 else B.C.g2
        ks = [int(v) for v in fr_from_array(_rand_fr(rs, 8))]
        self.k = ks + [(-k) % B.R for k in ks] + [0]
        ser = ark.ser_g1 if group == 1 else ark.ser_g2
        self.gen, self.ser = gen, ser
        self.raw = np.stack([np.frombuffer(ser(B.C, self.G.mul(gen, k) if k else None), dtype=np.uint8) for k in self.k])

    def points(self, idx):
        return self.raw[idx].tobytes()

    def expected(self, idx, scalars):
        s = sum(self.k[i] * v for i, v in zip(idx.tolist(), fr_from_array(scalars))) % B.R
        return self.ser(B.C, self.G.mul(self.gen, s) if s else None)


@pytest.mark.parametrize("group", [1, 2])
@pytest.mark.parametrize("n", [4099, 1 << 16])
def test_msm_pool(ctx, group, n):
    pool = Pool(group, 10 * group + n % 7)
    rs = np.random.RandomState(n)
    cases = []
    idx = rs.randint(0, 17, size=n)
    cases.append((idx, _rand_fr(rs, n)))                                # mixed pool, uniform scalars
    cases.append((np.zeros(n, dtype=np.int64), _rand_fr(rs, n)))        # one point: every bucket sums equal points
    pair = np.arange(n) % 2 * 8 + (np.arange(n) // 2) % 8               # k, -k alternating with equal scalars
    sc = _rand_fr(rs, n)
    sc[1::2] = sc[0:n - 1:2][: len(sc[1::2])]
    cases.append((pair, sc))                                            # cancelling pairs (sum is infinity when n is even)
    ones = fr_array([1 if v else 0 for v in rs.random_sample(n) < 0.9])
    cases.append((idx, ones))                                           # 90 % unit scalars
    for idx_, sc_ in cases:
        assert ctx.msm(group, pool.points(idx_), sc_) == pool.expected(idx_, sc_)


@pytest.mark.parametrize("group", [1, 2])
@pytest.mark.parametrize("n", [1 << 16, 1 << 18])
def test_msm_uniform(ctx, group, n):
    """Standalone G1 and G2 MSMs at 2^16 and 2^18: uniform scalars over the pool."""
    pool = Pool(group, 3 + group)
    rs = np.random.RandomState(7 + n + group)
    idx, sc = rs.randint(0, 16, size=n), _rand_fr(rs, n)
    assert ctx.msm(group, pool.points(idx), sc) == pool.expected(idx, sc)


# ------------------------------------------------------------------------------------------------- setup and proofs
def _check_whole_key(ctx, pk, r1, td):
    """Every point of a GPU-made key against the trapdoor.  Each point is a known multiple k_i of its generator, so each
    vector is checked at once: its points are canonical and on the curve, the point at infinity exactly where k_i = 0, and
    sum rho_i P_i (zkb_msm, checked above against independent answers) equals (sum rho_i k_i) G for random 128-bit rho_i,
    which any wrong point breaks except with probability 2^-128."""
    key = ark.pk_deserialize(B.C, pk)                  # the whole layout, no trailing bytes
    q = B.R
    d, a, b, cc, zt = ark.qap_at_tau(B.C, B.to_oracle(r1), td.tau)
    g1, g2 = B.G1.mul(B.C.g1, td.g1_k), B.G2.mul(B.C.g2, td.g2_k)
    for pt, G, g, k in ((key.alpha_g1, B.G1, g1, td.alpha), (key.beta_g2, B.G2, g2, td.beta), (key.gamma_g2, B.G2, g2, td.gamma),
                        (key.delta_g2, B.G2, g2, td.delta), (key.beta_g1, B.G1, g1, td.beta), (key.delta_g1, B.G1, g1, td.delta)):
        assert pt == G.mul(g, k)
    ginv, dinv = pow(td.gamma, -1, q), pow(td.delta, -1, q)
    m, ni = r1.num_variables, r1.num_instance
    abc = [(td.beta * a[i] + td.alpha * b[i] + cc[i]) % q for i in range(m)]
    hs = [zt * dinv % q * pow(td.tau, j, q) % q for j in range(d.n - 1)]
    vectors = (("gamma_abc", 1, key.gamma_abc_g1, [x * ginv % q for x in abc[:ni]]), ("a", 1, key.a_query, a),
               ("b_g1", 1, key.b_g1_query, b), ("b_g2", 2, key.b_g2_query, b), ("h", 1, key.h_query, hs),
               ("l", 1, key.l_query, [x * dinv % q for x in abc[ni:]]))
    rs = np.random.RandomState(len(pk) & 0xFFFF)
    for name, group, pts, ks in vectors:
        G, g = (B.G1, g1) if group == 1 else (B.G2, g2)
        ser = ark.ser_g1 if group == 1 else ark.ser_g2
        assert len(pts) == len(ks), name
        assert all((pt is None) == (k % q == 0) for pt, k in zip(pts, ks)), name
        assert all(G.is_on_curve(pt) for pt in pts), name
        coords = [c for pt in pts if pt is not None for c in (pt if group == 1 else pt[0] + pt[1])]
        assert all(c < B.P for c in coords), name
        rho = rs.randint(0, 1 << 62, size=(len(pts), 4)).astype(np.uint64)
        rho[:, 2:] = 0
        want = sum(int(x) * k for x, k in zip(fr_from_array(rho), ks)) % q
        got = ctx.msm(group, b"".join(ser(B.C, pt) for pt in pts), rho)
        assert got == ser(B.C, G.mul(g, want) if want else None), name


@pytest.mark.parametrize("n_cons", [13, 1000])
def test_setup_bytes(ctx, n_cons):
    """Keys of a 13-constraint and a 2^10-domain circuit byte for byte against tests/bls12_377_ref.py's setup."""
    r1, _ = synthetic.make("bls12_377", n_cons)
    h = ctx.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())
    assert ctx.setup(h, TD) == ark.pk_serialize(B.C, B.setup(B.to_oracle(r1), ark.Trapdoor(*TD)))
    ctx.r1cs_free(h)


@pytest.mark.parametrize("n_cons", [1000, (1 << 16) - 2])
def test_setup_whole_key(ctx, n_cons):
    r1, _ = synthetic.make_layered(ctx, "bls12_377", n_cons)
    h = ctx.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())
    _check_whole_key(ctx, ctx.setup(h, TD), r1, ark.Trapdoor(*TD))
    ctx.r1cs_free(h)


def _shard_prove(ctx, pk, h, z, world):
    parts = []
    for rank in range(world):
        pkh = ctx.pk_load(pk, rank, world)
        parts.append(ctx.prove_partial(pkh, h, z))
        ctx.pk_free(pkh)
    pkh = ctx.pk_load(pk)
    out = ctx.finalize(pkh, np.concatenate(parts), world, R_, S_)
    ctx.pk_free(pkh)
    return out


@pytest.mark.parametrize("log_n", [16, 20])
@pytest.mark.parametrize("dist", ["uniform", "bits"])
def test_proof_vs_trapdoor(ctx, log_n, dist):
    """2^k - 2 constraints: the proof equals the trapdoor prediction with window tables on and off; one passes the pairing
    check, and a different r gives different bytes."""
    r1, z = synthetic.make_layered(ctx, "bls12_377", (1 << log_n) - 2, distribution=dist)
    h = ctx.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())
    pk = ctx.setup(h, TD)
    expected = B.expected_proof_csr(r1, ark.Trapdoor(*TD), z, R_, S_)
    assert ctx.r1cs_check(h, z) is None
    for tables in (1, 0):
        ctx.set_option(OPT_TABLES, tables)
        pkh = ctx.pk_load(pk)
        assert ctx.prove(pkh, h, z, R_, S_) == expected, f"tables={tables}"
        if tables == 1:
            assert ctx.prove(pkh, h, z, R_ + 1, S_) != expected
        ctx.pk_free(pkh)
    ctx.set_option(OPT_TABLES, 1)
    for world in (3, 8):
        assert _shard_prove(ctx, pk, h, z, world) == expected, f"{world}-way sharded"
    if dist == "uniform":
        vk = pproof.vk_from_pk_bytes(BLS12_377, pk)
        pub = fr_from_array(z[1:r1.num_instance])
        prf = pproof.Proof.from_raw(BLS12_377, expected, pub)
        assert verify_proof(vk, prf)
    ctx.r1cs_free(h)


@pytest.mark.parametrize("ncons", [40, 300])
def test_gm17(gpu_lib, ncons):
    c = B.C
    oprog, pprog, inputs = rand_prog_pair(c, ncons, 2, 3, seed=ncons, curve_name="bls12_377")
    from oracle import ir as oir
    ow = oir.execute(c, oprog, inputs)
    r1cs, z = ark.synthesize(oprog, ow)
    td = gm17.Gm17Trapdoor(3 + ncons, 5, 7, 1234567 + ncons, 11, 13)
    pk_bytes = backend.B200.setup_gm17(pprog, [td.alpha, td.beta, td.gamma, td.tau, td.g1_k, td.g2_k], lib=gpu_lib)
    if ncons == 40:
        assert pk_bytes == gm17.pk_serialize(c, B.gm17_setup(r1cs, td))
    entropy = f"gm17-377-{ncons}"
    orng = ark.rng_from_entropy(entropy)
    d1, d2, r = ark.fr_rand(c, orng), ark.fr_rand(c, orng), ark.fr_rand(c, orng)
    pw = ir.Interpreter().execute(pprog, inputs)
    prf = backend.B200.generate_proof_gm17(pprog, pw, io.BytesIO(pk_bytes), prng.get_rng_from_entropy(entropy), lib=gpu_lib)
    assert prf.to_raw() == proof_bytes(c, B.gm17_expected_proof(r1cs, td, z, d1, d2, r))
    vk = pproof.gm17_vk_from_pk_bytes(BLS12_377, pk_bytes)
    assert verify_proof_gm17(vk, prf)
    pub = prf.input_values()
    assert not verify_proof_gm17(vk, pproof.Proof.from_raw(BLS12_377, prf.to_raw(), [(pub[0] + 1) % c.r] + pub[1:], scheme="gm17"))


def test_program_file_path(gpu_lib, ctx):
    """`out` file with the c2955ab5 header -> device witness -> proof; a bn128 program is refused by a BLS12-377 context."""
    V = ir.Variable
    x, y, t = V.new(0), V.new(1), V.new(2)
    prog = ir.Prog([ir.Parameter.private_(x), ir.Parameter.public(y)], 1, [
        ir.constraint(x, y, t),
        ir.Constraint(ir.QuadComb(ir.LinComb([(t, 1), (x, 5)]), ir.LinComb.one()), ir.LinComb.from_var(V.public(0)))],
        "bls12_377")
    data = zir.write_prog(prog)
    assert data[8:12].hex() == "c2955ab5"
    ph = ctx.prog_load(data)
    want = ir.Interpreter().execute(prog, [6, 7])
    assert ctx.prog_compute_witness(ph, [6, 7]) == want.write()
    ctx.prog_free(ph)
    kp = backend.B200.setup(prog, TD, lib=gpu_lib)
    prf = backend.B200.generate_proof_files(data, want.write(), io.BytesIO(kp.pk), prng.get_rng_from_entropy("file"),
                                            curve="bls12_377", lib=gpu_lib)
    assert prf.input_values() == [7, 6 * 7 + 5 * 6]
    assert verify_proof(kp.vk, prf)
    prog.curve = "bn128"
    with pytest.raises(ZkbError, match="another curve"):
        ctx.prog_load(zir.write_prog(prog))
