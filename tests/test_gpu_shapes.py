"""GPU tier (-m gpu): every NTT tile-pass shape, standalone MSMs above 2^20 and the 2^21 / 2^22 proofs, each against an
independent answer.

  * NTT, decimation in frequency (`zkb_ntt`, all four variants): the C oracle's radix-2 transform.  A mirror of
    `ntt_plan_passes` names each tile pass by (S, position), position one of single / top / middle / bottom; over log n 10-28
    and ZKB_OPT_NTT_MAX_S 5-10 there are 18 shapes, and the DIF cases below run all of them, with both tile kernels
    (ZKB_OPT_NTT_KERNEL 2 and 1) up to 2^22.  The launch count of every transform ties the mirror to the C++ planner.
  * NTT, decimation in time (the forward coset transform of the witness map, coset shift fused into its first pass): the
    C oracle's witness map.  Circuits of 2^10 ... 2^20 and the knob cases cover every DIT shape except the middle passes;
    the 2^21 and 2^22 circuits add the middle pass of S = 7.  The middle DIT passes of S = 8 and 9 only exist at 2^23 and
    above and stay uncovered.
  * MSM over the h_query of a GPU-made key, whose discrete logs follow from the setup trapdoor:
    h_query[i] = (g1_k (tau^n - 1) / delta * tau^i) G, so MSM(h_query[:m], s) = (K * sum s_i tau^i) G.
  * Proofs of 2^21 - 2 and 2^22 - 2 constraints: `zko_trapdoor_expected` (Fr arithmetic and three generator
    multiplications, no NTT, no MSM, no key).

Proof bytes and affine points are canonical, so equality is bit-exactness.  Nothing here reads the reference project."""
import random

import numpy as np
import pytest

from oracle import ark
from oracle.ff import BLS12_381, BN254, g1_group
from zokrates_b200 import synthetic
from zokrates_b200._lib import (OPT_BATCH_AFFINE, OPT_NTT_KERNEL, OPT_NTT_MAX_S, OPT_NTT_TILE_MIN, OPT_TABLES, Context,
                                fr_array)

pytestmark = pytest.mark.gpu
CURVES = [(0, BN254), (1, BLS12_381)]
TD = [3, 5, 7, 11, 1234567, 17, 19]          # alpha, beta, gamma, delta, tau, g1_k, g2_k
R, S = 1234567, 7654321
DEFAULTS = {OPT_NTT_KERNEL: 2, OPT_NTT_MAX_S: 10, OPT_NTT_TILE_MIN: 10, OPT_BATCH_AFFINE: 0, OPT_TABLES: 1}


def _reset(ctx):
    for opt, v in DEFAULTS.items():
        ctx.set_option(opt, v)


# ---- mirror of the NTT pass planner (engine.cuh: ntt_tile_min / ntt_max_s / ntt_tiled, ntt.cuh: ntt_plan_passes) ----------
TILE_LOG = 10                                 # NTT_TILE_LOG: 1024-element tiles


def plan_passes(log_n, max_s=10, tile_min=10):
    """The tile passes a transform of 2^log_n points runs, top stage bits first, as (S, lo_bit); [] means register passes."""
    if log_n < max(tile_min, TILE_LOG):
        return []
    max_s = min(max(max_s, 5), TILE_LOG)
    npass = -(-log_n // max_s)
    out, hi = [], log_n
    for i in range(npass):
        s = log_n // npass + (1 if i < log_n % npass else 0)
        lo = hi - s
        if lo and lo + s < TILE_LOG:          # interleaved groups need runs of 1024 >> S elements below lo_bit
            return []
        out.append((s, lo))
        hi = lo
    return out


def shapes(passes):
    def position(i, lo):
        if len(passes) == 1:
            return "single"
        return "top" if i == 0 else "bottom" if lo == 0 else "middle"
    return {(s, position(i, lo)) for i, (s, lo) in enumerate(passes)}


def pass_launches(log_n, passes):
    """One launch per tile pass; the register passes do 3 stages per launch."""
    return len(passes) if passes else -(-log_n // 3)


ALL_SHAPES = set().union(*(shapes(plan_passes(ln, ms)) for ln in range(10, 29) for ms in range(5, 11)))
DIT_UNCOVERED = {(8, "middle"), (9, "middle")}          # only at 2^23 and above
KNOBS = {10: 5, 15: 5, 17: 6}                            # the only plans with (5, top), (5, middle), (6, middle)
DIF_SIZES, DIF_LARGE, DIT_SIZES = range(10, 23), (23, 26), range(10, 21)
VARIANTS = {"fft": (False, False), "ifft": (True, False), "coset_fft": (False, True), "coset_ifft": (True, True)}


def test_planner_mirror_shapes():
    assert len(ALL_SHAPES) == 18, sorted(ALL_SHAPES)
    assert plan_passes(21) == [(7, 14), (7, 7), (7, 0)] and plan_passes(22) == [(8, 14), (7, 7), (7, 0)]
    assert plan_passes(26) == [(9, 17), (9, 8), (8, 0)] and plan_passes(12, 5) == [] and plan_passes(20, 10, 30) == []


def _rand_fr(seed, n, c):
    x = np.random.default_rng(seed).integers(0, 1 << 64, size=(n, 4), dtype=np.uint64)
    x[:, 3] &= np.uint64((1 << 60) - 1)
    x[:3] = fr_array([c.r - 1, 0, 1])
    return x


def _ntt_launches(log_n, passes, inverse, coset):
    """zkb_ntt (engine.cuh Engine::ntt): to Montgomery form, the forward coset scale, the DIF passes, the bit-reversing copy."""
    return 1 + (1 if coset and not inverse else 0) + pass_launches(log_n, passes) + 1


@pytest.mark.parametrize("cid,c", CURVES, ids=[c.name for _, c in CURVES])
def test_ntt_dif_every_tile_shape_vs_oracle(gpu_lib, oracle_c, cid, c):
    """Default max_s at 2^10 ... 2^22 and the knob cases, both tile kernels, all four variants; the register passes at 2^20;
    2^23 ((8, middle)) and 2^26 ((9, middle), the top of BASELINE config 5) with the default kernel, forward and coset
    inverse.  Every call's launch count equals the mirror's pass count plus the fixed launches of zkb_ntt."""
    cases = []
    for log_n in DIF_SIZES:
        configs = [(2, 10, 10), (1, 10, 10)]
        if log_n in KNOBS:
            configs += [(2, KNOBS[log_n], 10), (1, KNOBS[log_n], 10)]
        if log_n == 20:
            configs.append((2, 10, 30))
        cases.append((log_n, list(VARIANTS), configs))
    cases += [(log_n, ["fft", "coset_ifft"], [(2, 10, 10)]) for log_n in DIF_LARGE]
    ctx = Context(cid, 0, gpu_lib)
    seen = set()
    try:
        for log_n, variants, configs in cases:
            x = _rand_fr(log_n, 1 << log_n, c)
            warm = False
            for name in variants:
                inv, coset = VARIANTS[name]
                want = oracle_c.ntt(cid, x, inv, coset)
                for kernel, max_s, tile_min in configs:
                    ctx.set_option(OPT_NTT_KERNEL, kernel)
                    ctx.set_option(OPT_NTT_MAX_S, max_s)
                    ctx.set_option(OPT_NTT_TILE_MIN, tile_min)
                    passes = plan_passes(log_n, max_s, tile_min)
                    launches = _ntt_launches(log_n, passes, inv, coset)
                    case = (log_n, name, kernel, max_s, tile_min)
                    if not warm:                  # the first transform of a size also builds the domain: 4 table launches
                        before = ctx.launch_count()
                        ctx.ntt(x, inverse=inv, coset=coset)
                        assert ctx.launch_count() - before == launches + 4, case
                        warm = True
                    before = ctx.launch_count()
                    got = ctx.ntt(x, inverse=inv, coset=coset)
                    assert ctx.launch_count() - before == launches, case
                    assert np.array_equal(got, want), case
                    del got
                    seen |= shapes(passes)
                del want
            del x
    finally:
        _reset(ctx)
        ctx.close()
    assert seen == ALL_SHAPES, sorted(ALL_SHAPES - seen)


@pytest.mark.parametrize("cid,c", CURVES, ids=[c.name for _, c in CURVES])
def test_witness_map_dit_tile_shapes_vs_oracle(gpu_lib, oracle_c, cid, c):
    """The DIT passes (and the fused coset shift) through the witness map: circuits of 2^10 ... 2^20 at default max_s and the
    knob cases, both tile kernels.  Covers every DIT shape but the middle passes (S = 7 comes with the 2^21 / 2^22 circuits)."""
    ctx = Context(cid, 0, gpu_lib)
    seen = set()
    try:
        for log_n in DIT_SIZES:
            r1, z = synthetic.make_layered(ctx, c.name, (1 << log_n) - 2)
            h = ctx.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())
            want = oracle_c.witness_map(cid, r1, z)
            max_ss = [10] + ([KNOBS[log_n]] if log_n in KNOBS else [])
            for max_s in max_ss:
                for kernel in (2, 1):
                    ctx.set_option(OPT_NTT_KERNEL, kernel)
                    ctx.set_option(OPT_NTT_MAX_S, max_s)
                    assert np.array_equal(ctx.witness_map(h, z, r1.domain_size), want), (log_n, kernel, max_s)
                    seen |= shapes(plan_passes(log_n, max_s))
            ctx.r1cs_free(h)
    finally:
        _reset(ctx)
        ctx.close()
    assert seen == ALL_SHAPES - DIT_UNCOVERED - {(7, "middle")}, sorted(seen)


# ---- 2^21 / 2^22 circuits: witness map, proofs, sharding, and the h_query MSMs ----------------------------------------------
BIG = [(1, BLS12_381, 22, "uniform"), (0, BN254, 22, "bits"), (0, BN254, 21, "uniform")]


class BigCircuit:
    def __init__(self, lib, oracle_c, cid, c, log_n, dist):
        self.cid, self.c, self.log_n = cid, c, log_n
        self.ctx = Context(cid, 0, lib)
        self.r1, self.z = synthetic.make_layered(self.ctx, c.name, (1 << log_n) - 2, distribution=dist)
        self.h = self.ctx.r1cs_load(self.r1.num_constraints, self.r1.num_instance, self.r1.num_witness, self.r1.matrices())
        self.pk = self.ctx.setup(self.h, TD)
        self.expected = oracle_c.trapdoor_expected(cid, self.r1, TD, self.z, R, S, c.fq_bytes)

    def close(self):
        self.ctx.close()


@pytest.fixture(scope="module", params=BIG, ids=lambda p: f"{p[1].name}-2^{p[2]}-{p[3]}")
def big(request, gpu_lib, oracle_c):
    circ = BigCircuit(gpu_lib, oracle_c, *request.param)
    yield circ
    circ.close()


def test_large_witness_map_vs_oracle(big, oracle_c):
    """Three-pass plans ((7, 7, 7) at 2^21, (8, 7, 7) at 2^22): DIF and DIT middle passes, both tile kernels."""
    ctx = big.ctx
    assert (7, "middle") in shapes(plan_passes(big.log_n))
    want = oracle_c.witness_map(big.cid, big.r1, big.z)
    try:
        for kernel in (2, 1):
            ctx.set_option(OPT_NTT_KERNEL, kernel)
            assert np.array_equal(ctx.witness_map(big.h, big.z, big.r1.domain_size), want), kernel
    finally:
        _reset(ctx)


def test_large_proof_vs_trapdoor(big):
    """GPU proof == trapdoor prediction with the window tables (when they fit the free HBM) and with ZKB_OPT_TABLES = 0;
    a different r gives different bytes."""
    ctx = big.ctx
    assert ctx.r1cs_check(big.h, big.z) is None
    try:
        pkh = ctx.pk_load(big.pk)
        print(f"pk_table_info 2^{big.log_n} {big.c.name}: {ctx.pk_table_info(pkh)}")
        assert ctx.prove(pkh, big.h, big.z, R, S) == big.expected, "tables"
        assert ctx.prove(pkh, big.h, big.z, R + 1, S) != big.expected
        ctx.pk_free(pkh)
        ctx.set_option(OPT_TABLES, 0)
        pkh = ctx.pk_load(big.pk)
        assert ctx.pk_table_info(pkh)["table_bytes"] == 0
        assert ctx.prove(pkh, big.h, big.z, R, S) == big.expected, "no tables"
        ctx.pk_free(pkh)
    finally:
        _reset(ctx)


def test_large_sharded_proof_vs_trapdoor(big):
    """8-way index sharding (what the 8-GPU run of BASELINE config 4 does), here on one GPU."""
    ctx = big.ctx
    pkh = ctx.pk_load(big.pk)
    parts = []
    for rank in range(8):
        ph = ctx.pk_load(big.pk, rank, 8)
        parts.append(ctx.prove_partial(ph, big.h, big.z))
        ctx.pk_free(ph)
    assert ctx.finalize(pkh, np.concatenate(parts), 8, R, S) == big.expected
    ctx.pk_free(pkh)


def h_query(c, pk):
    """The h_query section of ark ProvingKey bytes (oracle/ark.py pk_serialize) as a memoryview, and its length."""
    g1, g2 = 2 * c.fq_bytes, 4 * c.fq_bytes
    view = memoryview(pk)
    off = g1 + 3 * g2

    def skip_vec(off, item):
        return off + 8 + int.from_bytes(pk[off:off + 8], "little") * item

    off = skip_vec(off, g1) + 2 * g1                     # gamma_abc_g1, beta_g1, delta_g1
    off = skip_vec(skip_vec(skip_vec(off, g1), g1), g2)  # a_query, b_g1_query, b_g2_query
    cnt = int.from_bytes(pk[off:off + 8], "little")
    return view[off + 8:off + 8 + cnt * g1], cnt


def _ints(a):
    b = np.ascontiguousarray(a).tobytes()
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


def _horner(vals, tau, r):
    acc = 0
    for v in reversed(vals):
        acc = (acc * tau + v) % r
    return acc


MSM_SIZES = ((1 << 22) - 1, 3 * (1 << 20) + 17, 1 << 21)


def test_large_msm_known_discrete_logs(big):
    """zkb_msm_g1 over h_query[:m] of the GPU-made key for m = 2^22 - 1, 3 * 2^20 + 17, 2^21 (the whole h_query of the 2^21
    circuit), batch-affine rounds off and on: uniform, 90 % {0, 1}, all equal (one bucket per window holds every point),
    all r - 1 (signed-digit carries into the top window), and a set summing to zero (the point at infinity)."""
    c, ctx = big.c, big.ctx
    r, n = c.r, 1 << big.log_n
    delta, tau, g1_k = TD[3], TD[4], TD[5]
    K = g1_k * (pow(tau, n, r) - 1) * pow(delta, -1, r) % r
    G1 = g1_group(c)
    pts, cnt = h_query(c, big.pk)
    assert cnt == n - 1
    g1b = 2 * c.fq_bytes
    for i in [0, 1, 2, n - 2] + random.Random(big.log_n).sample(range(n - 1), 4):   # the formula, on the key itself
        assert bytes(pts[i * g1b:(i + 1) * g1b]) == ark.ser_g1(c, G1.mul(c.g1, K * pow(tau, i, r))), i
    sizes = sorted({n - 1} | {m for m in MSM_SIZES if m < n})
    M = max(sizes)
    rng = np.random.default_rng(big.log_n + 10 * big.cid)
    uni = rng.integers(0, 1 << 64, size=(M, 4), dtype=np.uint64)
    uni[:, 3] &= np.uint64((1 << 60) - 1)
    bits = uni.copy()
    small = rng.random(M) < 0.9
    bits[small] = 0
    bits[small, 0] = rng.integers(0, 2, size=int(small.sum()), dtype=np.uint64)
    uni_v, bits_v = _ints(uni), _ints(bits)
    same = random.Random(big.log_n).randrange(1, r)
    try:
        for m in sizes:
            geo = (pow(tau, m, r) - 1) * pow(tau - 1, -1, r) % r          # sum of tau^i, i < m
            h_uni = _horner(uni_v[:m], tau, r)
            # the last scalar solved so that sum s_i tau^i == 0
            head = (h_uni - uni_v[m - 1] * pow(tau, m - 1, r)) % r
            zero = uni[:m].copy()
            zero[m - 1] = fr_array([-head * pow(tau, -(m - 1), r) % r])[0]
            sets = [("uniform", uni[:m], h_uni), ("bits", bits[:m], _horner(bits_v[:m], tau, r)),
                    ("equal", np.tile(fr_array([same]), (m, 1)), same * geo % r),
                    ("r-1", np.tile(fr_array([r - 1]), (m, 1)), (r - 1) * geo % r), ("zero-sum", zero, 0)]
            for name, sc, dlog in sets:
                e = K * dlog % r
                want = ark.ser_g1(c, G1.mul(c.g1, e) if e else None)
                if name == "zero-sum":
                    assert e == 0 and want[-4:] == (0x40000000).to_bytes(4, "little")
                for rounds in (0, 3):
                    ctx.set_option(OPT_BATCH_AFFINE, rounds)
                    assert ctx.msm(1, pts[:m * g1b], sc) == want, (m, name, rounds)
    finally:
        _reset(ctx)
