"""The exceptional branches of the MSM pipeline against known discrete logs: duplicate points, P + (-P), identity
accumulators and partials, runs of affine infinities, equal bucket sums, and sums that are the point at infinity.

Random scalars over distinct points reach these branches with probability ~1/r, yet real keys produce them (variables
with identical A / B columns give duplicate query points, 0/1-heavy witnesses fill one bucket, b-query infinities come in
runs).  Here every point is drawn from a small pool k_j G (8 random dlogs and their negatives) plus the point at
infinity (dlog 0), tiled to any length by numpy indexing, so the expected value of any MSM is (sum s_i k_j(i) mod r) G:
one scalar multiplication, no MSM or NTT code involved.

  * Standalone `zkb_msm_g1` / `zkb_msm_g2` on both curves (cases in `msm_cases`): G1 at m = 4099, 2^16 and 2^20, G2 at
    4099 and 2^16; at 2^16 over the knob grid batch-affine {0, 3} x bit-sum radix {2, 8} x chunk length {8, 64}.
  * Proofs with a crafted ark-format proving key (`crafted_key`) whose query points come from the pool, with an
    adversarial assignment (zeros, ones, r - 1, repeated and uniform values): the expected proof follows from the dlogs
    and the C oracle's witness map.  Window tables (cost-model c, forced c = 16, none), ZKB_OPT_Z_MODE 1 and 2,
    batch-affine and radix knobs, and 3- / 8-way index sharding.  At 2^16 the C oracle's prover gives the same bytes.
  * A key with fewer assignment pairs than ranks (3 pairs, 8 ranks: empty shard slices).

The small cases (m <= 2^11, a 2^10 circuit, the tiny key) also run in the CPU tier through the host emulation; the GPU
cases are marked `gpu`.  Nothing here reads the reference project."""
import random
import struct

import numpy as np
import pytest

from oracle import ark
from oracle.ff import BLS12_381, BN254, g1_group, g2_group
from zokrates_b200 import synthetic
from zokrates_b200._lib import (OPT_BATCH_AFFINE, OPT_BATCH_AFFINE_MIN_LOG, OPT_BITSUM_RADIX, OPT_TABLE_C, OPT_TABLE_MIN_LOG,
                                OPT_TABLES, OPT_Z_MODE, Context, fr_array)
from zokrates_b200.r1cs import R1CS

OPT_CHUNK_TARGET = 13                       # include/zkb.h ZKB_OPT_CHUNK_TARGET
CURVES = [(0, BN254), (1, BLS12_381)]
K = 16                                      # pool points; index K is the point at infinity
ALPHA, BETA, GAMMA, DELTA = 3, 5, 7, 11     # dlogs of the fixed key points
R, S = 1234567, 7654321
DEFAULTS = {OPT_BATCH_AFFINE: 0, OPT_BATCH_AFFINE_MIN_LOG: 16, OPT_BITSUM_RADIX: 2, OPT_CHUNK_TARGET: 600000,
            OPT_Z_MODE: 0}


# ---- construction ----------------------------------------------------------------------------------------------------
class Pool:
    """k_j G1 and k_j G2 for the same dlogs k_j (j < 8 random, k_(j+8) = -k_j), serialised once; row K is infinity."""

    def __init__(self, c, seed):
        self.c = c
        self.G = {1: g1_group(c), 2: g2_group(c)}
        self.gen = {1: c.g1, 2: c.g2}
        self.ser = {1: ark.ser_g1, 2: ark.ser_g2}
        rnd = random.Random(seed)
        half = [rnd.randrange(1, c.r) for _ in range(K // 2)]
        self.dlog = half + [c.r - d for d in half] + [0]
        self.raw = {}
        for g in (1, 2):
            pts = [self.G[g].mul(self.gen[g], d) for d in half]
            pts += [self.G[g].neg(P) for P in pts] + [None]
            self.raw[g] = np.frombuffer(b"".join(self.ser[g](c, P) for P in pts), np.uint8).reshape(K + 1, -1)

    def points(self, g, idx):
        return self.raw[g][idx].tobytes()

    def point(self, g, e):
        """Serialised e * generator (e mod r; 0 gives ark's infinity encoding)."""
        e %= self.c.r
        return self.ser[g](self.c, self.G[g].mul(self.gen[g], e) if e else None)

    def dlog_sum(self, idx, sc):
        """sum_i s_i k_idx[i] mod r for canonical scalars sc (m x 4 uint64), with per-pool-point limb sums in numpy."""
        sc32 = np.ascontiguousarray(sc, dtype=np.uint64).view(np.uint32).reshape(len(sc), 8)
        acc = 0
        for j in np.unique(idx):
            if self.dlog[j] == 0:
                continue
            col = sc32[idx == j].sum(axis=0, dtype=np.uint64)      # < 2^32 * 2^31 per column: exact
            acc += sum(int(v) << (32 * k) for k, v in enumerate(col)) * self.dlog[j]
        return acc % self.c.r


def uniform(rng, m):
    x = rng.integers(0, 1 << 64, size=(m, 4), dtype=np.uint64)
    x[:, 3] &= np.uint64((1 << 60) - 1)     # < 2^252 < r on both curves
    return x


def small(v):
    x = np.zeros((len(v), 4), dtype=np.uint64)
    x[:, 0] = v
    return x


def msm_cases(pool, m, seed):
    """(name, pool index per point, scalars) for one MSM size."""
    c, r = pool.c, pool.c.r
    rng = np.random.default_rng(seed)
    t = np.arange(m)
    cases = [("one-point", np.zeros(m, np.int64), uniform(rng, m)),     # a doubling in every bucket, equal chunk partials
             ("equal-buckets", np.zeros(m, np.int64), small(t % 8 + 1))]  # buckets 0..7 of window 0 hold equal sums
    # cancellation: (P_j, -P_j) with equal scalars in the first half, (P_j, P_j) with (s, r - s) in the second; the sum
    # is the point at infinity (an unpaired last point gets scalar 0)
    vals = [random.Random(seed + k).randrange(1, r) for k in range(64)]
    table = fr_array(vals + [r - v for v in vals] + [0])
    pair = (t // 2) % 8
    second = t >= m // 2
    idx = np.where(second, pair, pair + 8 * (t % 2))
    code = (t // 2) % 64 + np.where(second & (t % 2 == 1), 64, 0)
    if m % 2:
        code[-1] = 128
    cases.append(("cancellation", idx, table[code]))
    # runs of infinity: short runs every 64 positions, then a 2048-run and a 4096-run (whole view groups / tiles)
    idx = t % K
    inf = (t // 64) % 5 == 0
    inf |= ((t >= 1024) & (t < 1024 + 2048)) | ((t >= m // 2) & (t < m // 2 + 4096))
    idx = np.where(inf, K, idx)
    sc = np.where((t < m // 2)[:, None], small(t % 8 + 1), uniform(rng, m))
    cases.append(("infinity-runs", idx, sc))
    # skewed: 90 % unit scalars over the pool (one bucket spanning thousands of chunks, with duplicates in it)
    sc = uniform(rng, m)
    ones = rng.random(m) < 0.9
    sc[ones] = small(np.ones(int(ones.sum()), np.uint64))
    cases.append(("skewed", t % K, sc))
    # zero sum: the last scalar solved so that the total is 0
    idx = t % 8
    sc = uniform(rng, m)
    head = pool.dlog_sum(idx[:-1], sc[:-1])
    sc[-1] = fr_array([-head * pow(pool.dlog[idx[-1]], -1, r) % r])[0]
    cases.append(("zero-sum", idx, sc))
    return cases


def run_msm_cases(ctx, pool, g, m, configs, seed):
    for name, idx, sc in msm_cases(pool, m, seed):
        want = pool.point(g, pool.dlog_sum(idx, sc))
        if name in ("zero-sum", "cancellation"):
            assert want[-1] & 0x40, name          # ark's infinity flag
        pts = pool.points(g, idx)
        for cfg in configs:
            for opt, v in {**DEFAULTS, **cfg}.items():
                ctx.set_option(opt, v)
            assert ctx.msm(g, pts, sc) == want, (name, g, m, cfg)


def adversarial_z(c, m, seed):
    """z[0] = 1; blocks of 512 of zeros, ones, r - 1, one repeated value and uniform values."""
    rng = np.random.default_rng(seed)
    t = np.arange(m)
    rep = fr_array([random.Random(seed).randrange(c.r)])[0]
    kinds = np.stack([np.zeros((m, 4), np.uint64), small(np.ones(m, np.uint64)), np.tile(fr_array([c.r - 1]), (m, 1)),
                      np.tile(rep, (m, 1)), uniform(rng, m)])
    z = kinds[(t // 512) % 5, t]
    z[0] = fr_array([1])[0]
    return z


def crafted_key(pool, r1, z, seed):
    """An ark-format proving key (oracle/ark.py pk_serialize layout) for r1 whose query points come from the pool, and
    the z it pairs with (adjusted in place where a segment needs equal or 1..8 values).  Over the variable index:
      [0, m/4)     duplicate points in runs (a: 64, b: 16, l: 128)
      [m/4, m/2)   (k, -k) index pairs with equal z
      [m/2, 3m/4)  clustered infinity runs in a (whole 2048-runs and every third 32-group) and in b (most of it)
      [3m/4, m)    a, b and l all the same point, z = 1..8 in equal counts
    b_g1_query[i] and b_g2_query[i] share their dlog (so both are infinity together); h_query holds runs of duplicates
    and negation pairs.  Returns (key bytes, index arrays)."""
    c = pool.c
    m, ni, n = r1.num_variables, r1.num_instance, r1.domain_size
    t = np.arange(m)
    rng = np.random.default_rng(seed)
    q1, q2, q3 = m // 4, m // 2, 3 * m // 4
    ia, ib, il = (t // 64) % K, (t // 16) % K, (t // 128) % K
    seg = (t >= q1) & (t < q2)
    pair = (t // 2) % 8 + 8 * (t % 2)
    ia, ib, il = np.where(seg, pair, ia), np.where(seg, pair, ib), np.where(seg, (pair + 3) % K, il)
    odd = np.flatnonzero(seg & (t % 2 == 1))
    z[odd] = z[odd - 1]
    seg = (t >= q2) & (t < q3)
    ia = np.where(seg & (((t // 2048) % 2 == 0) | ((t // 32) % 3 == 0)), K, ia)
    ib = np.where(seg & ((t // 1000) % 8 != 7), K, ib)
    seg = t >= q3
    ia, ib, il = np.where(seg, 5, ia), np.where(seg, 5, ib), np.where(seg, 5, il)
    z[seg] = small(t[seg] % 8 + 1)
    z[0] = fr_array([1])[0]
    ih = np.where((np.arange(n - 1) // 4096) % 2 == 0, (np.arange(n - 1) // 32) % K, rng.integers(0, K, n - 1))
    P = pool.point
    head = [P(1, ALPHA), P(2, BETA), P(2, GAMMA), P(2, DELTA), struct.pack("<Q", ni)]
    head += [P(1, 13 + i) for i in range(ni)] + [P(1, BETA), P(1, DELTA)]
    body = [struct.pack("<Q", m), pool.points(1, ia), struct.pack("<Q", m), pool.points(1, ib), struct.pack("<Q", m),
            pool.points(2, ib), struct.pack("<Q", n - 1), pool.points(1, ih), struct.pack("<Q", m - ni), pool.points(1, il[ni:])]
    return b"".join(head + body), (ia, ib, il, ih)


def expected_proof(pool, r1, z, idx, h, r, s):
    """A = alpha + sum z_i a_i + r delta, B = beta + sum z_i b_i + s delta (G1 and G2),
    C = s A + r B1 - r s delta + sum_(i >= ni) z_i l_(i - ni) + sum_j h_j q_j."""
    ia, ib, il, ih = idx
    q, ni, n = pool.c.r, r1.num_instance, r1.domain_size
    a = (ALPHA + pool.dlog_sum(ia, z) + r * DELTA) % q
    b = (BETA + pool.dlog_sum(ib, z) + s * DELTA) % q
    cc = (s * a + r * b - r * s * DELTA + pool.dlog_sum(il[ni:], z[ni:]) + pool.dlog_sum(ih, h[:n - 1])) % q
    return pool.point(1, a) + pool.point(2, b) + pool.point(1, cc)


class Crafted:
    """A circuit of the make_layered family, the adversarial z, the crafted key and the expected proof."""

    def __init__(self, ctx, oracle_c, cid, c, n_constraints, seed=1):
        self.pool = Pool(c, seed)
        self.r1, _ = synthetic.make_layered(ctx, c.name, n_constraints)
        self.z = adversarial_z(c, self.r1.num_variables, seed)
        self.pk, idx = crafted_key(self.pool, self.r1, self.z, seed)
        self.h = oracle_c.witness_map(cid, self.r1, self.z)
        self.expected = expected_proof(self.pool, self.r1, self.z, idx, self.h, R, S)


def prove_modes(ctx, cr, modes, shards=(3, 8)):
    """The crafted proof under each (key options, prover options) mode, and index-sharded."""
    rh = ctx.r1cs_load(cr.r1.num_constraints, cr.r1.num_instance, cr.r1.num_witness, cr.r1.matrices())
    for key_opts, prove_opts in modes:
        for opt, v in {OPT_TABLES: 1, OPT_TABLE_C: 0, **key_opts}.items():
            ctx.set_option(opt, v)
        pkh = ctx.pk_load(cr.pk)
        for po in prove_opts:
            for opt, v in {**DEFAULTS, **po}.items():
                ctx.set_option(opt, v)
            assert ctx.prove(pkh, rh, cr.z, R, S) == cr.expected, (key_opts, po, ctx.pk_table_info(pkh))
        ctx.pk_free(pkh)
    for opt, v in {OPT_TABLES: 1, OPT_TABLE_C: 0, **DEFAULTS}.items():
        ctx.set_option(opt, v)
    pkh = ctx.pk_load(cr.pk)
    for world in shards:
        parts = []
        for rank in range(world):
            ph = ctx.pk_load(cr.pk, rank, world)
            parts.append(ctx.prove_partial(ph, rh, cr.z))
            ctx.pk_free(ph)
        assert ctx.finalize(pkh, np.concatenate(parts), world, R, S) == cr.expected, world
    ctx.pk_free(pkh)
    ctx.r1cs_free(rh)


def tiny_crafted(c, pool, z_vals):
    """Four variables (one, one public input, two witnesses), two constraints: 3 assignment pairs, a domain of 4."""
    one = fr_array([1])
    rows = (np.array([0, 1, 2], np.uint64), np.array([2, 3], np.uint32), np.tile(one, (2, 1)))
    r1 = R1CS(c.name, 2, 2, 2, rows, rows, (np.array([0, 1, 2], np.uint64), np.array([1, 1], np.uint32), np.tile(one, (2, 1))))
    z = fr_array([1] + z_vals)
    idx = (np.array([3, 0, 8, 0]), np.array([K, 0, K, 0]), np.array([0, 0, 0, 8]), np.array([1, 1, 9]))
    ia, ib, il, ih = idx
    P = pool.point
    pk = b"".join([P(1, ALPHA), P(2, BETA), P(2, GAMMA), P(2, DELTA), struct.pack("<Q", 2), P(1, 13), P(1, 14),
                   P(1, BETA), P(1, DELTA), struct.pack("<Q", 4), pool.points(1, ia), struct.pack("<Q", 4), pool.points(1, ib),
                   struct.pack("<Q", 4), pool.points(2, ib), struct.pack("<Q", 3), pool.points(1, ih), struct.pack("<Q", 2),
                   pool.points(1, il[2:])])
    return r1, z, pk, idx


def check_tiny(ctx, oracle_c, cid, c):
    """Fewer assignment pairs (3) than ranks (8): some shard slices are empty.  a_query[1] and [3] are the same point
    and a_query[2] its negation with an equal z; b_query[0] and [2] are infinity; h_query holds a duplicate and a
    negation."""
    pool = Pool(c, 5)
    r1, z, pk, idx = tiny_crafted(c, pool, [7, 7, c.r - 1])
    h = oracle_c.witness_map(cid, r1, z)
    want = expected_proof(pool, r1, z, idx, h, R, S)
    rh = ctx.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())
    pkh = ctx.pk_load(pk)
    assert ctx.prove(pkh, rh, z, R, S) == want
    for world in (2, 3, 8):
        parts = [ctx.prove_partial(ctx.pk_load(pk, rank, world), rh, z) for rank in range(world)]
        assert ctx.finalize(pkh, np.concatenate(parts), world, R, S) == want, world
    assert oracle_c.prove(cid, pk, r1, z, R, S, c.fq_bytes)[0] == want


# ---- CPU tier: the host emulation ------------------------------------------------------------------------------------
@pytest.mark.parametrize("cid,c", CURVES, ids=[c.name for _, c in CURVES])
def test_emu_msm_exceptional(emu_lib, cid, c):
    """G1 at m = 2^11 + 3 (default knobs, and batch-affine rounds with a short chunk), G2 at m = 259."""
    ctx = Context(cid, 0, emu_lib)
    pool = Pool(c, 11 + cid)
    run_msm_cases(ctx, pool, 1, 2051, [{}, {OPT_BATCH_AFFINE: 3, OPT_BATCH_AFFINE_MIN_LOG: 0, OPT_CHUNK_TARGET: 1000}], 2051)
    run_msm_cases(ctx, pool, 2, 259, [{}], 259)


@pytest.mark.parametrize("cid,c", CURVES, ids=[c.name for _, c in CURVES])
def test_emu_tiny_key_empty_shards(emu_lib, oracle_c, cid, c):
    check_tiny(Context(cid, 0, emu_lib), oracle_c, cid, c)


def test_emu_crafted_proof(emu_lib, oracle_c):
    """A 2^10 BN254 circuit with the crafted key: window tables (forced c = 16) under both z modes and both bit-sum
    radixes, no tables, 3- / 8-way sharding; the C oracle's prover gives the same bytes."""
    ctx = Context(0, 0, emu_lib)
    cr = Crafted(ctx, oracle_c, 0, BN254, (1 << 10) - 2)
    assert oracle_c.prove(0, cr.pk, cr.r1, cr.z, R, S, BN254.fq_bytes)[0] == cr.expected
    ctx.set_option(OPT_TABLE_MIN_LOG, 0)                       # window tables for this small key too
    modes = [({OPT_TABLE_C: 16}, [{OPT_Z_MODE: 1}, {OPT_Z_MODE: 2, OPT_BITSUM_RADIX: 8}]), ({OPT_TABLES: 0}, [{}])]
    prove_modes(ctx, cr, modes)


# ---- GPU tier --------------------------------------------------------------------------------------------------------
GRID = [{OPT_BATCH_AFFINE: ba, OPT_BATCH_AFFINE_MIN_LOG: 0, OPT_BITSUM_RADIX: rad, OPT_CHUNK_TARGET: ct}
        for ba in (0, 3) for rad in (2, 8) for ct in (600000, 1000)]
PLAIN = [{}, {OPT_BATCH_AFFINE: 3, OPT_BATCH_AFFINE_MIN_LOG: 0}]
MSM_RUNS = [(1, 1 << 16, GRID), (2, 1 << 16, GRID), (1, 4099, PLAIN), (2, 4099, PLAIN), (1, 1 << 20, PLAIN)]


@pytest.mark.gpu
@pytest.mark.parametrize("g,m,configs", MSM_RUNS, ids=[f"G{g}-{m}-{'grid' if cf is GRID else 'plain'}" for g, m, cf in MSM_RUNS])
@pytest.mark.parametrize("cid,c", CURVES, ids=[c.name for _, c in CURVES])
def test_msm_exceptional(gpu_lib, cid, c, g, m, configs):
    ctx = Context(cid, 0, gpu_lib)
    try:
        run_msm_cases(ctx, Pool(c, 11 + cid), g, m, configs, m + cid)
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cid,c", CURVES, ids=[c.name for _, c in CURVES])
def test_tiny_key_empty_shards(gpu_lib, oracle_c, cid, c):
    ctx = Context(cid, 0, gpu_lib)
    try:
        check_tiny(ctx, oracle_c, cid, c)
    finally:
        ctx.close()


PROOFS = [(0, BN254, 16), (1, BLS12_381, 16), (0, BN254, 20)]


@pytest.mark.gpu
@pytest.mark.parametrize("cid,c,log_n", PROOFS, ids=[f"{c.name}-2^{k}" for _, c, k in PROOFS])
def test_crafted_key_proof(gpu_lib, oracle_c, cid, c, log_n):
    """The crafted key of a 2^log_n - 2 constraint circuit: window tables by the cost model, forced c = 16 and none;
    ZKB_OPT_Z_MODE 1 (shared buckets over the tables) and 2 (per-window buckets); at 2^16 also batch-affine {0, 3} x radix
    {2, 8} and the C oracle's prover on the same key bytes; 3- and 8-way sharding."""
    ctx = Context(cid, 0, gpu_lib)
    try:
        cr = Crafted(ctx, oracle_c, cid, c, (1 << log_n) - 2)
        z_modes = [{OPT_Z_MODE: 1}, {OPT_Z_MODE: 2}]
        if log_n == 16:
            assert oracle_c.prove(cid, cr.pk, cr.r1, cr.z, R, S, c.fq_bytes)[0] == cr.expected
            knobs = [{**zm, OPT_BATCH_AFFINE: ba, OPT_BATCH_AFFINE_MIN_LOG: 0, OPT_BITSUM_RADIX: rad}
                     for zm in z_modes for ba in (0, 3) for rad in (2, 8)]
            modes = [({}, knobs), ({OPT_TABLE_C: 16}, z_modes), ({OPT_TABLES: 0}, z_modes)]
        else:
            modes = [({}, z_modes), ({OPT_TABLES: 0}, [{}])]
        prove_modes(ctx, cr, modes)
    finally:
        ctx.close()
