"""The device-only kernels of the MSM plan at their boundaries: the bucket-offset scan (engine.cuh `exclusive_scan`) and the
view compaction (`zkb_view_count` / `zkb_view_apply` and the pre32 / mask32 groups read by `msm_view_offsets_body`).

The host emulation replaces these kernels with serial loops, so only the GPU runs them.  Here the inputs are built so that
their boundaries fall where the kernels can go wrong, and every expected value is one scalar multiplication: the points
come from the k*G pool of tests/test_gpu_exceptional.py, and a scalar d * 2^(c w) with 1 <= d <= 2^(c-1) gives its point
exactly one nonzero digit, d in window w, so it lands in bucket key w * B + d - 1 (B = 2^(c-1)).  Bucket counts, and with
them every offset, follow from the multiplicities.

A Python mirror of the planner's shape (`msm_pick_c`, `msm_pick_c_pre`, `plan_w`, NB = K * (pre ? 1 : W) * B) picks the
cases.  The device build counts the scan and view launches, the emulation does not, so the launch counts of one call on
both builds differ by exactly what the mirror predicts (1 launch for the single-block scan of NB <= 4096 counters, 3 for the
tile-sum / single-block / tile-apply scan above): that ties the mirror to the C++ planner.

  * Standalone G1 / G2 MSMs at c = 8 (NB = 4096 exactly: the single-block scan), c = 9 (NB = 7424: the three-phase scan
    with a partial last 2048-tile) and c = 11 (NB = 24576: full tiles only): all entries in one bucket, counts only at keys
    2047, 2048, 4095, 4096 and the last reachable key, empty leading and trailing tiles, one entry in the last bucket.
  * Batched proofs with window tables at c = 16 (16 scan tiles of 2048 per proof): K = 64 gives 1024 tile sums, K = 65
    gives 1040, where the single-block scan of the tile sums takes 2 per thread.  Every proof equals the single proof and
    the trapdoor prediction.
  * View compaction: crafted keys whose a_query / b_query infinities are chosen per bucket and small z values that fix the
    bucket layout, so every bucket is wholly kept or wholly dropped in each view and the expected lists do not depend on the
    device's arrival order.  Bucket offsets at lanes 0, 1, 30 and 31 of a 32-position group; groups fully kept, fully
    dropped, keeping only lane 0 or only lane 31; whole 2048-tiles dropped in one view and kept in the other; M mod 2048 in
    {0, 1, 2047} and M mod 32 = 0.  Both z modes; each proof equals the dlog prediction, and at 2^16 the C oracle's bytes."""
import time

import numpy as np
import pytest

from oracle.ff import BLS12_381, BN254
from tests.test_batch_prove import TD, reassign
from tests.test_gpu_exceptional import K as POOL_K, R, S, Pool, expected_proof, key_bytes
from zokrates_b200 import synthetic
from zokrates_b200._lib import (OPT_BATCH_PASS_MAX, OPT_TABLE_C, OPT_TABLE_MIN_LOG, OPT_TABLES, OPT_Z_MODE, Context, fr_array)

CURVES = {0: BN254, 1: BLS12_381}
FR_BITS = {0: 254, 1: 255}          # C::FR_BITS
SCAN_TILE, SCAN_SINGLE_MAX, VIEW_TILE = 2048, 4096, 2048


# ---- mirror of the planner (engine.cuh) ------------------------------------------------------------------------------
def msm_pick_c(n, fr_bits):
    best, best_cost = 4, float("inf")
    for c in range(4, 17):
        W = (fr_bits + c) // c
        cost = W * (10.0 * n + 40.0 * (1 << (c - 1)))
        if cost < best_cost:
            best, best_cost = c, cost
    return best


def msm_pick_c_pre(n, fr_bits, max_w=16):
    best, best_cost = 0, float("inf")
    for c in range(4, 23):
        W = (fr_bits + c) // c
        if W > max_w or n * W >= 1 << 31:
            continue
        cost = W * 10.0 * n + 70.0 * (1 << (c - 1))
        if cost < best_cost:
            best, best_cost = c, cost
    return best


def plan_w(c, fr_bits):
    return (fr_bits + c) // c


def nbuckets(n, fr_bits, K=1, pre_c=0):
    c = pre_c or msm_pick_c(n, fr_bits)
    return K * (1 if pre_c else plan_w(c, fr_bits)) * (1 << (c - 1))


def scan_launches(n):
    return 3 if n > SCAN_SINGLE_MAX else 1


def tile_sum_per(n):
    """the per-thread count of the single-block scan that scans the tile sums of an n-counter three-phase scan"""
    ntiles = -(-n // SCAN_TILE)
    return -(-ntiles // 1024)


@pytest.fixture(scope="module", autouse=True)
def wall_time():
    t0 = time.time()
    yield
    print("\ntest_gpu_plan_kernels wall time: %.1f s" % (time.time() - t0))


# ---- bucket-offset scan: standalone MSMs -----------------------------------------------------------------------------
def key_scalar(key, c, B):
    w, d = divmod(key, B)
    return (d + 1) << (c * w)


def reachable(key, c, B, r):
    return key_scalar(key, c, B) < r


def bucket_cases(c_, n, c, fr_bits):
    """(name, pool index per point, scalar per point) with the bucket keys placed at the scan's boundaries"""
    r, B = c_.r, 1 << (c - 1)
    NB = plan_w(c, fr_bits) * B
    last = max(k for k in range(NB - 1, NB - 1 - B, -1) if reachable(k, c, B, r))
    idx = np.arange(n) % (POOL_K + 1)                  # row POOL_K is the point at infinity
    t = np.arange(n)
    out = [("one-bucket", [2048] * n)]
    keys = [k for k in (2047, 2048, 4095, 4096, last) if k < NB and reachable(k, c, B, r)]
    weights = np.array([1, 7, 3, 2, 5][:len(keys)])
    pick = np.searchsorted(np.cumsum(weights), t % weights.sum(), side="right")
    out.append(("boundary-keys", [None if i % 11 == 0 else keys[p] for i, p in zip(t, pick)]))
    out.append(("middle-only", [2100 + (i % 37) for i in t]))     # empty leading tile and empty trailing tiles
    out.append(("last-bucket-once", [last] + [None] * (n - 1)))
    for name, ks in out:
        sc = fr_array([0 if k is None else key_scalar(k, c, B) for k in ks])
        yield name, idx, sc


SHAPES = [(0, 1, 8, 2000), (0, 1, 9, 5000), (0, 1, 11, 24000), (1, 1, 9, 5000), (0, 2, 8, 2000), (0, 2, 9, 5000)]


@pytest.mark.gpu
@pytest.mark.parametrize("cid,g,c,n", SHAPES, ids=[f"{CURVES[cid].name}-G{g}-c{c}" for cid, g, c, n in SHAPES])
def test_bucket_offset_scan(gpu_lib, emu_lib, cid, g, c, n):
    cv, fb = CURVES[cid], FR_BITS[cid]
    assert msm_pick_c(n, fb) == c
    NB = nbuckets(n, fb)
    pool = Pool(cv, 40 + c)
    ctx, emu = Context(cid, 0, gpu_lib), Context(cid, 0, emu_lib)
    try:
        for k, (name, idx, sc) in enumerate(bucket_cases(cv, n, c, fb)):
            pts = pool.points(g, idx)
            want = pool.point(g, pool.dlog_sum(idx, sc))
            before = ctx.launch_count()
            assert ctx.msm(g, pts, sc) == want, name
            launches = ctx.launch_count() - before
            if k == 0 and g == 1 and c < 11:      # the tie: device launches - emulated launches = the scan's launches
                before = emu.launch_count()
                assert emu.msm(g, pts, sc) == want, name
                assert launches - (emu.launch_count() - before) == scan_launches(NB), (name, NB)
    finally:
        ctx.close()
        emu.close()
    if c == 8:
        assert NB == 4096 and scan_launches(NB) == 1
    elif c == 9:
        assert NB == 7424 and NB % SCAN_TILE and scan_launches(NB) == 3
    else:
        assert NB % SCAN_TILE == 0 and scan_launches(NB) == 3


# ---- bucket-offset scan: batched proofs with more than 1024 tile sums --------------------------------------------------
TABLE_OPTS = {OPT_TABLES: 2, OPT_TABLE_MIN_LOG: 4, OPT_TABLE_C: 16, OPT_Z_MODE: 1}


@pytest.mark.gpu
def test_batch_tile_sum_scan(gpu_lib, emu_lib, oracle_c):
    """Window tables at c = 16 put 2^15 buckets per proof in one set: K = 64 proofs need 1024 scan tiles, K = 65 need 1040
    (2 tile sums per thread).  Satisfying reassignments of one circuit; each proof equals the single proof and the trapdoor
    prediction."""
    cv, fb = BN254, FR_BITS[0]
    r1, z = synthetic.make("bn128", 1000)
    m0 = r1.num_variables - r1.num_constraints
    rnd = np.random.RandomState(65)
    zs = [z] + [reassign(r1, z, [int(v) for v in rnd.randint(1, 1 << 62, size=m0 - 1)]) for _ in range(4)]
    pk_bytes = oracle_c.setup(0, r1, TD)
    ctx, emu = Context(0, 0, gpu_lib), Context(0, 0, emu_lib)
    m, n_h = r1.num_variables - 1, r1.domain_size - 1
    try:
        # the tie: device-only launches of one proof with tables minus one without, on both builds, against the mirror
        extra, handles = {}, {}
        for tables in (0, 1):
            for x in (ctx, emu):
                for o, v in TABLE_OPTS.items():
                    x.set_option(o, v if tables else {OPT_TABLES: 0, OPT_Z_MODE: 0}.get(o, v))
                h = x.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())
                pk = x.pk_load(pk_bytes)
                info = x.pk_table_info(pk)
                before = x.launch_count()
                assert x.prove(pk, h, zs[0], 7, 8) == oracle_c.trapdoor_expected(0, r1, TD, zs[0], 7, 8, cv.fq_bytes)
                extra[tables] = extra.get(tables, 0) + (x.launch_count() - before) * (1 if x is ctx else -1)
                if tables:
                    assert info["z_tables"] == "built" and info["c_z"] == 16, info
                    handles[x is ctx] = (h, pk, info)
        h, pk, info = handles[True]
        pre_h = info["h_table"] == "built"

        def mirror(cz, ch):
            """scan of the z plan's buckets, the two view compactions and their tile scans, scan of the h plan's buckets"""
            Wz = plan_w(cz or msm_pick_c(m, fb), fb)
            return scan_launches(nbuckets(m, fb, 1, cz)) + 2 + 2 * scan_launches(-(-m * Wz // VIEW_TILE)) + \
                scan_launches(nbuckets(n_h, fb, 1, ch))
        want = mirror(16, info["c_h"] if pre_h else 0) - mirror(0, 0)
        assert extra[1] - extra[0] == want, (extra, want)
        assert scan_launches(nbuckets(m, fb, 1, 16)) == 3 and scan_launches(nbuckets(m, fb)) == 1
        ctx.set_option(OPT_BATCH_PASS_MAX, 65)
        for K in (64, 65):
            NB = nbuckets(m, fb, K, 16)
            assert -(-NB // SCAN_TILE) == 16 * K and tile_sum_per(NB) == (1 if K == 64 else 2)
            rs, ss = [100 + k for k in range(K)], [300 + 7 * k for k in range(K)]
            got = ctx.prove_batch(pk, h, [zs[k % 5] for k in range(K)], rs, ss)
            for k in range(K):
                assert got[k] == ctx.prove(pk, h, zs[k % 5], rs[k], ss[k]), (K, k)
            for k in (0, 1, K - 1):
                assert got[k] == oracle_c.trapdoor_expected(0, r1, TD, zs[k % 5], rs[k], ss[k], cv.fq_bytes), (K, k)
    finally:
        ctx.close()
        emu.close()


# ---- view compaction -------------------------------------------------------------------------------------------------
def view_layout(M_target, seed):
    """Buckets (z value d, count, kept in view 1, kept in view 2), laid out from sorted position 0: offsets at lanes 0, 1,
    30 and 31; groups fully kept, fully dropped, keeping only lane 0 or only lane 31; a whole 2048-tile dropped in view 1 and
    kept in view 2 and one the other way round; then filler buckets up to exactly M_target entries."""
    rnd = np.random.RandomState(seed)
    bk = []
    pos = 0

    def add(cnt, k1, k2):
        nonlocal pos
        bk.append((len(bk) + 1, cnt, k1, k2))
        pos += cnt

    add(32, 1, 1)                  # group 0 fully kept: offset at lane 0
    add(32, 0, 0)                  # group 1 fully dropped
    add(1, 1, 0)                   # group 2: lane 0 kept in view 1 only, the next bucket starts at lane 1
    add(29, 0, 1)                  # lanes 1..29; the next bucket starts at lane 30
    add(1, 0, 0)                   # lane 30
    add(1, 1, 1)                   # lane 31 alone, kept in both
    add(31, 0, 0)                  # group 3: only lane 31 kept
    add(1, 1, 1)
    add(2048 - pos % 2048, 1, 1)   # up to the next tile border
    add(2048, 0, 1)                # a whole tile dropped in view 1, kept in view 2
    add(2048, 1, 0)                # and the reverse
    while pos < M_target:
        cnt = int(min(M_target - pos, rnd.choice([1, 2, 30, 31, 32, 33, 63, 64, 65, 500, 1000])))
        add(cnt, int(rnd.rand() < 0.5), int(rnd.rand() < 0.5))
    return bk


def crafted_view_key(pool, r1, bk, seed):
    """z (small values: one digit each, in window 0) and the key's pool indices: a_query / b_query at infinity exactly for
    the variables of the buckets dropped in view 1 / view 2"""
    m = r1.num_variables
    M = sum(cnt for _, cnt, _, _ in bk)
    assert M <= m - 1 and len(bk) <= 512           # z values stay one digit in window 0 for any c >= 10
    rnd = np.random.RandomState(seed)
    vals = np.zeros(m, np.uint64)
    k1 = np.ones(m, bool)
    k2 = np.ones(m, bool)
    order = 1 + rnd.permutation(m - 1)[:M]          # which variables carry the entries (z[0] = 1 stays out of the plan)
    p = 0
    for d, cnt, a, b in bk:
        sel = order[p:p + cnt]
        vals[sel], k1[sel], k2[sel] = d, bool(a), bool(b)
        p += cnt
    z = np.zeros((m, 4), np.uint64)
    z[:, 0] = vals
    z[0, 0] = 1
    t = np.arange(m)
    ia = np.where(k1, t % POOL_K, POOL_K)
    ib = np.where(k2, (t // 3) % POOL_K, POOL_K)
    il = (t // 5) % (POOL_K + 1)
    ih = rnd.randint(0, POOL_K + 1, r1.domain_size - 1)
    return z, (ia, ib, il, ih)


VIEW_CASES = [(0, 16, 0), (0, 16, 1), (0, 16, 2047), (0, 14, 224), (1, 14, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("cid,log_n,rem", VIEW_CASES, ids=[f"{CURVES[c].name}-2^{k}-Mmod2048={m}" for c, k, m in VIEW_CASES])
def test_view_compaction(gpu_lib, oracle_c, cid, log_n, rem):
    """M (entries of the z plan) = 2048 * tiles + rem (rem = 224: M mod 32 = 0 inside a tile); both z modes, with and
    without window tables; equal to the dlog prediction, and at 2^16 to the C oracle's prover."""
    cv = CURVES[cid]
    ctx = Context(cid, 0, gpu_lib)
    try:
        r1, _ = synthetic.make_layered(ctx, cv.name, (1 << log_n) - 2)
        m = r1.num_variables
        M = ((m - 1) // 2048 - 1) * 2048 + rem
        bk = view_layout(M, log_n + rem)
        assert sum(cnt for _, cnt, _, _ in bk) == M and M % 2048 == rem and M < m
        pool = Pool(cv, 70 + cid)
        z, idx = crafted_view_key(pool, r1, bk, log_n + rem)
        pk = key_bytes(pool, r1, idx)
        h = oracle_c.witness_map(cid, r1, z)
        want = expected_proof(pool, r1, z, idx, h, R, S)
        if log_n == 16 and rem == 0:
            assert oracle_c.prove(cid, pk, r1, z, R, S, cv.fq_bytes)[0] == want
        rh = ctx.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())
        for tables in (1, 0):
            ctx.set_option(OPT_TABLES, tables)
            ctx.set_option(OPT_TABLE_MIN_LOG, 4)
            pkh = ctx.pk_load(pk)
            for mode in (1, 2):
                ctx.set_option(OPT_Z_MODE, mode)
                assert ctx.prove(pkh, rh, z, R, S) == want, (tables, mode, ctx.pk_table_info(pkh))
            ctx.pk_free(pkh)
    finally:
        ctx.close()
