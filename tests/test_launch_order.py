"""No kernel may depend on the order in which the device runs its threads and blocks.

The host emulation (tests/host_emu/libzkb_emu.so, zokrates_b200/csrc/rt.cuh) runs every launch in ascending thread order by
default, and its atomics follow that order.  A race inside a launch then always resolves in the writer's favour, and the
bucket ranks always equal the point index order, so a kernel that reads another thread's output of the same launch, or a
schedule that puts a reader in its writer's level, still passes there and fails on the device.  Here the same constructions
as the rest of the CPU tier run with the emulation's threads, blocks and block-phase threads in descending order and in
seeded pseudo-random orders (zkb_emu_launch_order, exported by the emulation build only), and every result must equal the
independent answer the original test uses: the C oracle, the trapdoor prediction, the dlog prediction of the k*G pool, the
Python interpreter, or (where the original compares two device paths) the ascending run.  The exceptional MSMs take more
seeds, because there the order decides which special branch of the XYZZ addition meets a duplicate or negated point."""
import contextlib
import ctypes

import numpy as np
import pytest

from oracle.ff import BLS12_381, BN254
from tests import bls12_377_ref as B
from tests.test_batch_prove import RS, TD, Circuit, set_options
from tests.test_gm17_scale import TD6, circuit, load, mask_cases, predict
from tests.test_gpu_exceptional import (OPT_CHUNK_TARGET, Crafted, Pool, check_tiny, prove_modes, run_msm_cases)
from tests.test_prog_native import check_program, random_program, solver_program
from tests.test_witness_batch import (check_batch, check_prove_batch, check_unsat, chain_program, input_sets, sha_check,
                                      solver_sets)
from zokrates_b200 import sha256_circuit, synthetic, witness_gpu, zir
from zokrates_b200._lib import (OPT_BATCH_AFFINE, OPT_BATCH_AFFINE_MIN_LOG, OPT_BATCH_PASS_MAX, OPT_TABLE_C, OPT_TABLE_MIN_LOG,
                                OPT_TABLES, OPT_Z_MODE, Context)
from zokrates_b200.r1cs import synthesize

ASCENDING, DESCENDING, SEEDED = 0, 1, 2          # rt.cuh EMU_ORDER_*
ORDERS = [(ASCENDING, 0), (DESCENDING, 0)] + [(SEEDED, s) for s in (1, 2, 3)]
MANY = ORDERS + [(SEEDED, s) for s in (4, 5, 6, 7, 8, 9)]       # 9 seeds for the exceptional MSMs


def order_id(o):
    return {ASCENDING: "ascending", DESCENDING: "descending"}.get(o[0], f"seed{o[1]}")


_current = [(ASCENDING, 0)]


def set_order(lib, mode, seed):
    fn = lib.dll.zkb_emu_launch_order
    fn.argtypes, fn.restype = [ctypes.c_uint32, ctypes.c_uint64], ctypes.c_int32
    st = fn(mode, seed)
    if st == 0:
        _current[0] = (mode, seed)
    return st


@pytest.fixture
def order(request, emu_lib):
    """Runs the test under launch order request.param; ascending again afterwards (emu_lib is shared by the session)."""
    assert set_order(emu_lib, *request.param) == 0
    yield request.param
    assert set_order(emu_lib, ASCENDING, 0) == 0


@contextlib.contextmanager
def ascending(lib):
    """Reference values built inside a test: ascending order, then back to the test's order."""
    current = _current[0]
    assert set_order(lib, ASCENDING, 0) == 0
    try:
        yield
    finally:
        assert set_order(lib, *current) == 0


def orders(lst=ORDERS):
    return pytest.mark.parametrize("order", lst, ids=[order_id(o) for o in lst], indirect=True)


def test_order_setter_refuses_unknown_modes(emu_lib):
    assert set_order(emu_lib, 3, 0) == 1                             # ZKB_E_ARG; the order stays ascending


# ---- Groth16 ---------------------------------------------------------------------------------------------------------
CURVES = [(0, BN254), (1, BLS12_381), (2, B.C)]
TD7 = [3, 5, 7, 11, 1234567, 17, 19]


class Keyed:
    """A synthetic circuit with a key from TD7 and its trapdoor prediction for (r, s) = RS[0].  BN254 and BLS12-381 take the
    key and the prediction from the C oracle; BLS12-377 (no C oracle) sets up in the emulation and predicts with
    tests/bls12_377_ref.py."""

    def __init__(self, ctx, oracle_c, cid, c, n_constraints):
        self.r1, self.z = synthetic.make(c.name, n_constraints)
        self.h = ctx.r1cs_load(self.r1.num_constraints, self.r1.num_instance, self.r1.num_witness, self.r1.matrices())
        if cid == 2:
            self.pk = ctx.setup(self.h, TD7)
            self.want = B.expected_proof_csr(self.r1, B.ark.Trapdoor(*TD7), self.z, *RS[0])
        else:
            self.pk = oracle_c.setup(cid, self.r1, TD7)
            self.want = oracle_c.trapdoor_expected(cid, self.r1, TD7, self.z, *RS[0], c.fq_bytes)


@pytest.fixture(scope="module")
def keyed(emu_lib, oracle_c):
    """(cid, n_constraints) -> (context, Keyed), built on first use under ascending order"""
    ctxs, cache = {}, {}

    def get(cid, n):
        if (cid, n) not in cache:
            if cid not in ctxs:
                ctxs[cid] = Context(cid, 0, emu_lib)
            with ascending(emu_lib):
                cache[(cid, n)] = (ctxs[cid], Keyed(ctxs[cid], oracle_c, cid, CURVES[cid][1], n))
        return cache[(cid, n)]
    return get


@orders()
@pytest.mark.parametrize("cid", [0, 1, 2], ids=[c.name for _, c in CURVES])
def test_groth16_proofs(keyed, order, cid):
    """Below (2^8: register NTT passes) and above (2^10: tile passes) the tile threshold, and 3-way sharded partials."""
    for n in (200, 1000):
        ctx, k = keyed(cid, n)
        pkh = ctx.pk_load(k.pk)
        assert ctx.prove(pkh, k.h, k.z, *RS[0]) == k.want, n
        if n == 200:
            parts = [ctx.prove_partial(ctx.pk_load(k.pk, rank, 3), k.h, k.z) for rank in range(3)]
            assert ctx.finalize(pkh, np.concatenate(parts), 3, *RS[0]) == k.want
        ctx.pk_free(pkh)


@orders()
def test_groth16_msm_modes(keyed, order):
    """BN254 at 2^10: window tables forced on (ZKB_OPT_Z_MODE 1: shared buckets over the tables, 2: per-window buckets) and
    off (both z modes)."""
    ctx, k = keyed(0, 1000)
    try:
        for tables in (2, 0):
            set_options(ctx, {OPT_TABLES: tables, OPT_TABLE_MIN_LOG: 4})
            pkh = ctx.pk_load(k.pk)
            assert ctx.pk_table_info(pkh)["z_tables"] == ("built" if tables == 2 else "disabled")
            for mode in (1, 2):
                ctx.set_option(OPT_Z_MODE, mode)
                assert ctx.prove(pkh, k.h, k.z, *RS[0]) == k.want, (tables, mode)
            ctx.pk_free(pkh)
    finally:
        set_options(ctx, {OPT_TABLES: 1, OPT_TABLE_MIN_LOG: 14, OPT_Z_MODE: 0})


@orders()
def test_groth16_setup_key_bytes(keyed, order, oracle_c):
    ctx, k = keyed(0, 200)
    assert ctx.setup(k.h, TD7) == k.pk


@pytest.fixture(scope="module")
def batch_circuit(emu_lib, oracle_c):
    """The five assignments of test_batch_prove on a BN254 2^10 circuit and their single proofs in ascending order; the
    satisfying one (uniform) equals the trapdoor prediction."""
    assert set_order(emu_lib, ASCENDING, 0) == 0
    ctx = Context(0, 0, emu_lib)
    cc = Circuit(ctx, "bn128", 1000, pk_bytes=oracle_c.setup(0, synthetic.make("bn128", 1000)[0], TD))
    singles = [cc.single(k) for k in range(5)]
    assert singles[0] == oracle_c.trapdoor_expected(0, cc.r1, TD, cc.zs[0], *RS[0], BN254.fq_bytes)
    return cc, singles


@orders()
def test_groth16_batch_three_passes(batch_circuit, order):
    """K = 5 in three passes (ZKB_OPT_BATCH_PASS_MAX = 2)."""
    cc, singles = batch_circuit
    try:
        cc.ctx.set_option(OPT_BATCH_PASS_MAX, 2)
        got = cc.ctx.prove_batch(cc.pk, cc.h, cc.zs, [r for r, _ in RS[:5]], [s for _, s in RS[:5]])
        assert got == singles
    finally:
        cc.ctx.set_option(OPT_BATCH_PASS_MAX, 0)


# ---- GM17 ------------------------------------------------------------------------------------------------------------
@orders()
def test_gm17_setup_and_prove(emu_lib, oracle_c, order):
    """BN254 at a SAP domain of 2^11 (adversarial assignment): the device key proves the trapdoor-predicted bytes."""
    ctx = Context(0, 0, emu_lib)
    r1, z = circuit(ctx, BN254, "least", 11, "adversarial")
    rh = load(ctx, r1)
    pkh = ctx.gm17_pk_load(ctx.gm17_setup(rh, TD6))
    m = mask_cases(BN254, 11)["random"]
    assert ctx.gm17_prove(pkh, rh, z, *m) == predict(oracle_c, 0, BN254, r1, z, m)
    ctx.close()


# ---- the exceptional MSMs of tests/test_gpu_exceptional.py -----------------------------------------------------------
@orders(MANY)
@pytest.mark.parametrize("cid,c", [(0, BN254), (1, BLS12_381)], ids=["bn128", "bls12_381"])
def test_exceptional_msms(emu_lib, order, cid, c):
    """2051 G1 and 259 G2 points from the k*G pool: duplicates, (P, -P) pairs, infinity runs, equal bucket sums, zero sums;
    the order of the additions inside a bucket follows the permuted ranks."""
    ctx = Context(cid, 0, emu_lib)
    pool = Pool(c, 11 + cid)
    run_msm_cases(ctx, pool, 1, 2051, [{}, {OPT_BATCH_AFFINE: 3, OPT_BATCH_AFFINE_MIN_LOG: 0, OPT_CHUNK_TARGET: 1000}], 2051)
    run_msm_cases(ctx, pool, 2, 259, [{}], 259)
    ctx.close()


@orders(MANY)
def test_exceptional_tiny_key(emu_lib, oracle_c, order):
    check_tiny(Context(0, 0, emu_lib), oracle_c, 0, BN254)


@pytest.fixture(scope="module")
def crafted(emu_lib, oracle_c):
    ctx = Context(0, 0, emu_lib)
    return ctx, Crafted(ctx, oracle_c, 0, BN254, (1 << 10) - 2)


@orders(MANY)
def test_exceptional_crafted_proof(crafted, order):
    """The crafted 2^10 key with window tables (c = 16), in both z modes."""
    ctx, cr = crafted
    ctx.set_option(OPT_TABLE_MIN_LOG, 0)
    try:
        prove_modes(ctx, cr, [({OPT_TABLE_C: 16}, [{OPT_Z_MODE: 1}, {OPT_Z_MODE: 2}])], shards=())
    finally:
        set_options(ctx, {OPT_TABLE_MIN_LOG: 14, OPT_TABLES: 1, OPT_TABLE_C: 0, OPT_Z_MODE: 0})


# ---- witness generation ----------------------------------------------------------------------------------------------
@orders()
def test_witness_solver_and_random_programs(emu_lib, order):
    """The solver program and random programs, single (witness file equals the interpreter's) and batched (K = 5)."""
    check_program(emu_lib, solver_program("bn128", 254), [2 ** 200 + 12345, 99, 3])
    ctx = Context(0, 0, emu_lib)
    sets = solver_sets("bn128", 8, 5, 13)
    sets[2][1] = sets[2][0]
    check_batch(ctx, solver_program("bn128", 8), sets)
    for seed in range(3):
        prog, inputs = random_program("bn128", seed)
        check_program(emu_lib, prog, inputs)
        sets = input_sets("bn128", 3, 5, seed)
        sets[0] = sets[-1] = inputs
        check_batch(ctx, prog, sets)
    ctx.close()


@pytest.fixture(scope="module")
def sha_program():
    prog = sha256_circuit.make_prog("bn128")
    return prog, zir.write_prog(prog)


@orders()
def test_witness_sha256_program(emu_lib, order, sha_program):
    """sha256packed (28 k solver directives over many levels), batched; each digest equals hashlib's."""
    sha_check(emu_lib, sha_program, [[0, 0, 0, 5], [2 ** 128 - 1, 12345678901234567890, 0, 2 ** 127 + 99]])


@orders()
def test_witness_unsatisfied_sets(emu_lib, order):
    """The first violated row of each failing set of a batch."""
    check_unsat(Context(0, 0, emu_lib), "bn128", 5, {1, 3})


@pytest.fixture(scope="module")
def chain_keyed(emu_lib, oracle_c):
    """chain_program (one level per row) on BN254 with a C-oracle key, and its batch proofs in ascending order."""
    assert set_order(emu_lib, ASCENDING, 0) == 0
    ctx = Context(0, 0, emu_lib)
    prog = chain_program("bn128", 190)
    h = ctx.prog_load(zir.write_prog(prog))
    info = ctx.prog_info(h)
    pk = ctx.pk_load(oracle_c.setup(0, synthesize(prog), TD))
    sets, rs, ss = input_sets("bn128", 2, 5, 5), [100 + k for k in range(5)], [200 + 3 * k for k in range(5)]
    want = check_prove_batch(ctx, h, info, pk, sets, rs, ss)
    return ctx, h, info, pk, sets, rs, ss, want


@orders()
def test_prog_prove_batch(chain_keyed, order):
    """zkb_prog_prove_batch: witness generation and proofs of K = 5 input sets equal the ascending run (itself equal to the
    single calls), also in three passes."""
    ctx, h, info, pk, sets, rs, ss, want = chain_keyed
    assert ctx.prog_prove_batch(h, pk, sets, rs, ss) == (want, [None] * 5)
    try:
        ctx.set_option(OPT_BATCH_PASS_MAX, 2)
        assert ctx.prog_prove_batch(h, pk, sets, rs, ss) == (want, [None] * 5)
    finally:
        ctx.set_option(OPT_BATCH_PASS_MAX, 0)


@orders()
def test_witness_eval_and_first_violated_row(emu_lib, order):
    """zkb_witness_eval recomputes a synthetic circuit level by level; zkb_r1cs_check reports the first violated row
    (an atomic minimum) exactly, with violations spread over many rows of one launch."""
    ctx = Context(0, 0, emu_lib)
    n = 300
    r1, z = synthetic.make("bn128", n, seed=11)
    h = ctx.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())
    m0 = r1.num_variables - n
    level_ptr, rows, out_var = witness_gpu.levelize(r1, range(m0))
    z0 = z.copy()
    z0[m0:] = 0
    assert np.array_equal(ctx.witness_eval(h, z0, level_ptr, rows, out_var), z)
    assert ctx.r1cs_check(h) is None
    for cols in ([m0 + n // 2], [m0 + n - 1, m0 + 7, m0 + n // 3], list(range(m0 + 40, m0 + n, 13))):
        bad = z.copy()
        for col in cols:
            bad[col, 0] ^= np.uint64(1)
        want = next(i for i in range(n) if not row_holds(r1, bad, i))
        assert ctx.r1cs_check(h, bad) == want, cols
    ctx.close()


def row_holds(r1, z, i):
    """(A z)_i (B z)_i == (C z)_i, in Python integers"""
    r = BN254.r
    zi = [int(w[0]) | int(w[1]) << 64 | int(w[2]) << 128 | int(w[3]) << 192 for w in z]

    def dot(m):
        ptr, col, val = m
        return sum(zi[col[e]] * (int(val[e][0]) | int(val[e][1]) << 64 | int(val[e][2]) << 128 | int(val[e][3]) << 192)
                   for e in range(int(ptr[i]), int(ptr[i + 1]))) % r
    return dot(r1.a) * dot(r1.b) % r == dot(r1.c)
