"""No proof may depend on when its streams run.

A proof runs on up to six streams (main, witness map, one tail per MSM, a finish stream per proof slot, the optional plan
stream, and in the multi-GPU exchange the caller's), and two proofs may be in flight on one context.  What orders them is the
engine's Event record / wait / sync calls and the rule that the host reads pinned memory only after a sync.  The host
emulation runs every operation when it is issued by default, so a missing wait can never show there, and on the device one
schedule nearly always wins.  Here the same constructions as the rest of the CPU tier run with the emulation's streams
deferred (zkb_emu_stream_order, exported by the emulation build only, rt.cuh): LAZY runs only the dependency closure of
whatever the host needs, SEEDED runs ready queue heads in seeded random interleavings, and both hand out poisoned (nonzero)
fresh device and pinned memory.  Every result must equal the independent answer the original test uses: the C oracle's
trapdoor prediction (BN254, BLS12-381), tests/bls12_377_ref.py (BLS12-377), the dlog prediction of the k*G pool, the C
oracle's NTT and witness map, or the Python interpreter.

The GPU tier runs the stream-ordered paths that have no other test (the no-host-sync chain exchange, the plan stream, a
resident-assignment write inside an open proof, other work between submit and collect) once each at real sizes."""
import contextlib
import ctypes

import numpy as np
import pytest

from oracle.ff import BN254
from tests import bls12_377_ref as B
from tests.test_batch_prove import RS, TD, reassign, set_options
from tests.test_gm17_scale import TD6, circuit, load, mask_cases, predict
from tests.test_gpu_exceptional import K as POOL_K, Pool
from tests.test_launch_order import CURVES, TD7
from tests.test_witness_batch import chain_program, input_sets
from zokrates_b200 import ir, synthetic, witness_gpu, zir
from zokrates_b200._lib import (OPT_BATCH_PASS_MAX, OPT_TABLE_MIN_LOG, OPT_TABLES, OPT_Z_MODE, Context, ZkbError, fr_array)
from zokrates_b200.distributed import wm_chain_mask
from zokrates_b200.r1cs import synthesize

EAGER, LAZY, SEEDED = 0, 1, 2              # rt.cuh EMU_STREAMS_*
POISON = 1                                 # rt.cuh EMU_STREAM_POISON
OPT_PLAN_STREAM = 12                       # include/zkb.h ZKB_OPT_PLAN_STREAM
NO_HOST_SYNC = 0x80000000                  # chain_mask flag: the caller orders the exchange with stream events
POLICIES = [(EAGER, 0), (LAZY, 0)] + [(SEEDED, s) for s in (1, 2, 3)]
DEFERRED = POLICIES[1:]
TWO = [(LAZY, 0), (SEEDED, 1)]             # the 2^10 runs (tile NTT passes), which cost four times the 2^8 ones


def policy_id(p):
    return {EAGER: "eager", LAZY: "lazy"}.get(p[0], f"seed{p[1]}")


_current = [(EAGER, 0)]


def set_policy(lib, mode, seed):
    fn = lib.dll.zkb_emu_stream_order
    fn.argtypes, fn.restype = [ctypes.c_uint32, ctypes.c_uint64, ctypes.c_uint32], ctypes.c_int32
    st = fn(mode, seed, POISON if mode != EAGER else 0)
    if st == 0:
        _current[0] = (mode, seed)
    return st


def stats(lib):
    fn = lib.dll.zkb_emu_stream_stats
    fn.argtypes, fn.restype = [ctypes.POINTER(ctypes.c_uint64)], ctypes.c_int32
    out = (ctypes.c_uint64 * 2)()
    assert fn(out) == 0
    return {"reordered": int(out[0]), "peak_queued": int(out[1])}


@pytest.fixture
def policy(request, emu_lib):
    """Runs the test under stream policy request.param; eager again afterwards (emu_lib is shared by the session)."""
    assert set_policy(emu_lib, *request.param) == 0
    yield request.param
    assert set_policy(emu_lib, EAGER, 0) == 0


@contextlib.contextmanager
def eager(lib):
    """Reference values built inside a test: eager streams, then back to the test's policy."""
    current = _current[0]
    assert set_policy(lib, EAGER, 0) == 0
    try:
        yield
    finally:
        assert set_policy(lib, *current) == 0


def policies(lst=POLICIES):
    return pytest.mark.parametrize("policy", lst, ids=[policy_id(p) for p in lst], indirect=True)


def test_policy_setter_refuses_unknown_modes(emu_lib):
    fn = emu_lib.dll.zkb_emu_stream_order
    fn.argtypes, fn.restype = [ctypes.c_uint32, ctypes.c_uint64, ctypes.c_uint32], ctypes.c_int32
    assert fn(3, 0, 0) == 1 and fn(1, 0, 2) == 1                    # ZKB_E_ARG; the policy stays eager


# ---- Groth16 circuits with three satisfying assignments ----------------------------------------------------------------
class Keyed:
    """A synthetic circuit, three satisfying assignments of it and a key from TD7; want(i, j) is the trapdoor prediction for
    assignment i and (r, s) = RS[j] (C oracle for BN254 and BLS12-381, tests/bls12_377_ref.py for BLS12-377, whose key comes
    from the emulation's setup)."""

    def __init__(self, ctx, oracle_c, cid, c, n_constraints):
        self.cid, self.c, self.oracle_c = cid, c, oracle_c
        self.r1, z = synthetic.make(c.name, n_constraints)
        self.m0 = self.r1.num_variables - self.r1.num_constraints
        rnd = np.random.RandomState(n_constraints + cid)
        self.zs = [z] + [reassign(self.r1, z, [int(v) % c.r for v in rnd.randint(1, 1 << 62, size=self.m0 - 1)]) for _ in range(2)]
        assert all(not np.array_equal(self.zs[i], self.zs[j]) for i, j in ((0, 1), (0, 2), (1, 2)))   # else a case can go vacuous
        self.h = ctx.r1cs_load(self.r1.num_constraints, self.r1.num_instance, self.r1.num_witness, self.r1.matrices())
        self.pk_bytes = ctx.setup(self.h, TD7) if cid == 2 else oracle_c.setup(cid, self.r1, TD7)
        self.pk = ctx.pk_load(self.pk_bytes)
        self._want = {}

    def want(self, i, j):
        if (i, j) not in self._want:
            if self.cid == 2:
                self._want[(i, j)] = B.expected_proof_csr(self.r1, B.ark.Trapdoor(*TD7), self.zs[i], *RS[j])
            else:
                self._want[(i, j)] = self.oracle_c.trapdoor_expected(self.cid, self.r1, TD7, self.zs[i], *RS[j], self.c.fq_bytes)
        return self._want[(i, j)]


@pytest.fixture(scope="module")
def keyed(emu_lib, oracle_c):
    """(cid, n_constraints) -> (context, Keyed), built on first use under eager streams"""
    ctxs, cache = {}, {}

    def get(cid, n):
        if (cid, n) not in cache:
            with eager(emu_lib):
                if cid not in ctxs:
                    ctxs[cid] = Context(cid, 0, emu_lib)
                cache[(cid, n)] = (ctxs[cid], Keyed(ctxs[cid], oracle_c, cid, CURVES[cid][1], n))
        return cache[(cid, n)]
    return get


def two_in_flight(ctx, k, pk):
    """Two proofs with different z and (r, s) in flight, collected last-first, then first-first."""
    t0 = ctx.prove_submit(pk, k.h, k.zs[1], *RS[1])
    t1 = ctx.prove_submit(pk, k.h, k.zs[2], *RS[2])
    assert ctx.prove_collect(t1) == k.want(2, 2)
    assert ctx.prove_collect(t0) == k.want(1, 1)
    t0 = ctx.prove_submit(pk, k.h, k.zs[2], *RS[3])
    t1 = ctx.prove_submit(pk, k.h, k.zs[0], *RS[4])
    assert ctx.prove_collect(t0) == k.want(2, 3)
    assert ctx.prove_collect(t1) == k.want(0, 4)


def pipeline(ctx, k, pk, count=6):
    """A rolling pipeline: proof i is submitted before proof i - 1 is collected, host and resident assignments alternate,
    so both slots are reused with the other one busy."""
    prev = None
    for i in range(count):
        zi = i % 3
        if i % 2:
            ctx.set_assignment(k.h, k.zs[zi])
            t = ctx.prove_submit(pk, k.h, None, *RS[i])
        else:
            t = ctx.prove_submit(pk, k.h, k.zs[zi], *RS[i])
        if prev:
            assert ctx.prove_collect(prev[0]) == k.want(*prev[1]), prev
        prev = (t, (zi, i))
    assert ctx.prove_collect(prev[0]) == k.want(*prev[1]), prev


@policies()
@pytest.mark.parametrize("cid", [0, 1, 2], ids=[c.name for _, c in CURVES])
def test_two_proofs_in_flight(keyed, policy, cid):
    """Below the tile threshold of the transforms (2^8: register NTT passes)."""
    ctx, k = keyed(cid, 200)
    two_in_flight(ctx, k, k.pk)
    pipeline(ctx, k, k.pk)


@policies(TWO)
@pytest.mark.parametrize("cid", [0, 1, 2], ids=[c.name for _, c in CURVES])
def test_two_proofs_in_flight_tiled(keyed, policy, cid):
    """Above the tile threshold (2^10: shared-memory tile passes)."""
    ctx, k = keyed(cid, 1000)
    two_in_flight(ctx, k, k.pk)
    pipeline(ctx, k, k.pk)


@policies(TWO)
def test_two_proofs_in_flight_msm_modes(keyed, policy):
    """BN254 at 2^10: window tables forced on and off, each with ZKB_OPT_Z_MODE 1 (shared buckets) and 2 (per window)."""
    ctx, k = keyed(0, 1000)
    try:
        for tables in (2, 0):
            set_options(ctx, {OPT_TABLES: tables, OPT_TABLE_MIN_LOG: 4})
            pk = ctx.pk_load(k.pk_bytes)
            for mode in (1, 2):
                ctx.set_option(OPT_Z_MODE, mode)
                two_in_flight(ctx, k, pk)
            ctx.pk_free(pk)
    finally:
        set_options(ctx, {OPT_TABLES: 1, OPT_TABLE_MIN_LOG: 14, OPT_Z_MODE: 0})


@policies()
def test_plan_stream(keyed, policy):
    """ZKB_OPT_PLAN_STREAM = 1: the z digit plan on its own stream, ordered into the main stream by an event; 2^10 under two
    deferred policies."""
    for n in (200, 1000) if policy in TWO else (200,):
        ctx, k = keyed(0, n)
        try:
            ctx.set_option(OPT_PLAN_STREAM, 1)
            two_in_flight(ctx, k, k.pk)
            pipeline(ctx, k, k.pk)
        finally:
            ctx.set_option(OPT_PLAN_STREAM, 0)


# ---- writers of the resident assignment while a proof that reads it is open -------------------------------------------
def open_proof_forms(ctx, pk, h, want_open, want_next, set_first, write, rs_open, rs_next):
    """A proof of the resident assignment (set_first()) is begun, write() replaces the resident assignment, the proof is
    finished: it must be the proof of the assignment it began with, and the next resident proof that of the new one.  Three
    forms: begin_async .. end_async, the legacy begin .. end, and submit .. collect."""
    set_first()
    t, _, _ = ctx.prove_begin_async(pk, h, None, 7)
    write()
    ctx.prove_end_async(t)
    assert ctx.finalize(pk, ctx.prove_collect_partial(t), 1, *rs_open) == want_open, "begin_async"
    assert ctx.prove_resident(pk, h, *rs_next) == want_next, "begin_async: next"
    set_first()
    ctx.prove_begin(pk, h, None, 7)
    write()
    assert ctx.finalize(pk, ctx.prove_end(pk, h), 1, *rs_open) == want_open, "begin"
    assert ctx.prove_resident(pk, h, *rs_next) == want_next, "begin: next"
    set_first()
    t = ctx.prove_submit(pk, h, None, *rs_open)
    write()
    assert ctx.prove_collect(t) == want_open, "submit"
    assert ctx.prove_resident(pk, h, *rs_next) == want_next, "submit: next"


@policies()
def test_resident_writers_inside_an_open_proof(keyed, policy):
    """zkb_r1cs_set_assignment, zkb_r1cs_check(z) and zkb_witness_eval each overwrite the resident assignment."""
    ctx, k = keyed(0, 200)
    level_ptr, rows, out_var = witness_gpu.levelize(k.r1, range(k.m0))
    z0 = k.zs[2].copy()
    z0[k.m0:] = 0

    def witness_eval():
        assert np.array_equal(ctx.witness_eval(k.h, z0, level_ptr, rows, out_var), k.zs[2])

    writers = {"set_assignment": lambda: ctx.set_assignment(k.h, k.zs[2]),
               "r1cs_check": lambda: ctx.r1cs_check(k.h, k.zs[2]) is None or pytest.fail("r1cs_check"),
               "witness_eval": witness_eval}
    for name, write in writers.items():
        open_proof_forms(ctx, k.pk, k.h, k.want(1, 0), k.want(2, 1), lambda: ctx.set_assignment(k.h, k.zs[1]), write, RS[0], RS[1])


@policies([(LAZY, 0)])
def test_resident_writers_inside_an_open_proof_tiled(keyed, policy):
    """The same at 2^10 (tile NTT passes), under the policy that catches a missing order here."""
    ctx, k = keyed(0, 1000)
    open_proof_forms(ctx, k.pk, k.h, k.want(1, 0), k.want(2, 1), lambda: ctx.set_assignment(k.h, k.zs[1]),
                     lambda: ctx.set_assignment(k.h, k.zs[2]), RS[0], RS[1])


def chain_case(ctx, oracle_c):
    """chain_program on BN254 with a C-oracle key and two distinct input sets, their assignments and witness files by the
    interpreter: (r1cs, program handle, R1CS handle, key handle, sets, witness files, assignments)"""
    prog = chain_program("bn128", 190)
    r1 = synthesize(prog)
    h = ctx.prog_load(zir.write_prog(prog))
    pk = ctx.pk_load(oracle_c.setup(0, r1, TD))
    sets = input_sets("bn128", 2, 3, 9)[:2]          # K = 3: two distinct sets, then the first again
    wits = [ir.Interpreter().execute(prog, x) for x in sets]
    zs = [r1.assignment(w) for w in wits]
    files = [w.write() for w in wits]
    assert sets[0] != sets[1] and files[0] != files[1] and not np.array_equal(zs[0], zs[1])   # else the case goes vacuous
    return r1, h, ctx.prog_info(h)["r1cs"], pk, sets, files, zs


def program_writers(ctx, oracle_c, case):
    """zkb_prog_set_witness and zkb_prog_compute_witness overwrite the program's resident assignment inside an open proof."""
    r1, h, rh, pk, sets, files, zs = case
    want = [[oracle_c.trapdoor_expected(0, r1, TD, z, *RS[j], BN254.fq_bytes) for j in range(2)] for z in zs]

    def compute():
        assert ctx.prog_compute_witness(h, sets[1]) == files[1]

    for write in (lambda: ctx.prog_set_witness(h, files[1]), compute):
        open_proof_forms(ctx, pk, rh, want[0][0], want[1][1], lambda: ctx.prog_set_witness(h, files[0]), write, RS[0], RS[1])


@pytest.fixture(scope="module")
def chain_prog(emu_lib, oracle_c):
    with eager(emu_lib):
        ctx = Context(0, 0, emu_lib)
        return (ctx,) + chain_case(ctx, oracle_c)


@policies()
def test_program_writers_inside_an_open_proof(chain_prog, oracle_c, policy):
    ctx, *case = chain_prog
    program_writers(ctx, oracle_c, case)


# ---- other work on the context between submit and collect --------------------------------------------------------------
@pytest.fixture(scope="module")
def quiet(emu_lib, keyed, oracle_c):
    """What the interleaved calls must return, each computed alone on a context of its own under eager streams."""
    _, k = keyed(0, 200)
    with eager(emu_lib):
        ctx = Context(0, 0, emu_lib)
        h = ctx.r1cs_load(k.r1.num_constraints, k.r1.num_instance, k.r1.num_witness, k.r1.matrices())
        gm17 = ctx.gm17_setup(h, TD6)
        ctx.close()
    rnd = np.random.RandomState(4)
    pool = Pool(BN254, 21)
    msm = {}
    for g, n in ((1, 300), (2, 40)):
        idx = rnd.randint(0, POOL_K + 1, size=n)
        sc = fr_array([int(v) % BN254.r for v in rnd.randint(0, 1 << 62, size=n)])
        sc[::7] = 0
        msm[g] = (pool.raw[g][idx].tobytes(), sc, pool.point(g, pool.dlog_sum(idx, sc)))
    data = fr_array([int(v) for v in rnd.randint(0, 1 << 62, size=512)])
    wm = oracle_c.witness_map(0, k.r1, k.zs[2])
    return {"gm17": gm17, "msm": msm, "ntt": (data, oracle_c.ntt(0, data)), "wm": wm}


@policies()
def test_other_work_between_submit_and_collect(keyed, quiet, policy):
    """Standalone G1 / G2 MSMs, zkb_ntt, Groth16 and GM17 setup, a second key with window tables and a proof under it, and
    zkb_witness_map (refused while slot 0 is busy, the oracle's witness map once slot 0 is free and slot 1 is not)."""
    ctx, k = keyed(0, 200)
    t = ctx.prove_submit(k.pk, k.h, k.zs[1], *RS[1])
    for g in (1, 2):
        pts, sc, want = quiet["msm"][g]
        assert ctx.msm(g, pts, sc) == want, g
    data, want = quiet["ntt"]
    assert np.array_equal(ctx.ntt(data), want)
    assert ctx.setup(k.h, TD7) == k.pk_bytes
    assert ctx.gm17_setup(k.h, TD6) == quiet["gm17"]
    try:
        set_options(ctx, {OPT_TABLES: 2, OPT_TABLE_MIN_LOG: 4})
        pk2 = ctx.pk_load(k.pk_bytes)
        assert ctx.pk_table_info(pk2)["z_tables"] == "built"
    finally:
        set_options(ctx, {OPT_TABLES: 1, OPT_TABLE_MIN_LOG: 14})
    assert ctx.prove(pk2, k.h, k.zs[2], *RS[2]) == k.want(2, 2)
    n = k.r1.domain_size
    with pytest.raises(ZkbError):
        ctx.witness_map(k.h, k.zs[2], n)                          # slot 0 holds t
    t2 = ctx.prove_submit(pk2, k.h, k.zs[0], *RS[3])             # slot 1
    assert ctx.prove_collect(t) == k.want(1, 1)
    assert np.array_equal(ctx.witness_map(k.h, k.zs[2], n), quiet["wm"])
    assert ctx.prove_collect(t2) == k.want(0, 3)
    ctx.pk_free(pk2)


# ---- the shared witness map of several ranks in one process --------------------------------------------------------------
def shared_wm_round(lib, ranks, k, world, form, ext=None):
    """Two proofs in flight on every rank (assignments 1 and 2), then the partials of each gathered and finalized.  ranks:
    (context, key shard, R1CS handle) per rank."""
    open_ = []
    for zi, j in ((1, 5), (2, 6)):
        flag = NO_HOST_SYNC if form == "stream" else 0
        tickets = [ctx.prove_begin_async(pk, h, k.zs[zi], wm_chain_mask(q, world) | flag) for q, (ctx, pk, h) in enumerate(ranks)]
        if form == "host":                     # every rank's own chains are in memory once begin returns
            for c in range(3):
                for q in range(world):
                    if q != c % world:
                        ctypes.memmove(tickets[q][1][c], tickets[c % world][1][c], tickets[q][2])
        else:
            for q, (ctx, _, _) in enumerate(ranks):
                ctx.prove_chains_to_stream(tickets[q][0], ext)
            copy = lib.dll.zkb_emu_stream_copy
            copy.argtypes, copy.restype = [ctypes.c_void_p] * 3 + [ctypes.c_uint64], ctypes.c_int32
            for c in range(3):
                for q in range(world):
                    if q != c % world:
                        assert copy(ext, tickets[q][1][c], tickets[c % world][1][c], tickets[q][2]) == 0
            for q, (ctx, _, _) in enumerate(ranks):
                ctx.prove_stream_to_finish(tickets[q][0], ext)
        for q, (ctx, _, _) in enumerate(ranks):
            ctx.prove_end_async(tickets[q][0])
        open_.append(((zi, j), tickets))
    for (zi, j), tickets in open_:
        parts = np.concatenate([ctx.prove_collect_partial(tickets[q][0]) for q, (ctx, _, _) in enumerate(ranks)])
        assert k.ctx_finalize(parts, world, j) == k.want(zi, j), (form, world, zi)


@pytest.fixture(scope="module")
def rank_ctxs(emu_lib, keyed):
    """world -> [(context, key shard, R1CS handle)] on the BN254 2^8 circuit, one context per rank"""
    _, k = keyed(0, 200)
    out = {}
    with eager(emu_lib):
        for world in (3, 4):
            ranks = []
            for q in range(world):
                ctx = Context(0, 0, emu_lib)
                h = ctx.r1cs_load(k.r1.num_constraints, k.r1.num_instance, k.r1.num_witness, k.r1.matrices())
                ranks.append((ctx, ctx.pk_load(k.pk_bytes, q, world), h))
            out[world] = ranks
    return out


@policies()
@pytest.mark.parametrize("world", [3, 4])
def test_shared_witness_map(emu_lib, keyed, rank_ctxs, policy, world):
    """The chains exchanged by the host after begin (host-sync form), then through an emulated caller stream that waits for
    every rank's chains, copies them (zkb_emu_stream_copy, standing in for the NCCL broadcasts) and is waited for by every
    rank's finish step (ZKB_CHAIN_NO_HOST_SYNC, zkb_groth16_prove_chains_to_stream / _stream_to_finish)."""
    ctx, k = keyed(0, 200)
    k.ctx_finalize = lambda parts, world_, j: ctx.finalize(k.pk, parts, world_, *RS[j])
    ranks = rank_ctxs[world]
    shared_wm_round(emu_lib, ranks, k, world, "host")
    create = emu_lib.dll.zkb_emu_stream_create
    create.argtypes, create.restype = [ctypes.POINTER(ctypes.c_void_p)], ctypes.c_int32
    destroy = emu_lib.dll.zkb_emu_stream_destroy
    destroy.argtypes, destroy.restype = [ctypes.c_void_p], ctypes.c_int32
    ext = ctypes.c_void_p()
    assert create(ctypes.byref(ext)) == 0
    try:
        shared_wm_round(emu_lib, ranks, k, world, "stream", ext.value)
    finally:
        assert destroy(ext.value) == 0


# ---- single-stream paths: the pinned and pageable copy rules -------------------------------------------------------------
@policies(DEFERRED)
def test_single_stream_paths(keyed, chain_prog, oracle_c, emu_lib, policy):
    """A K = 5 batch in three passes, zkb_prog_prove_batch, zkb_prog_compute_witness_batch and a GM17 proof."""
    ctx, k = keyed(0, 1000)
    try:
        ctx.set_option(OPT_BATCH_PASS_MAX, 2)
        zi = [0, 1, 2, 1, 0]
        got = ctx.prove_batch(k.pk, k.h, [k.zs[i] for i in zi], [r for r, _ in RS[:5]], [s for _, s in RS[:5]])
        assert got == [k.want(i, j) for j, i in enumerate(zi)]
    finally:
        ctx.set_option(OPT_BATCH_PASS_MAX, 0)
    pctx, r1, h, rh, pk, sets, files, zs = chain_prog
    rs, ss = [100, 101], [200, 203]
    proofs, first = pctx.prog_prove_batch(h, pk, sets, rs, ss)
    assert first == [None, None]
    for q in range(2):
        assert proofs[q][0] == oracle_c.trapdoor_expected(0, r1, TD, zs[q], rs[q], ss[q], BN254.fq_bytes), q
    assert pctx.prog_compute_witness_batch(h, sets) == (files, [None, None])
    gctx = Context(0, 0, emu_lib)
    r1g, zg = circuit(gctx, BN254, "least", 11, "uniform")
    rg = load(gctx, r1g)
    with eager(emu_lib):
        pkg = gctx.gm17_pk_load(gctx.gm17_setup(rg, TD6))
    m = mask_cases(BN254, 11)["random"]
    assert gctx.gm17_prove(pkg, rg, zg, *m) == predict(oracle_c, 0, BN254, r1g, zg, m)
    gctx.close()


# ---- the policy is live ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("policy", [(EAGER, 0), (LAZY, 0), (SEEDED, 1)], ids=["eager", "lazy", "seed1"], indirect=True)
def test_policy_is_live(keyed, emu_lib, policy):
    """Two proofs in flight: the deferred policies queue work and run some of it out of enqueue order, eager does neither."""
    ctx, k = keyed(0, 200)
    set_policy(emu_lib, *policy)                               # resets the statistics
    two_in_flight(ctx, k, k.pk)
    st = stats(emu_lib)
    if policy[0] == EAGER:
        assert st == {"reordered": 0, "peak_queued": 0}
    else:
        assert st["reordered"] > 0 and st["peak_queued"] > 1, st


# ---- GPU tier ----------------------------------------------------------------------------------------------------------------
class Full:
    """A BN254 synthetic circuit of 2^log_n rows on the GPU (make_layered), a second satisfying assignment (new inputs, the
    rest solved level by level on the device and checked), a GPU setup key and the C oracle's trapdoor predictions."""

    def __init__(self, ctx, oracle_c, log_n):
        self.ctx, self.oracle_c = ctx, oracle_c
        self.r1, z = synthetic.make_layered(ctx, "bn128", (1 << log_n) - 2)
        self.h = ctx.r1cs_load(self.r1.num_constraints, self.r1.num_instance, self.r1.num_witness, self.r1.matrices())
        m0 = self.r1.num_variables - self.r1.num_constraints
        z0 = z.copy()
        z0[1:m0] = fr_array([7 + 1000003 * q for q in range(1, m0)])
        z0[m0:] = 0
        self.z0, self.levels = z0, witness_gpu.levelize_wavefront(self.r1, range(m0))
        z2 = ctx.witness_eval(self.h, z0, *self.levels)
        assert ctx.r1cs_check(self.h, z2) is None and not np.array_equal(z2, z)
        self.zs = [z, z2]
        self.pk_bytes = ctx.setup(self.h, TD)
        self.pk = ctx.pk_load(self.pk_bytes)
        self._want = {}

    def want(self, i, j):
        if (i, j) not in self._want:
            self._want[(i, j)] = self.oracle_c.trapdoor_expected(0, self.r1, TD, self.zs[i], *RS[j], BN254.fq_bytes)
        return self._want[(i, j)]


@pytest.fixture(scope="module")
def full16(gpu_lib, oracle_c):
    ctx = Context(0, 0, gpu_lib)
    return ctx, Full(ctx, oracle_c, 16)


@pytest.fixture(scope="module")
def full20(gpu_lib, oracle_c):
    ctx = Context(0, 0, gpu_lib)
    return ctx, Full(ctx, oracle_c, 20)


def gpu_stream_exchange(gpu_lib, f, world):
    """world contexts on cuda:0, each with its key shard and two proofs in flight; the chains copied by torch on a side
    stream between zkb_groth16_prove_chains_to_stream and _stream_to_finish (ZKB_CHAIN_NO_HOST_SYNC)."""
    import torch
    from zokrates_b200.distributed import chain_tensor
    dev = torch.device("cuda", 0)
    ranks = []
    for q in range(world):
        ctx = Context(0, 0, gpu_lib)
        h = ctx.r1cs_load(f.r1.num_constraints, f.r1.num_instance, f.r1.num_witness, f.r1.matrices())
        ranks.append((ctx, ctx.pk_load(f.pk_bytes, q, world), h))
    stream = torch.cuda.Stream(device=dev)
    open_ = []
    for zi, j in ((0, 5), (1, 6)):
        tickets = [ctx.prove_begin_async(pk, h, f.zs[zi], wm_chain_mask(q, world) | NO_HOST_SYNC)
                   for q, (ctx, pk, h) in enumerate(ranks)]
        for q, (ctx, _, _) in enumerate(ranks):
            ctx.prove_chains_to_stream(tickets[q][0], stream.cuda_stream)
        with torch.cuda.stream(stream):
            for c in range(3):
                src = chain_tensor(tickets[c % world][1][c], tickets[0][2], dev)
                for q in range(world):
                    if q != c % world:
                        chain_tensor(tickets[q][1][c], tickets[q][2], dev).copy_(src)
        for q, (ctx, _, _) in enumerate(ranks):
            ctx.prove_stream_to_finish(tickets[q][0], stream.cuda_stream)
            ctx.prove_end_async(tickets[q][0])
        open_.append(((zi, j), tickets))
    for (zi, j), tickets in open_:
        parts = np.concatenate([ctx.prove_collect_partial(tickets[q][0]) for q, (ctx, _, _) in enumerate(ranks)])
        assert f.ctx.finalize(f.pk, parts, world, *RS[j]) == f.want(zi, j), (world, zi)
    torch.cuda.synchronize(dev)
    for ctx, _, _ in ranks:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [3, 4])
def test_gpu_stream_exchange_2_16(gpu_lib, full16, world):
    gpu_stream_exchange(gpu_lib, full16[1], world)


@pytest.mark.gpu
def test_gpu_stream_exchange_2_20(gpu_lib, full20):
    """The 2^20 - 2 benchmark circuit size, world 3 and world 4."""
    for world in (3, 4):
        gpu_stream_exchange(gpu_lib, full20[1], world)


@pytest.mark.gpu
def test_gpu_plan_stream_2_20(full20):
    ctx, f = full20
    try:
        ctx.set_option(OPT_PLAN_STREAM, 1)
        t0 = ctx.prove_submit(f.pk, f.h, f.zs[0], *RS[0])
        t1 = ctx.prove_submit(f.pk, f.h, f.zs[1], *RS[1])
        assert ctx.prove_collect(t0) == f.want(0, 0)
        assert ctx.prove_collect(t1) == f.want(1, 1)
    finally:
        ctx.set_option(OPT_PLAN_STREAM, 0)


@pytest.mark.gpu
def test_gpu_resident_write_inside_an_open_proof_2_20(full20):
    """zkb_r1cs_set_assignment, zkb_r1cs_check(z) and zkb_witness_eval (level by level, the second assignment) as writers."""
    ctx, f = full20

    def witness_eval():
        assert np.array_equal(ctx.witness_eval(f.h, f.z0, *f.levels), f.zs[1])

    for write in (lambda: ctx.set_assignment(f.h, f.zs[1]),
                  lambda: ctx.r1cs_check(f.h, f.zs[1]) is None or pytest.fail("r1cs_check"), witness_eval):
        open_proof_forms(ctx, f.pk, f.h, f.want(0, 2), f.want(1, 3), lambda: ctx.set_assignment(f.h, f.zs[0]), write, RS[2], RS[3])


@pytest.mark.gpu
def test_gpu_program_writers_inside_an_open_proof(gpu_lib, oracle_c):
    """zkb_prog_set_witness and zkb_prog_compute_witness on the device (the program of the CPU case)."""
    ctx = Context(0, 0, gpu_lib)
    program_writers(ctx, oracle_c, chain_case(ctx, oracle_c))
    ctx.close()


@pytest.mark.gpu
def test_gpu_other_work_between_submit_and_collect_2_16(full16, oracle_c):
    ctx, f = full16
    rnd = np.random.RandomState(5)
    pool = Pool(BN254, 22)
    t = ctx.prove_submit(f.pk, f.h, f.zs[1], *RS[1])
    for g, n in ((1, 1 << 14), (2, 1 << 10)):
        idx = rnd.randint(0, POOL_K + 1, size=n)
        sc = fr_array([int(v) % BN254.r for v in rnd.randint(0, 1 << 62, size=n)])
        assert ctx.msm(g, pool.raw[g][idx].tobytes(), sc) == pool.point(g, pool.dlog_sum(idx, sc)), g
    data = fr_array([int(v) for v in rnd.randint(0, 1 << 62, size=1 << 12)])
    assert np.array_equal(ctx.ntt(data), oracle_c.ntt(0, data))
    try:
        set_options(ctx, {OPT_TABLES: 2, OPT_TABLE_MIN_LOG: 4})
        pk2 = ctx.pk_load(f.pk_bytes)
    finally:
        set_options(ctx, {OPT_TABLES: 1, OPT_TABLE_MIN_LOG: 14})
    assert ctx.prove(pk2, f.h, f.zs[0], *RS[2]) == f.want(0, 2)
    n = 1 << 16
    with pytest.raises(ZkbError):
        ctx.witness_map(f.h, f.zs[0], n)
    t2 = ctx.prove_submit(pk2, f.h, f.zs[0], *RS[3])
    assert ctx.prove_collect(t) == f.want(1, 1)
    assert np.array_equal(ctx.witness_map(f.h, f.zs[0], n), oracle_c.witness_map(0, f.r1, f.zs[0]))
    assert ctx.prove_collect(t2) == f.want(0, 3)
    ctx.pk_free(pk2)
