"""Batched proving (zkb_groth16_prove_batch): K proofs of one circuit under one key in one GPU pass.

Every proof of a batch must be byte-identical to zkb_groth16_prove with the same assignment and (r, s).  The CPU tier runs
the engine through the host emulation (tests/host_emu/libzkb_emu.so) on synthetic circuits below and above the 2^10 tile
threshold of the transforms, under every option that changes the device path, and checks the refusals, the launch count
and the Python / file-level front doors.  The GPU tier (-m gpu) checks the same equality on the H100 from 2^10 to 2^20,
several passes, and a batch against the oracle's trapdoor prediction and the host pairing check."""
import importlib.util
import io
import os

import numpy as np
import pytest

from oracle.ff import BN254
from zokrates_b200 import backend, ir, rng as prng, synthetic, zir
from zokrates_b200._lib import (OPT_BATCH_PASS_MAX, OPT_NTT_KERNEL, OPT_NTT_TILE_MIN, OPT_TABLE_MIN_LOG, OPT_TABLES, OPT_Z_MODE,
                                Context, ZkbError, fr_array)
from zokrates_b200.curves import curve as get_curve
from zokrates_b200.proof import Proof, vk_from_pk_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TD = [5, 6, 7, 8, 99, 2, 3]
CURVES = [(0, "bn128"), (1, "bls12_381"), (2, "bls12_377")]


def assignments(curve, n_constraints):
    """The circuit and five assignments: uniform, bits-only, all-zero witness part, the uniform one again (the batch gives
    it different (r, s)), and bits again.  The prover is a fixed function of z, so an assignment need not satisfy the circuit
    for the batch to have to equal the single proofs."""
    r1, zu = synthetic.make(curve, n_constraints)
    _, zb = synthetic.make(curve, n_constraints, distribution="bits")
    z0 = zu.copy()
    z0[r1.num_instance:] = 0
    return r1, [zu, zb, z0, zu, zb]


RS = [(11 + k, 1000003 * (k + 1)) for k in range(8)]


class Circuit:
    def __init__(self, ctx, curve, n_constraints, pk_bytes=None):
        self.ctx = ctx
        self.r1, self.zs = assignments(curve, n_constraints)
        self.h = ctx.r1cs_load(self.r1.num_constraints, self.r1.num_instance, self.r1.num_witness, self.r1.matrices())
        self.pk_bytes = pk_bytes or ctx.setup(self.h, TD)
        self.pk = ctx.pk_load(self.pk_bytes)
        self._single = {}

    def single(self, k):
        """proof k of the reference sequence: assignment zs[k], (r, s) = RS[k], by zkb_groth16_prove"""
        if k not in self._single:
            self._single[k] = self.ctx.prove(self.pk, self.h, self.zs[k], *RS[k])
        return self._single[k]

    def check(self, ks, pk=None):
        got = self.ctx.prove_batch(pk or self.pk, self.h, [self.zs[k] for k in ks], [RS[k][0] for k in ks], [RS[k][1] for k in ks])
        assert got == [self.single(k) for k in ks]


def set_options(ctx, opts):
    for k, v in opts.items():
        ctx.set_option(k, v)


# ---- CPU tier -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu_ctx(emu_lib):
    return {cid: Context(cid, 0, emu_lib) for cid, _ in CURVES}


@pytest.mark.parametrize("n_constraints", [200, 1000], ids=["2^8", "2^10"])
@pytest.mark.parametrize("cid,curve", CURVES, ids=[c for _, c in CURVES])
def test_emu_batch_equals_single_proofs(emu_ctx, cid, curve, n_constraints):
    """K = 1, 2 and 5 against K single proofs; the 2^10 domain runs the tile passes, the 2^8 one the register passes."""
    cc = Circuit(emu_ctx[cid], curve, n_constraints)
    for ks in ([0], [1, 2], [0, 1, 2, 3, 4]):
        cc.check(ks)


@pytest.fixture(scope="module")
def bn_circuit(emu_ctx):
    return Circuit(emu_ctx[0], "bn128", 1000)


@pytest.mark.parametrize("opts", [{OPT_Z_MODE: 1}, {OPT_Z_MODE: 2}, {OPT_NTT_TILE_MIN: 64}, {OPT_NTT_TILE_MIN: 10, OPT_NTT_KERNEL: 1},
                                  {OPT_BATCH_PASS_MAX: 2}],
                         ids=["z_mode1", "z_mode2", "ntt_register", "ntt_tile", "three_passes"])
def test_emu_batch_options(bn_circuit, opts):
    ctx = bn_circuit.ctx
    try:
        set_options(ctx, opts)
        bn_circuit.check([0, 1, 2, 3, 4])
    finally:
        set_options(ctx, {OPT_Z_MODE: 0, OPT_NTT_TILE_MIN: 10, OPT_NTT_KERNEL: 2, OPT_BATCH_PASS_MAX: 0})


@pytest.mark.parametrize("tables", [0, 2])
def test_emu_batch_window_tables(bn_circuit, tables):
    """ZKB_OPT_TABLES 0 (no tables) and 2 (tables forced for this small key): the shared-bucket table mode and the per-window
    buckets, with the sparse/dense choice made from the batch's sample."""
    ctx = bn_circuit.ctx
    try:
        set_options(ctx, {OPT_TABLES: tables, OPT_TABLE_MIN_LOG: 4})
        pk = ctx.pk_load(bn_circuit.pk_bytes)
        assert ctx.pk_table_info(pk)["z_tables"] == ("built" if tables == 2 else "disabled")
        bn_circuit.check([0, 1, 2, 3, 4], pk=pk)
        for mode in (1, 2):
            ctx.set_option(OPT_Z_MODE, mode)
            bn_circuit.check([3, 1], pk=pk)
    finally:
        set_options(ctx, {OPT_TABLES: 1, OPT_TABLE_MIN_LOG: 14, OPT_Z_MODE: 0})


def test_emu_batch_key_with_infinities(bn_circuit):
    """The synthetic key has a_query / b_query points at infinity (variables that occur only in C), so the batch runs the
    filtered MSM views; every such point is skipped in every proof of the batch."""
    c = get_curve("bn128")
    pk = bn_circuit.pk_bytes
    g1, g2 = 2 * c.fq_bytes, 4 * c.fq_bytes
    off = g1 + 3 * g2
    ni = int.from_bytes(pk[off:off + 8], "little")
    off += 8 + ni * g1 + 2 * g1
    m = int.from_bytes(pk[off:off + 8], "little")
    a_inf = sum(pk[off + 8 + (i + 1) * g1 - 1] & 0x40 != 0 for i in range(m))
    assert 0 < a_inf < m
    bn_circuit.check([2, 0, 4])


def test_emu_batch_three_pair_key(emu_lib):
    """The 3-pair crafted key: duplicate and negated points, infinities in b_query, a domain of 4."""
    from tests.test_gpu_exceptional import Pool, tiny_crafted
    ctx = Context(0, 0, emu_lib)
    c = BN254
    r1, z, pk, _ = tiny_crafted(c, Pool(c, 5), [7, 7, c.r - 1])
    zs = [z, fr_array([1, 0, 0, 0]), fr_array([1, 3, c.r - 1, 5]), z]
    rh = ctx.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())
    pkh = ctx.pk_load(pk)
    rs = [r for r, _ in RS[:4]]
    ss = [s for _, s in RS[:4]]
    assert ctx.prove_batch(pkh, rh, zs, rs, ss) == [ctx.prove(pkh, rh, zs[k], rs[k], ss[k]) for k in range(4)]


def test_emu_batch_launches_do_not_scale_with_the_batch(bn_circuit):
    """One pass is one set of launches: K = 6 launches what K = 2 launches, except that the segmented reduction of the
    chunk-boundary partials (msm.cuh, msm_accum2_body) takes one more level per 4x more chunks, at most one per MSM for 3x
    the proofs.  A loop over the proofs would add four proofs' worth of launches."""
    cc = bn_circuit
    ctx = cc.ctx

    def launches(k):
        before = ctx.launch_count()
        cc.ctx.prove_batch(cc.pk, cc.h, [cc.zs[0]] * k, [1] * k, [2] * k)
        return ctx.launch_count() - before

    l2, l6 = launches(2), launches(6)
    before = ctx.launch_count()
    ctx.prove(cc.pk, cc.h, cc.zs[0], 1, 2)
    one = ctx.launch_count() - before
    assert l2 <= l6 <= l2 + 5, (l2, l6)
    assert l6 < l2 + one
    # a circuit where the partial reduction of every MSM takes as many levels for 6 proofs as for 2: equal launch counts
    small = Circuit(ctx, "bn128", 254)
    before = ctx.launch_count()
    ctx.prove_batch(small.pk, small.h, [small.zs[0]] * 2, [1, 1], [2, 2])
    s2 = ctx.launch_count() - before
    before = ctx.launch_count()
    ctx.prove_batch(small.pk, small.h, [small.zs[0]] * 6, [1] * 6, [2] * 6)
    assert ctx.launch_count() - before == s2


def test_emu_batch_refusals(bn_circuit, emu_lib):
    cc = bn_circuit
    ctx = cc.ctx
    with pytest.raises(ZkbError) as e:
        ctx.prove_batch(cc.pk, cc.h, [], [], [])
    assert e.value.code == 1
    # proofs_out one byte short of two proofs
    z = np.ascontiguousarray(np.stack([cc.zs[0], cc.zs[1]]), dtype=np.uint64)
    r, s = fr_array([1, 2]), fr_array([3, 4])
    out = np.zeros(2 * ctx.proof_bytes, dtype=np.uint8)
    assert emu_lib.dll.zkb_groth16_prove_batch(ctx.h, cc.pk, cc.h, 2, z.ctypes.data, r.ctypes.data, s.ctypes.data,
                                               out.ctypes.data, 2 * ctx.proof_bytes - 1) == 1
    # a key share of a 2-way sharded key
    with pytest.raises(ZkbError) as e:
        ctx.prove_batch(ctx.pk_load(cc.pk_bytes, 0, 2), cc.h, cc.zs[:2], [1, 2], [3, 4])
    assert e.value.code == 1
    # a key of another circuit
    other = Circuit(ctx, "bn128", 300)
    with pytest.raises(ZkbError) as e:
        ctx.prove_batch(other.pk, cc.h, cc.zs[:2], [1, 2], [3, 4])
    assert e.value.code == 1
    # a proof in flight: refused, and the in-flight proof still collects to its own bytes
    t = ctx.prove_submit(cc.pk, cc.h, cc.zs[1], *RS[1])
    with pytest.raises(ZkbError) as e:
        ctx.prove_batch(cc.pk, cc.h, cc.zs[:2], [1, 2], [3, 4])
    assert e.value.code == 1
    assert ctx.prove_collect(t) == cc.single(1)
    cc.check([0, 1])


def test_emu_generate_proofs_mirror(emu_lib):
    """B200.generate_proofs draws (r, s) proof after proof: the same tagged JSON as sequential generate_proof calls."""
    a, b = ir.Variable.new(0), ir.Variable.new(1)
    prog = ir.Prog([ir.Parameter.private_(a), ir.Parameter.public(b)], 0, [ir.constraint(a, a, b)], "bn128")
    r = get_curve("bn128").r
    witnesses = [ir.Interpreter().execute(prog, [x, x * x % r]) for x in (337, 5, 0, 337, r - 1)]
    kp = backend.B200.setup(prog, TD, lib=emu_lib)
    got = backend.B200.generate_proofs(prog, witnesses, io.BytesIO(kp.pk), prng.get_rng_from_entropy("batch"), lib=emu_lib)
    seq_rng = prng.get_rng_from_entropy("batch")
    want = [backend.B200.generate_proof(prog, w, io.BytesIO(kp.pk), seq_rng, lib=emu_lib) for w in witnesses]
    assert [p.to_tagged_json() for p in got] == [p.to_tagged_json() for p in want]
    assert all(backend.B200.verify(kp.vk, p) for p in got[:2])


@pytest.fixture
def emu_default_library(emu_lib, monkeypatch):
    """The file-level tool reaches the library through the process-wide default: point it at the host emulation."""
    from zokrates_b200 import _lib
    monkeypatch.setattr(_lib, "_default", emu_lib)
    monkeypatch.setattr(backend, "_contexts", {})
    return emu_lib


def test_emu_generate_proofs_files_and_tool(emu_default_library, tmp_path):
    """generate_proofs_files equals sequential generate_proof_files on an identically seeded rng, and
    `zkb_generate_proof.py --witnesses .. --proof-dir DIR` writes exactly those JSON files."""
    a, b = ir.Variable.new(0), ir.Variable.new(1)
    prog = ir.Prog([ir.Parameter.private_(a), ir.Parameter.public(b)], 0, [ir.constraint(a, a, b)], "bn128")
    out_bytes = zir.write_prog(prog)
    wits = [ir.Interpreter().execute(prog, [x, x * x]).write() for x in (3, 4, 3)]
    kp = backend.B200.setup(prog, TD)
    got = backend.B200.generate_proofs_files(out_bytes, wits, kp.pk, prng.get_rng_from_entropy("files"))
    seq_rng = prng.get_rng_from_entropy("files")
    want = [backend.B200.generate_proof_files(out_bytes, w, kp.pk, seq_rng) for w in wits]
    assert [p.to_tagged_json() for p in got] == [p.to_tagged_json() for p in want]

    paths = []
    for i, w in enumerate(wits):
        paths.append(tmp_path / f"witness{i}")
        paths[-1].write_bytes(w)
    (tmp_path / "out").write_bytes(out_bytes)
    (tmp_path / "proving.key").write_bytes(kp.pk)
    spec = importlib.util.spec_from_file_location("zkb_generate_proof", os.path.join(ROOT, "tools", "zkb_generate_proof.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    assert tool.main(["-i", str(tmp_path / "out"), "-p", str(tmp_path / "proving.key"), "--witnesses", *map(str, paths),
                      "--proof-dir", str(tmp_path / "proofs"), "-e", "files"]) == 0
    written = sorted(os.listdir(tmp_path / "proofs"))
    assert written == [f"proof_{i}.json" for i in range(len(wits))]
    assert [(tmp_path / "proofs" / f).read_text() for f in written] == [p.to_tagged_json() for p in want]


# ---- GPU tier -----------------------------------------------------------------------------------------------------
def random_assignments(c, m, ni, K, seed):
    """K assignments of m variables: uniform, 90 % {0, 1}, and all-zero witness parts in turn (z[0] = 1)."""
    rnd = np.random.RandomState(seed)
    zs = []
    for k in range(K):
        z = np.zeros((m, 4), dtype=np.uint64)
        kind = k % 3
        if kind == 0:
            z[:] = rnd.randint(0, 1 << 62, size=(m, 4), dtype=np.int64).astype(np.uint64)
            z[:, 3] &= np.uint64((1 << 60) - 1)
        elif kind == 1:
            z[:, 0] = (rnd.rand(m) < 0.5).astype(np.uint64)
            big = rnd.rand(m) < 0.1
            z[big, 0] = rnd.randint(0, 1 << 62, size=int(big.sum()), dtype=np.int64).astype(np.uint64)
        else:
            z[1:ni, 0] = rnd.randint(0, 1 << 62, size=ni - 1, dtype=np.int64).astype(np.uint64)
        z[0] = [1, 0, 0, 0]
        zs.append(z)
    return zs


def gpu_check(ctx, r1, zs, pk_bytes=None):
    h = ctx.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())
    pk = ctx.pk_load(pk_bytes or ctx.setup(h, TD))
    K = len(zs)
    rs = [1000 + 7 * k for k in range(K)]
    ss = [2000 + 13 * k for k in range(K)]
    got = ctx.prove_batch(pk, h, zs, rs, ss)
    want = [ctx.prove(pk, h, zs[k], rs[k], ss[k]) for k in range(K)]
    bad = [k for k in range(K) if got[k] != want[k]]
    assert not bad, bad
    return ctx, h, pk


@pytest.mark.gpu
@pytest.mark.parametrize("log_n,K", [(10, 64), (14, 64), (16, 16), (18, 8)])
def test_gpu_batch_bn254(gpu_lib, log_n, K):
    ctx = Context(0, 0, gpu_lib)
    r1, _ = synthetic.make_layered(ctx, "bn128", (1 << log_n) - 2)
    ctx2, h, pk = gpu_check(ctx, r1, random_assignments(get_curve("bn128"), r1.num_variables, r1.num_instance, K, log_n))
    if log_n == 14:   # the window tables are built from 2^14 pairs on (ZKB_OPT_TABLE_MIN_LOG) when HBM allows
        print("z tables:", ctx.pk_table_info(pk)["z_tables"])


@pytest.mark.gpu
@pytest.mark.parametrize("cid,curve", CURVES[1:], ids=[c for _, c in CURVES[1:]])
def test_gpu_batch_bls_curves(gpu_lib, cid, curve):
    ctx = Context(cid, 0, gpu_lib)
    r1, _ = synthetic.make_layered(ctx, curve, (1 << 12) - 2)
    gpu_check(ctx, r1, random_assignments(get_curve(curve), r1.num_variables, r1.num_instance, 8, cid))


@pytest.mark.gpu
def test_gpu_batch_several_passes_and_kernels(gpu_lib):
    """ZKB_OPT_BATCH_PASS_MAX = 3 over 8 proofs (three passes), and the register and round-1 tile transform paths."""
    ctx = Context(0, 0, gpu_lib)
    r1, _ = synthetic.make_layered(ctx, "bn128", (1 << 12) - 2)
    zs = random_assignments(get_curve("bn128"), r1.num_variables, r1.num_instance, 8, 7)
    ctx.set_option(OPT_BATCH_PASS_MAX, 3)
    _, h, pk = gpu_check(ctx, r1, zs)
    ctx.set_option(OPT_BATCH_PASS_MAX, 0)
    for opts in ({OPT_NTT_TILE_MIN: 64}, {OPT_NTT_KERNEL: 1}, {OPT_Z_MODE: 2}):
        set_options(ctx, opts)
        rs, ss = list(range(1, 9)), list(range(11, 19))
        assert ctx.prove_batch(pk, h, zs, rs, ss) == [ctx.prove(pk, h, zs[k], rs[k], ss[k]) for k in range(8)], opts
        set_options(ctx, {OPT_NTT_TILE_MIN: 10, OPT_NTT_KERNEL: 2, OPT_Z_MODE: 0})


def reassign(r1, z, inputs):
    """Another satisfying assignment of a `synthetic.make` circuit: new values for the input variables, every row's output
    variable solved from (A z)(B z) = C z (its C coefficient is 1 or r - 1, the other C terms come earlier)."""
    r = get_curve(r1.curve).r
    vals = [sum(int(x) << (64 * q) for q, x in enumerate(row)) for row in np.asarray(z)]
    m0 = r1.num_variables - r1.num_constraints
    vals[1:m0] = inputs
    mats = r1.matrices()

    def row(k, i):
        rp, col, val = mats[k]
        lo, hi = int(rp[i]), int(rp[i + 1])
        return [(int(col[e]), sum(int(x) << (64 * q) for q, x in enumerate(val[e]))) for e in range(lo, hi)]

    for i in range(r1.num_constraints):
        w = m0 + i
        a = sum(v * vals[j] for j, v in row(0, i)) % r
        b = sum(v * vals[j] for j, v in row(1, i)) % r
        cw, rest = 0, 0
        for j, v in row(2, i):
            if j == w:
                cw = v
            else:
                rest += v * vals[j]
        vals[w] = (a * b - rest) * pow(cw, -1, r) % r
    return fr_array(vals)


@pytest.mark.gpu
def test_gpu_batch_against_the_trapdoor(gpu_lib, oracle_c):
    """Four satisfying assignments of one 2^16 BN254 circuit in one batch: each proof equals the oracle's trapdoor
    prediction (independent of both prover paths) and passes the host pairing check."""
    c = get_curve("bn128")
    r1, z = synthetic.make("bn128", (1 << 16) - 2)
    m0 = r1.num_variables - r1.num_constraints
    rnd = np.random.RandomState(16)
    zs = [z] + [reassign(r1, z, [int(v) % c.r for v in rnd.randint(1, 1 << 62, size=m0 - 1)]) for _ in range(3)]
    ctx = Context(0, 0, gpu_lib)
    h = ctx.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())
    for zk in zs[1:]:
        assert ctx.r1cs_check(h, zk) is None
    pk_bytes = ctx.setup(h, TD)
    pk = ctx.pk_load(pk_bytes)
    rs, ss = [31, 32, 33, 34], [41, 42, 43, 44]
    got = ctx.prove_batch(pk, h, zs, rs, ss)
    vk = vk_from_pk_bytes(c, pk_bytes)
    for k in range(4):
        assert got[k] == oracle_c.trapdoor_expected(0, r1, TD, zs[k], rs[k], ss[k], c.fq_bytes), k
        inputs = [sum(int(x) << (64 * q) for q, x in enumerate(zs[k][1]))]
        assert backend.B200.verify(vk, Proof.from_raw(c, got[k], inputs)), k


@pytest.mark.gpu
def test_gpu_batch_2_20(gpu_lib):
    """2^20 constraints, K = 2: whichever path the size selects (the two-slot pipeline here), the single proofs' bytes."""
    ctx = Context(0, 0, gpu_lib)
    r1, _ = synthetic.make_layered(ctx, "bn128", (1 << 20) - 2)
    gpu_check(ctx, r1, random_assignments(get_curve("bn128"), r1.num_variables, r1.num_instance, 2, 20))
