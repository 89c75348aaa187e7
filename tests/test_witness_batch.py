"""Batched witness generation and proving from inputs (zkb_prog_compute_witness_batch / zkb_prog_prove_batch): K input sets of
one program in one level sweep.

Every witness file of a batch must be byte-identical to zkb_prog_compute_witness (and the host interpreter) on the same inputs,
and every proof to zkb_prog_compute_witness + zkb_groth16_prove_resident with the same (r, s).  The CPU tier runs the engine
through the host emulation (tests/host_emu/libzkb_emu.so): every solver, random programs, the out-of-range `Bits` path, the
sha256packed program, unsatisfied sets, the refusals, the launch count, the untouched resident assignment, proofs on all three
curves below and above the 2^10 tile threshold, and the file-level tool.  The GPU tier (-m gpu) checks the same equalities on
the H100 at K up to 64 and proofs up to the 2^18 pipeline branch."""
import hashlib
import importlib.util
import io
import os
import random

import numpy as np
import pytest

from tests.test_prog_native import random_program, solver_program
from zokrates_b200 import backend, ir, rng as prng, sha256_circuit, witness_gpu, zir
from zokrates_b200._lib import OPT_BATCH_PASS_MAX, OPT_Z_MODE, Context, ZkbError, fr_array
from zokrates_b200.curves import curve as get_curve
from zokrates_b200.ir import Constraint, Directive, LinComb, Parameter, Prog, QuadComb, Variable
from zokrates_b200.proof import Proof, vk_from_pk_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V = Variable
TD = [5, 6, 7, 8, 99, 2, 3]
CURVES = [(0, "bn128"), (1, "bls12_381"), (2, "bls12_377")]
CID = {c: i for i, c in CURVES}
MAX = (1 << 64) - 1


def input_sets(curve, n_args, K, seed):
    """K - 1 distinct random input sets, then the first one again (K >= 2); K = 1: one set"""
    rnd = random.Random(seed)
    r = get_curve(curve).r
    sets = [[rnd.randrange(r) for _ in range(n_args)] for _ in range(max(K - 1, 1))]
    return (sets + [sets[0]])[:K]


def solver_sets(curve, width, K, seed):
    """input sets of solver_program(curve, width): x below 2^width (its Bits recomposition is checked)"""
    r = get_curve(curve).r
    sets = input_sets(curve, 3, K, seed)
    for x in sets:
        x[0] = x[0] % min(1 << width, r)
    return sets


def singles(ctx, h, sets, try_oor=False):
    return [ctx.prog_compute_witness(h, x, try_oor) for x in sets]


def check_batch(ctx, prog, sets, try_oor=False, interp=True):
    """the batch equals the single calls and the interpreter, set by set"""
    h = ctx.prog_load(zir.write_prog(prog))
    try:
        wits, first = ctx.prog_compute_witness_batch(h, sets, try_oor)
        assert first == [None] * len(sets)
        assert wits == singles(ctx, h, sets, try_oor)
        if interp:
            assert wits == [ir.Interpreter(try_oor).execute(prog, x).write() for x in sets]
    finally:
        ctx.prog_free(h)


def chain_program(curve, n):
    """a private and b public; t_1 = a * a, t_{i+1} = t_i * (t_i + b) for n - 1 rows, ~out_0 = t_n * 1, plus a Bits directive
    on a with its booleanity and recomposition checks (n + 10 constraints in all)"""
    a, b = V.new(0), V.new(1)
    st = [Constraint(QuadComb(LinComb.from_var(a), LinComb.from_var(a)), LinComb.from_var(V.new(2)))]
    for i in range(2, n):
        t = V.new(i)
        st.append(Constraint(QuadComb(LinComb.from_var(t), LinComb([(t, 1), (b, 1)])), LinComb.from_var(V.new(i + 1))))
    st.append(Constraint(QuadComb(LinComb.from_var(V.new(n)), LinComb.one()), LinComb.from_var(V.public(0))))
    bits = [V.new(n + 1 + i) for i in range(8)]
    st.append(Directive([QuadComb(LinComb.from_var(a), LinComb.one())], bits, "Bits", 8))
    for t in bits:
        st.append(Constraint(QuadComb(LinComb.from_var(t), LinComb.from_var(t)), LinComb.from_var(t)))
    return Prog([Parameter.private_(a), Parameter.public(b)], 1, st, curve)


def check_program(curve):
    """x private, y public: t = x * x, then the CHECK t == y (fails for y != x^2), and a ConditionEq directive on x - y"""
    r = get_curve(curve).r
    x, y, t, bb, inv = V.new(0), V.new(1), V.new(2), V.new(3), V.new(4)
    diff = LinComb([(x, 1), (y, r - 1)])
    return Prog([Parameter.private_(x), Parameter.public(y)], 1, [
        Directive([QuadComb(diff, LinComb.one())], [bb, inv], "ConditionEq"),
        Constraint(QuadComb(diff, LinComb.from_var(inv)), LinComb.from_var(bb)),
        ir.constraint(x, x, t),
        Constraint(QuadComb(LinComb.from_var(t), LinComb.one()), LinComb.from_var(y)),
        Constraint(QuadComb(LinComb([(t, 1), (bb, 3)]), LinComb.one()), LinComb.from_var(V.public(0)))], curve)


# ---- CPU tier -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu_ctx(emu_lib):
    return {cid: Context(cid, 0, emu_lib) for cid, _ in CURVES}


@pytest.mark.parametrize("cid,curve", CURVES, ids=[c for _, c in CURVES])
def test_emu_solver_program_batches(emu_ctx, cid, curve):
    """every solver; x == y in one set reaches ConditionEq's zero branch"""
    for width in (8, 254):
        prog = solver_program(curve, width)
        for K in (1, 2, 5):
            sets = solver_sets(curve, width, K, K + width)
            if K == 5:
                sets[2][1] = sets[2][0]
            check_batch(emu_ctx[cid], prog, sets)


@pytest.mark.parametrize("curve", ["bn128", "bls12_381", "bls12_377"])
def test_emu_random_program_batches(emu_ctx, curve):
    for seed in range(4):
        prog, inputs = random_program(curve, seed)
        for K in (1, 2, 5):
            sets = input_sets(curve, 3, K, seed)
            sets[0] = sets[-1] = inputs
            check_batch(emu_ctx[CID[curve]], prog, sets)


@pytest.mark.parametrize("curve", ["bn128", "bls12_381"])
def test_emu_out_of_range_bits_batches(emu_ctx, curve):
    """the flag applies to every set of the batch; the sets mix values whose x + r fits the bit length and values where it does not"""
    c = get_curve(curve)
    req = c.r.bit_length()
    x = V.new(0)
    bits = [V.new(1 + i) for i in range(req)]
    prog = Prog([Parameter.private_(x)], 0, [Directive([QuadComb(LinComb.from_var(x), LinComb.one())], bits, "Bits", req)] +
                [Constraint(QuadComb(LinComb([(t, pow(2, req - 1 - i, c.r)) for i, t in enumerate(bits)]), LinComb.one()),
                            LinComb.from_var(x))], curve)
    vals = [[5], [(1 << req) - c.r - 1], [(1 << req) - c.r], [c.r - 1], [5]]
    for K in (1, 2, 5):
        for oor in (True, False):
            check_batch(emu_ctx[CID[curve]], prog, vals[:K], try_oor=oor)


def sha_digest(inputs):
    d = hashlib.sha256(b"".join(int(v).to_bytes(16, "big") for v in inputs)).digest()
    return [int.from_bytes(d[:16], "big"), int.from_bytes(d[16:], "big")]


@pytest.fixture(scope="module")
def sha_program():
    prog = sha256_circuit.make_prog("bn128")
    return prog, zir.write_prog(prog)


def sha_check(lib, sha_program, sets):
    prog, data = sha_program
    ctx = Context(0, 0, lib)
    h = ctx.prog_load(data)
    try:
        wits, first = ctx.prog_compute_witness_batch(h, sets)
        assert first == [None] * len(sets)
        for k, (x, w) in enumerate(zip(sets, wits)):
            assert ir.Witness.read(w, "bn128").return_values() == sha_digest(x), k
        assert wits == singles(ctx, h, sets)
    finally:
        ctx.prog_free(h)


def test_emu_sha256_program_batch(emu_lib, sha_program):
    sha_check(emu_lib, sha_program, [[0, 0, 0, 5], [2 ** 128 - 1, 12345678901234567890, 0, 2 ** 127 + 99], [7, 8, 9, 10]])


def unsat_case(ctx, curve, K, bad):
    """K sets of check_program; the sets in `bad` violate the check t == y"""
    r = get_curve(curve).r
    rnd = random.Random(K)
    sets = []
    for k in range(K):
        xv = rnd.randrange(1, r)
        sets.append([xv, xv * xv % r if k not in bad else (xv * xv + 1 + k) % r])
    return sets


def check_unsat(ctx, curve, K, bad):
    prog = check_program(curve)
    sets = unsat_case(ctx, curve, K, bad)
    h = ctx.prog_load(zir.write_prog(prog))
    try:
        wits, first = ctx.prog_compute_witness_batch(h, sets)
        for k in range(K):
            if k in bad:
                with pytest.raises(ZkbError) as e:
                    ctx.prog_compute_witness(h, sets[k])
                assert e.value.code == 5
                assert first[k] == int(str(e.value).split("constraint ")[1].split()[0]) and wits[k] is None
            else:
                assert first[k] is None and wits[k] == ctx.prog_compute_witness(h, sets[k])
        # the raw call: ZKB_E_UNSAT, failing slots zero-filled
        lib = ctx.lib
        arr = np.stack([fr_array(x) for x in sets])
        ln = __import__("ctypes").c_size_t(0)
        size = len(wits[min(set(range(K)) - set(bad))])
        out = np.full(K * size, 0xAB, dtype=np.uint8)
        fu = np.zeros(K, dtype=np.uint64)
        assert lib.dll.zkb_prog_compute_witness_batch(ctx.h, h, K, arr.ctypes.data, 2, 0, out.ctypes.data, K * size,
                                                      __import__("ctypes").byref(ln), fu.ctypes.data) == 5
        assert ln.value == size
        for k in range(K):
            chunk = out[k * size:(k + 1) * size]
            assert (not chunk.any()) if k in bad else chunk.tobytes() == wits[k]
            assert (int(fu[k]) == MAX) == (k not in bad)
    finally:
        ctx.prog_free(h)
    return prog, sets


def test_emu_unsatisfied_sets(emu_ctx):
    ctx = emu_ctx[0]
    prog, sets = check_unsat(ctx, "bn128", 5, {1, 3})
    with pytest.raises(ir.UnsatisfiedConstraint, match="input set 1: constraint"):
        witness_gpu.generate_witnesses(prog, sets, ctx=ctx)


@pytest.fixture(scope="module")
def bn_keyed(emu_ctx):
    """chain_program(200) on BN254 loaded with a key from the fixed trapdoor"""
    ctx = emu_ctx[0]
    prog = chain_program("bn128", 200)
    h = ctx.prog_load(zir.write_prog(prog))
    info = ctx.prog_info(h)
    pk_bytes = ctx.setup(info["r1cs"], TD)
    return ctx, prog, h, info, pk_bytes, ctx.pk_load(pk_bytes)


def test_emu_refusals(emu_ctx, emu_lib, bn_keyed):
    import ctypes as C
    ctx = emu_ctx[0]
    prog = solver_program("bn128", 8)
    h = ctx.prog_load(zir.write_prog(prog))
    good = solver_sets("bn128", 8, 3, 1)
    size = len(ctx.prog_compute_witness(h, good[0]))

    def raw(sets, n, cap):
        arr = np.stack([fr_array(x) for x in sets]) if sets and n else np.zeros((1, 1, 4), dtype=np.uint64)
        out = np.zeros(max(cap, 1), dtype=np.uint8)
        fu = np.zeros(max(len(sets), 1), dtype=np.uint64)
        return emu_lib.dll.zkb_prog_compute_witness_batch(ctx.h, h, len(sets), arr.ctypes.data, n, 0, out.ctypes.data, cap,
                                                          C.byref(C.c_size_t(0)), fu.ctypes.data)
    assert raw([], 3, 0) == 1                                                 # K = 0
    assert raw([x[:2] for x in good], 2, 3 * size) == 1                       # wrong input count
    r = get_curve("bn128").r
    assert raw(good[:2] + [[1, 2, r]], 3, 3 * size) == 1                      # non-canonical input in the last set
    assert raw(good, 3, 3 * size - 1) == 1                                    # witness buffer one byte short
    assert raw(good, 3, 3 * size) == 0
    with pytest.raises(ZkbError, match="WrongInputCount"):
        ctx.prog_compute_witness_batch(h, [[1, 2]])
    ctx.prog_free(h)
    # an unschedulable program: ZKB_E_FORMAT like the single call
    x, y, t = V.new(0), V.new(1), V.new(2)
    hb = ctx.prog_load(zir.write_prog(Prog([Parameter.private_(x)], 0, [ir.constraint(t, x, y)], "bn128")))
    with pytest.raises(ZkbError, match="no value yet") as e:
        ctx.prog_compute_witness_batch(hb, [[3], [4]])
    assert e.value.code == 2
    ctx.prog_free(hb)
    # an unsupported directive (a Zir solver) when the parser keeps it
    hz = ctx.prog_load(zir.write_prog(Prog([Parameter.private_(x)], 0, [Directive([QuadComb(LinComb.from_var(x), LinComb.one())], [y], "Zir", None)], "bn128")))
    if ctx.prog_info(hz)["unsupported_directives"]:
        with pytest.raises(ZkbError, match="no device path"):
            ctx.prog_compute_witness_batch(hz, [[3], [4]])
        with pytest.raises(NotImplementedError):
            witness_gpu.generate_witnesses(Prog([Parameter.private_(x)], 0, [Directive([QuadComb(LinComb.from_var(x), LinComb.one())], [y], "Zir", None)], "bn128"), [[3]], ctx=ctx)
    ctx.prog_free(hz)
    with pytest.raises(ValueError, match="WrongInputCount"):
        witness_gpu.generate_witnesses(prog, [[1, 2, 3], [1, 2]], ctx=ctx)
    # prog_prove_batch: a key share of a 2-way sharded key, a proof in flight, a key of another circuit
    ctx, prog, h, info, pk_bytes, pk = bn_keyed
    sets = input_sets("bn128", 2, 2, 9)
    with pytest.raises(ZkbError) as e:
        ctx.prog_prove_batch(h, ctx.pk_load(pk_bytes, 0, 2), sets, [1, 2], [3, 4])
    assert e.value.code == 1
    ctx.prog_compute_witness(h, sets[0])
    want = ctx.prove_resident(pk, info["r1cs"], 5, 6)
    t = ctx.prove_submit(pk, info["r1cs"], None, 5, 6)
    with pytest.raises(ZkbError) as e:
        ctx.prog_prove_batch(h, pk, sets, [1, 2], [3, 4])
    assert e.value.code == 1
    assert ctx.prove_collect(t) == want
    other = chain_program("bn128", 300)
    ho = ctx.prog_load(zir.write_prog(other))
    pko = ctx.pk_load(ctx.setup(ctx.prog_info(ho)["r1cs"], TD))
    with pytest.raises(ZkbError) as e:
        ctx.prog_prove_batch(h, pko, sets, [1, 2], [3, 4])
    assert e.value.code == 1
    with pytest.raises(ZkbError) as e:
        ctx.prog_prove_batch(h, pk, [], [], [])
    assert e.value.code == 1
    ctx.prog_free(ho)


def test_emu_launch_count(emu_ctx, bn_keyed):
    """the witness sweep's launches do not grow with K; proving from inputs launches at most what prove_batch launches plus
    the witness sweep of one set"""
    ctx = emu_ctx[0]
    prog = solver_program("bn128", 8)
    h = ctx.prog_load(zir.write_prog(prog))

    def launches(fn):
        before = ctx.launch_count()
        fn()
        return ctx.launch_count() - before
    l1 = launches(lambda: ctx.prog_compute_witness_batch(h, solver_sets("bn128", 8, 1, 0)))
    l6 = launches(lambda: ctx.prog_compute_witness_batch(h, solver_sets("bn128", 8, 6, 0)))
    assert l1 == l6 and l1 >= ctx.prog_info(h)["levels"]
    ctx.prog_free(h)
    ctx, prog, h, info, _, pk = bn_keyed
    sets = input_sets("bn128", 2, 6, 3)
    zs = []
    for x in sets:
        ctx.prog_compute_witness(h, x)
        zs.append(ctx.prog_assignment(h))
    sweep = launches(lambda: ctx.prog_compute_witness(h, sets[0]))
    pb = launches(lambda: ctx.prove_batch(pk, info["r1cs"], zs, list(range(1, 7)), list(range(7, 13))))
    ppb = launches(lambda: ctx.prog_prove_batch(h, pk, sets, list(range(1, 7)), list(range(7, 13))))
    assert ppb <= pb + sweep, (ppb, pb, sweep)


def test_emu_resident_state_untouched(bn_keyed):
    ctx, prog, h, info, _, pk = bn_keyed
    sets = input_sets("bn128", 2, 3, 4)
    ctx.prog_compute_witness(h, sets[0])
    z, pub, proof = ctx.prog_assignment(h), ctx.prog_public_inputs(h), ctx.prove_resident(pk, info["r1cs"], 9, 10)
    ctx.prog_compute_witness_batch(h, sets[1:])
    ctx.prog_prove_batch(h, pk, sets[1:], [1, 2], [3, 4])
    assert np.array_equal(ctx.prog_assignment(h), z) and ctx.prog_public_inputs(h) == pub
    assert ctx.prove_resident(pk, info["r1cs"], 9, 10) == proof


def check_prove_batch(ctx, h, info, pk, sets, rs, ss):
    got, first = ctx.prog_prove_batch(h, pk, sets, rs, ss)
    assert first == [None] * len(sets)
    for k, x in enumerate(sets):
        ctx.prog_compute_witness(h, x)
        assert got[k] == (ctx.prove_resident(pk, info["r1cs"], rs[k], ss[k]), ctx.prog_public_inputs(h)), k
    return got


@pytest.mark.parametrize("n_constraints", [200, 1000], ids=["2^8", "2^10"])
@pytest.mark.parametrize("cid,curve", CURVES, ids=[c for _, c in CURVES])
def test_emu_prove_from_inputs_batch(emu_ctx, cid, curve, n_constraints):
    ctx = emu_ctx[cid]
    prog = chain_program(curve, n_constraints - 10)
    h = ctx.prog_load(zir.write_prog(prog))
    info = ctx.prog_info(h)
    pk_bytes = ctx.setup(info["r1cs"], TD)
    pk = ctx.pk_load(pk_bytes)
    try:
        for K in (1, 2, 5):
            sets = input_sets(curve, 2, K, K)
            got = check_prove_batch(ctx, h, info, pk, sets, [100 + k for k in range(K)], [200 + 3 * k for k in range(K)])
        if n_constraints == 200:
            c = get_curve(curve)
            assert backend.B200.verify(vk_from_pk_bytes(c, pk_bytes), Proof.from_raw(c, *got[1]))
    finally:
        ctx.prog_free(h)


@pytest.mark.parametrize("opts", [{OPT_BATCH_PASS_MAX: 2}, {OPT_Z_MODE: 1}, {OPT_Z_MODE: 2}], ids=["three_passes", "z_mode1", "z_mode2"])
def test_emu_prove_from_inputs_options(bn_keyed, opts):
    ctx, prog, h, info, _, pk = bn_keyed
    try:
        for k, v in opts.items():
            ctx.set_option(k, v)
        check_prove_batch(ctx, h, info, pk, input_sets("bn128", 2, 5, 11), [1, 2, 3, 4, 5], [6, 7, 8, 9, 10])
        check_unsat_proofs(ctx, pk)
    finally:
        ctx.set_option(OPT_BATCH_PASS_MAX, 0)
        ctx.set_option(OPT_Z_MODE, 0)


def check_unsat_proofs(ctx, pk=None):
    """unsatisfied sets of a proof batch: their first violated rows, empty slots; the other proofs are complete"""
    prog = check_program("bn128")
    h = ctx.prog_load(zir.write_prog(prog))
    info = ctx.prog_info(h)
    pk = ctx.pk_load(ctx.setup(info["r1cs"], TD))
    sets = unsat_case(ctx, "bn128", 5, {1, 3})
    try:
        got, first = ctx.prog_prove_batch(h, pk, sets, [1, 2, 3, 4, 5], [6, 7, 8, 9, 10])
        for k, x in enumerate(sets):
            if k in (1, 3):
                assert got[k] is None
                with pytest.raises(ZkbError):
                    ctx.prog_compute_witness(h, x)
                assert first[k] is not None
            else:
                ctx.prog_compute_witness(h, x)
                assert first[k] is None and got[k] == (ctx.prove_resident(pk, info["r1cs"], k + 1, k + 6), ctx.prog_public_inputs(h))
    finally:
        ctx.prog_free(h)


def test_emu_prove_from_inputs_batch_mirror(emu_lib):
    """prove_from_inputs_batch draws (r, s) proof after proof: sequential prove_from_inputs on the same rng gives the same proofs,
    for a program with directives and a directive-free one"""
    a, b = V.new(0), V.new(1)
    plain = Prog([Parameter.private_(a), Parameter.public(b)], 0, [ir.constraint(a, a, b)], "bn128")
    r = get_curve("bn128").r
    for prog, sets in ((chain_program("bn128", 40), input_sets("bn128", 2, 4, 2)),
                       (plain, [[x, x * x % r] for x in (337, 5, 0, 337)])):
        kp = backend.B200.setup(prog, TD, lib=emu_lib)
        got = witness_gpu.prove_from_inputs_batch(prog, sets, io.BytesIO(kp.pk), prng.get_rng_from_entropy("inputs"), lib=emu_lib)
        seq = prng.get_rng_from_entropy("inputs")
        want = [witness_gpu.prove_from_inputs(prog, x, io.BytesIO(kp.pk), seq, lib=emu_lib) for x in sets]
        assert [p.to_tagged_json() for p in got] == [p.to_tagged_json() for p in want]
        assert [w.write() for w in witness_gpu.generate_witnesses(prog, sets, lib=emu_lib)] == \
            [ir.Interpreter().execute(prog, x).write() for x in sets]


@pytest.fixture
def emu_default_library(emu_lib, monkeypatch):
    from zokrates_b200 import _lib
    monkeypatch.setattr(_lib, "_default", emu_lib)
    monkeypatch.setattr(backend, "_contexts", {})
    return emu_lib


def _tool():
    spec = importlib.util.spec_from_file_location("zkb_compute_witness", os.path.join(ROOT, "tools", "zkb_compute_witness.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    return tool


def test_emu_tool_arguments_file(emu_default_library, tmp_path):
    tool = _tool()
    prog = solver_program("bn128", 8)
    (tmp_path / "out").write_bytes(zir.write_prog(prog))
    sets = solver_sets("bn128", 8, 3, 5)
    (tmp_path / "args.txt").write_text("".join(" ".join(map(str, x)) + "\n" for x in sets))
    assert tool.main(["-i", str(tmp_path / "out"), "--arguments-file", str(tmp_path / "args.txt"), "--witness-dir",
                      str(tmp_path / "w"), "--json"]) == 0
    for k, x in enumerate(sets):
        assert tool.main(["-i", str(tmp_path / "out"), "-o", str(tmp_path / f"single{k}"), "-a", *map(str, x), "--json"]) == 0
        assert (tmp_path / "w" / f"witness_{k}").read_bytes() == (tmp_path / f"single{k}").read_bytes()
        assert (tmp_path / "w" / f"witness_{k}.json").read_text() == (tmp_path / f"single{k}.json").read_text()
    # a failing line exits non-zero and names its line
    cprog = check_program("bn128")
    (tmp_path / "cout").write_bytes(zir.write_prog(cprog))
    (tmp_path / "bad.txt").write_text("3 9\n3 10\n")
    with pytest.raises(SystemExit, match="line 2"):
        tool.main(["-i", str(tmp_path / "cout"), "--arguments-file", str(tmp_path / "bad.txt"), "--witness-dir", str(tmp_path / "b")])


# ---- GPU tier -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_sha256_program_batch(gpu_lib, sha_program):
    rnd = random.Random(64)
    sets = [[0, 0, 0, 5]] + [[rnd.randrange(1 << 128) for _ in range(4)] for _ in range(64)]
    sha_check(gpu_lib, sha_program, sets)


@pytest.mark.gpu
def test_gpu_batches_equal_single_calls(gpu_lib):
    for cid, curve in CURVES:
        ctx = Context(cid, 0, gpu_lib)
        for K in (1, 7, 64):
            check_batch(ctx, solver_program(curve, 254), solver_sets(curve, 254, K, K), interp=K < 64)
            check_batch(ctx, random_program(curve, 100 + cid, n=200)[0], input_sets(curve, 3, K, K), interp=K < 64)


@pytest.mark.gpu
def test_gpu_unsatisfied_sets(gpu_lib):
    check_unsat(Context(0, 0, gpu_lib), "bn128", 64, {1, 3, 17, 40, 63})


@pytest.mark.gpu
@pytest.mark.parametrize("n_constraints", [(1 << 16) - 4, (1 << 18) - 4], ids=["2^16", "2^18"])
def test_gpu_prove_from_inputs(gpu_lib, n_constraints):
    """a 2^16 domain: the witness sweep writes the batched prover's buffers; a 2^18 domain: the two-slot pipeline branch"""
    ctx = Context(0, 0, gpu_lib)
    c = get_curve("bn128")
    prog = chain_program("bn128", n_constraints - 8)
    h = ctx.prog_load(zir.write_prog(prog))
    info = ctx.prog_info(h)
    pk_bytes = ctx.setup(info["r1cs"], TD)
    pk = ctx.pk_load(pk_bytes)
    try:
        for K in (16, 4):
            sets = input_sets("bn128", 2, K, K)
            got = check_prove_batch(ctx, h, info, pk, sets, [31 + k for k in range(K)], [41 + k for k in range(K)])
        assert backend.B200.verify(vk_from_pk_bytes(c, pk_bytes), Proof.from_raw(c, *got[2]))
    finally:
        ctx.prog_free(h)
