"""Witness generation on the GPU for constraint-defined programs (SURVEY.md §8 rows a9–a11).

`zokrates compute-witness` runs `Interpreter::execute_with_log_stream`
(/root/reference/zokrates_interpreter/src/lib.rs:61-138) statement by statement: a constraint whose linear side is one
variable with coefficient one that has no value yet ASSIGNS it the value of the quadratic side, every other constraint is
CHECKED (`Error::UnsatisfiedConstraint`), directives call a solver.  The assignments form a dependency DAG; all statements
of one depth are independent, so the device evaluates the program level by level (`zkb_witness_eval`, one thread per
statement).  This module does the host part for constraint-only programs: it derives the levels from the R1CS rows (same rule,
same statement order for ties) and maps the result back to `ir.Witness`.  Programs with solver directives go through the
native front door (`zkb_prog_load` / `zkb_prog_compute_witness`: the library schedules constraints AND directives by level and
runs the solver kernels of csrc/solvers.cuh) — `generate_witness` and `prove_from_inputs` route them there.
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence, Tuple

import numpy as np

from ._lib import fr_array, fr_from_array
from .curves import curve as _curve
from .ir import Constraint, Directive, Prog, UnsatisfiedConstraint, Variable, Witness
from .r1cs import R1CS, synthesize

CHECK = 0xFFFFFFFF


def levelize(r1cs: R1CS, defined_cols: Iterable[int]) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(level_ptr, rows, out_var) for `zkb_witness_eval`.  `defined_cols`: columns that hold values before the first
    statement runs (the constant one and the program arguments)."""
    (ap, ac, _), (bp, bc, _), (cp, cc, cv) = r1cs.a, r1cs.b, r1cs.c
    m, N = r1cs.num_variables, r1cs.num_constraints
    level = np.full(m, -1, dtype=np.int64)
    for c in defined_cols:
        level[c] = 0
    row_level = np.zeros(N, dtype=np.int64)
    out_var = np.full(N, CHECK, dtype=np.uint32)
    one = np.array([1, 0, 0, 0], dtype=np.uint64)
    for k in range(N):
        quad = np.concatenate([ac[int(ap[k]):int(ap[k + 1])], bc[int(bp[k]):int(bp[k + 1])]])
        lin = cc[int(cp[k]):int(cp[k + 1])]
        if quad.size and level[quad].min() < 0:
            raise KeyError(f"constraint {k} reads a variable that has no value yet")
        base = int(level[quad].max()) if quad.size else 0
        if lin.size == 1 and level[lin[0]] < 0 and np.array_equal(cv[int(cp[k])], one):
            out_var[k] = lin[0]
            row_level[k] = base + 1
            level[lin[0]] = base + 1
        else:
            if lin.size and level[lin].min() < 0:
                raise KeyError(f"constraint {k} reads a variable that has no value yet")
            row_level[k] = max(base, int(level[lin].max()) if lin.size else 0) + 1
    order = np.argsort(row_level, kind="stable").astype(np.uint32)
    n_levels = int(row_level.max()) if N else 0
    counts = np.bincount(row_level, minlength=n_levels + 1)[1:]
    level_ptr = np.zeros(n_levels + 1, dtype=np.uint32)
    np.cumsum(counts, out=level_ptr[1:])
    return level_ptr, order, out_var[order]


def levelize_wavefront(r1cs: R1CS, defined_cols: Iterable[int], max_levels: int = 4096):
    """Same result as `levelize`, computed level by level with numpy (one O(nnz) sweep per level instead of a Python loop
    over the rows) — for circuits with many rows and few levels (the 2^20-constraint benchmark family has 64).  Returns None
    when the program is deeper than `max_levels` or when a row reads a variable no earlier row defines (use `levelize`)."""
    (ap, ac, _), (bp, bc, _), (cp, cc, cv) = r1cs.a, r1cs.b, r1cs.c
    m, N = r1cs.num_variables, r1cs.num_constraints
    if N == 0:
        return np.zeros(1, dtype=np.uint32), np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint32)
    ap, bp, cp = ap.astype(np.int64), bp.astype(np.int64), cp.astype(np.int64)
    level = np.full(m, -1, dtype=np.int64)
    level[np.fromiter(defined_cols, dtype=np.int64)] = 0
    one = np.array([1, 0, 0, 0], dtype=np.uint64)
    single = (cp[1:] - cp[:-1]) == 1
    first_c = np.where(single, cc[np.minimum(cp[:-1], len(cc) - 1)] if len(cc) else 0, 0).astype(np.int64)
    coeff_one = np.zeros(N, dtype=bool)
    if len(cc):
        coeff_one[single] = (cv[cp[:-1][single]] == one).all(axis=1)
    # a row ASSIGNS iff its linear side is one coefficient-one variable that no EARLIER row (and no input) defined:
    # the first such row in statement order wins, exactly as the sequential interpreter sees it
    cand = single & coeff_one & (level[first_c] < 0)
    out_var = np.full(N, CHECK, dtype=np.uint32)
    if cand.any():
        rows_c = np.flatnonzero(cand)
        _, first_idx = np.unique(first_c[rows_c], return_index=True)
        winners = rows_c[first_idx]
        out_var[winners] = first_c[winners].astype(np.uint32)
    assigns = out_var != CHECK
    # An assigning row must come BEFORE (in statement order) every row that reads its variable: the sequential interpreter
    # fails on a read of a variable that has no value yet (zokrates_interpreter/src/lib.rs:366-378 unwraps the lookup).  The
    # level recurrence alone would simply schedule such a reader after its writer, so check the order explicitly and leave
    # invalid programs to `levelize`, which raises like the reference.
    writer_row = np.full(m, -1, dtype=np.int64)          # -1: defined before the first statement (inputs, one)
    undefined = level < 0
    writer_row[undefined] = N                            # never written: any read is an error
    writer_row[out_var[assigns].astype(np.int64)] = np.flatnonzero(assigns)
    for ptr, cols, skip_own in ((ap, ac, False), (bp, bc, False), (cp, cc, True)):
        if not len(cols):
            continue
        reader = np.repeat(np.arange(N, dtype=np.int64), ptr[1:] - ptr[:-1])
        bad = writer_row[cols] >= reader
        if skip_own:                                     # the assigned variable itself sits on the linear side of its writer
            bad &= ~(assigns[reader] & (out_var[reader].astype(np.int64) == cols))
        if bad.any():
            return None

    def seg_max(ptr, cols):
        out = np.zeros(N, dtype=np.int64)
        lens = ptr[1:] - ptr[:-1]
        nz = lens > 0
        if len(cols) and nz.any():
            # reduceat over the NON-EMPTY rows only: their start offsets are strictly increasing and < len(cols), so each
            # segment is exactly one row (a clipped start index for a trailing empty row would cut the last term off the
            # preceding row)
            vals = level[cols]
            idx = ptr[:-1][nz]
            red = np.maximum.reduceat(vals, idx)
            mn = np.minimum.reduceat(vals, idx)
            out[nz] = np.where(mn < 0, -1, red)
        return out                                  # -1: some operand has no level yet; 0 for empty combinations

    row_level = np.full(N, -1, dtype=np.int64)
    pending = np.ones(N, dtype=bool)
    for lvl in range(1, max_levels + 1):
        qa, qb = seg_max(ap, ac), seg_max(bp, bc)
        ready = pending & (qa >= 0) & (qb >= 0)
        lin = seg_max(cp, cc)
        ready &= assigns | (lin >= 0)
        base = np.maximum(qa, qb)
        base = np.where(assigns, base, np.maximum(base, lin))
        ready &= base == lvl - 1                     # rows whose deepest operand sits exactly one level below
        if not ready.any():
            if not pending.any():
                break
            if not (pending & (qa >= 0) & (qb >= 0) & (assigns | (lin >= 0))).any():
                return None                          # something reads a variable nobody defines (or defined later)
            continue
        row_level[ready] = lvl
        pending &= ~ready
        w = ready & assigns
        level[out_var[w].astype(np.int64)] = lvl
        if not pending.any():
            break
    if pending.any():
        return None
    order = np.argsort(row_level, kind="stable").astype(np.uint32)
    n_levels = int(row_level.max())
    counts = np.bincount(row_level, minlength=n_levels + 1)[1:]
    if (counts == 0).any():
        return None
    level_ptr = np.zeros(n_levels + 1, dtype=np.uint32)
    np.cumsum(counts, out=level_ptr[1:])
    return level_ptr, order, out_var[order]


def levels_for(r1cs: R1CS, defined_cols) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """`levelize`, through the numpy wavefront for large shallow systems."""
    defined_cols = list(defined_cols)
    if r1cs.num_constraints > 2048:
        res = levelize_wavefront(r1cs, defined_cols)
        if res is not None:
            return res
    return levelize(r1cs, defined_cols)


def generate_witness(prog: Prog, inputs: Sequence[int], ctx=None, lib=None) -> Witness:
    """`Interpreter::execute` for a directive-free program, evaluated on the device.  Same result as `ir.Interpreter`
    (every variable of the constraint system gets its value) and the same failures: wrong input count, unsatisfied
    constraint."""
    from . import backend
    c = _curve(prog.curve)
    if len(inputs) != len(prog.arguments):
        raise ValueError(f"WrongInputCount: expected {len(prog.arguments)}, received {len(inputs)}")
    if any(isinstance(s, Directive) for s in prog.statements):
        return _generate_witness_native(prog, inputs, ctx, lib)
    r1cs = synthesize(prog)
    cols = {v: i for i, v in enumerate(r1cs.instance_vars)}
    cols.update({v: r1cs.num_instance + i for i, v in enumerate(r1cs.witness_vars)})
    vals = [0] * r1cs.num_variables
    vals[0] = 1
    for p, x in zip(prog.arguments, inputs):
        vals[cols[p.id]] = int(x) % c.r
    level_ptr, rows, out_var = levels_for(r1cs, [0] + [cols[p.id] for p in prog.arguments])
    ctx = ctx or backend.context(c, 0, lib)
    h = ctx.r1cs_load(r1cs.num_constraints, r1cs.num_instance, r1cs.num_witness, r1cs.matrices())
    try:
        if len(level_ptr) > 1:
            from ._lib import ZkbError
            try:
                z = ctx.witness_eval(h, fr_array(vals), level_ptr, rows, out_var)
            except ZkbError as e:
                if e.code == 5:
                    raise UnsatisfiedConstraint(str(e))
                raise
            vals = fr_from_array(z)
    finally:
        ctx.r1cs_free(h)
    w = Witness(curve=c)
    for v, col in cols.items():
        w.insert(v, vals[col])
    return w


def _generate_witness_native(prog: Prog, inputs: Sequence[int], ctx=None, lib=None, try_out_of_range: bool = False) -> Witness:
    """Programs with solver directives: the program file goes to the library, which schedules every statement and runs the
    solver kernels (same failures: UnsatisfiedConstraint; a solver without a device path — Zir functions — raises
    NotImplementedError)."""
    from . import backend, zir
    from ._lib import ZkbError
    c = _curve(prog.curve)
    ctx = ctx or backend.context(c, 0, lib)
    with ctx.lock:
        h = ctx.prog_load(zir.write_prog(prog))
        try:
            if ctx.prog_info(h)["unsupported_directives"]:
                raise NotImplementedError("the program calls a solver that has no device path: use ir.Interpreter")
            try:
                data = ctx.prog_compute_witness(h, [int(x) % c.r for x in inputs], try_out_of_range)
            except ZkbError as e:
                if e.code == 5:
                    raise UnsatisfiedConstraint(str(e))
                raise
        finally:
            ctx.prog_free(h)
    return Witness.read(data, c)


def prove_from_inputs(prog: Prog, inputs: Sequence[int], proving_key, rng, device: int = 0, lib=None):
    """Inputs -> proof with the assignment never leaving the device between witness generation and proving:
    `zkb_witness_eval` leaves z resident, `zkb_groth16_prove_resident` consumes it (the reference runs
    `compute-witness` and `generate-proof` as two processes with a witness file in between).  Same result as
    `B200.generate_proof(prog, Interpreter().execute(prog, inputs), proving_key, rng)`; directive-free programs only."""
    from . import backend
    from ._lib import ZkbError
    from .proof import Proof
    from .rng import fr_rand
    c = _curve(prog.curve)
    if len(inputs) != len(prog.arguments):
        raise ValueError(f"WrongInputCount: expected {len(prog.arguments)}, received {len(inputs)}")
    pk_bytes = proving_key.read() if hasattr(proving_key, "read") else bytes(proving_key)
    r = fr_rand(c, rng)                                      # create_random_proof draws r then s before synthesis
    s = fr_rand(c, rng)
    if any(isinstance(st, Directive) for st in prog.statements):
        # native front door: witness generation (solver kernels included) leaves z resident in the program's R1CS
        from . import zir
        ctx = backend.context(c, device, lib)
        with ctx.lock:
            h = ctx.prog_load(zir.write_prog(prog))
            pk_h = None
            try:
                info = ctx.prog_info(h)
                if info["unsupported_directives"]:
                    raise NotImplementedError("the program calls a solver that has no device path")
                try:
                    ctx.prog_compute_witness(h, [int(x) % c.r for x in inputs])
                except ZkbError as e:
                    if e.code == 5:
                        raise UnsatisfiedConstraint(str(e))
                    raise
                public = ctx.prog_public_inputs(h)
                pk_h = ctx.pk_load(pk_bytes, 0, 1)
                raw = ctx.prove_resident(pk_h, info["r1cs"], r, s)
            finally:
                if pk_h:
                    ctx.pk_free(pk_h)
                ctx.prog_free(h)
        return Proof.from_raw(c, raw, public)
    r1cs = synthesize(prog)
    cols = {v: i for i, v in enumerate(r1cs.instance_vars)}
    cols.update({v: r1cs.num_instance + i for i, v in enumerate(r1cs.witness_vars)})
    vals = [0] * r1cs.num_variables
    vals[0] = 1
    for p, x in zip(prog.arguments, inputs):
        vals[cols[p.id]] = int(x) % c.r
    level_ptr, rows, out_var = levels_for(r1cs, [0] + [cols[p.id] for p in prog.arguments])
    sess = backend.ProverSession(c, r1cs, pk_bytes, device, lib=lib)
    try:
        z = fr_array(vals)
        if len(level_ptr) > 1:
            try:
                z = sess.ctx.witness_eval(sess.r1cs_h, z, level_ptr, rows, out_var)
            except ZkbError as e:
                if e.code == 5:
                    raise UnsatisfiedConstraint(str(e))
                raise
        else:
            sess.ctx.set_assignment(sess.r1cs_h, z)
        raw = sess.ctx.prove_resident(sess.pk_h, sess.r1cs_h, r, s)
        public = fr_from_array(z[1:r1cs.num_instance]) if r1cs.num_instance > 1 else []   # instance columns ...
    finally:
        sess.close()
    # ... but the proof lists public arguments first and return values after them (ir/mod.rs:278-288)
    by_var = dict(zip(r1cs.instance_vars[1:], public))
    ordered = [by_var[p.id] for p in prog.arguments if not p.private] + [by_var[Variable.public(i)] for i in range(prog.return_count)]
    return Proof.from_raw(c, raw, ordered)


def _load_program(ctx, prog: Prog):
    """zkb_prog_load of the program; refuses one whose solvers have no device path"""
    from . import zir
    h = ctx.prog_load(zir.write_prog(prog))
    info = ctx.prog_info(h)
    if info["unsupported_directives"]:
        ctx.prog_free(h)
        raise NotImplementedError("the program calls a solver that has no device path: use ir.Interpreter")
    return h, info


def _raise_first_failure(first):
    for k, f in enumerate(first):
        if f is not None:
            raise UnsatisfiedConstraint(f"input set {k}: constraint {f} is not satisfied")


def generate_witnesses(prog: Prog, inputs_list: Sequence[Sequence[int]], ctx=None, lib=None, try_out_of_range: bool = False) -> List[Witness]:
    """`Interpreter::execute` of K input sets of one program in one level sweep on the device (zkb_prog_compute_witness_batch);
    every program goes through the native front door.  Witness k equals `generate_witness(prog, inputs_list[k])`.  Raises
    UnsatisfiedConstraint naming the first failing input set and its constraint, ValueError on a wrong input count."""
    from . import backend
    from ._lib import ZkbError
    c = _curve(prog.curve)
    for x in inputs_list:
        if len(x) != len(prog.arguments):
            raise ValueError(f"WrongInputCount: expected {len(prog.arguments)}, received {len(x)}")
    if not inputs_list:
        return []
    ctx = ctx or backend.context(c, 0, lib)
    with ctx.lock:
        h, _ = _load_program(ctx, prog)
        try:
            try:
                wits, first = ctx.prog_compute_witness_batch(h, [[int(v) % c.r for v in x] for x in inputs_list], try_out_of_range)
            except ZkbError as e:
                if e.code == 5:
                    raise UnsatisfiedConstraint(str(e))
                raise
        finally:
            ctx.prog_free(h)
    _raise_first_failure(first)
    return [Witness.read(w, c) for w in wits]


def prove_from_inputs_batch(prog: Prog, inputs_list: Sequence[Sequence[int]], proving_key, rng, device: int = 0, lib=None):
    """K input sets -> K proofs with the assignments resident on the device (zkb_prog_prove_batch).  (r, s) are drawn proof
    after proof, so the result equals `[prove_from_inputs(prog, x, proving_key, rng) for x in inputs_list]` on the same rng
    state.  Same failures as prove_from_inputs; an unsatisfied set raises UnsatisfiedConstraint naming it."""
    from . import backend
    from .proof import Proof
    from .rng import fr_rand
    c = _curve(prog.curve)
    for x in inputs_list:
        if len(x) != len(prog.arguments):
            raise ValueError(f"WrongInputCount: expected {len(prog.arguments)}, received {len(x)}")
    if not inputs_list:
        return []
    pk_bytes = proving_key.read() if hasattr(proving_key, "read") else bytes(proving_key)
    rs, ss = [], []
    for _ in inputs_list:
        rs.append(fr_rand(c, rng))
        ss.append(fr_rand(c, rng))
    ctx = backend.context(c, device, lib)
    with ctx.lock:
        h, _ = _load_program(ctx, prog)
        pk_h = None
        try:
            pk_h = ctx.pk_load(pk_bytes, 0, 1)
            res, first = ctx.prog_prove_batch(h, pk_h, [[int(v) % c.r for v in x] for x in inputs_list], rs, ss)
        finally:
            if pk_h:
                ctx.pk_free(pk_h)
            ctx.prog_free(h)
    _raise_first_failure(first)
    return [Proof.from_raw(c, raw, public) for raw, public in res]
