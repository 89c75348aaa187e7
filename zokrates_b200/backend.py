"""`B200`: the Groth16 proving backend behind the reference's `Backend<T, G16>` interface.

Python mirror of the trait the Rust shim implements (INTEGRATION.md):

    pub trait Backend<T: Field, S: Scheme<T>> {
        fn generate_proof(program, witness, proving_key: impl Read, rng: &mut impl RngCore) -> Proof<T, S>;
        fn verify(vk: S::VerificationKey, proof: Proof<T, S>) -> bool;
    }                                         /root/reference/zokrates_proof_systems/src/lib.rs:98-112
    pub trait NonUniversalBackend { fn setup(program, rng) -> SetupKeypair<T, S>; }        lib.rs:113-118

Same argument meaning and error behaviour as `impl Backend<T, G16> for Ark`
(/root/reference/zokrates_ark/src/groth16.rs:21-109): static methods, program + witness consumed,
proving key = the bytes of `proving.key`, failures raise (the reference panics).  All arithmetic runs
in libzkb200.so on the GPU; this module only flattens the IR, draws r and s, and formats the proof.
"""
from __future__ import annotations

import threading
from typing import Dict, Optional, Tuple

import numpy as np

from . import _lib
from .curves import Curve, curve as _curve
from .ir import Prog, Witness
from .proof import Proof, SetupKeypair, vk_from_pk_bytes
from .r1cs import R1CS, synthesize
from .rng import StdRng, fr_rand

_lock = threading.Lock()
_contexts: Dict[Tuple[int, int], "_lib.Context"] = {}


def context(curve, device: int = 0, lib: Optional[_lib.Library] = None) -> "_lib.Context":
    """Process-global lazily created context per (curve, device) — the trait's methods are static, so
    the device state lives behind the FFI (SURVEY.md §8b)."""
    c = _curve(curve)
    if lib is not None:
        return _lib.Context(c.id, device, lib)
    with _lock:
        key = (c.id, device)
        if key not in _contexts:
            _contexts[key] = _lib.Context(c.id, device)
        return _contexts[key]


class ProverSession:
    """Proving key and R1CS resident on one GPU; many proofs (the timed region of SURVEY.md §8d)."""

    def __init__(self, curve, r1cs: R1CS, pk_bytes: bytes, device: int = 0, rank: int = 0, world: int = 1,
                 lib: Optional[_lib.Library] = None):
        self.curve: Curve = _curve(curve)
        self.ctx = context(self.curve, device, lib)
        self.r1cs = r1cs
        self.rank, self.world = rank, world
        self.pk_h = self.r1cs_h = None
        try:
            self.r1cs_h = self.ctx.r1cs_load(r1cs.num_constraints, r1cs.num_instance, r1cs.num_witness, r1cs.matrices())
            self.pk_h = self.ctx.pk_load(pk_bytes, rank, world)
            ni, m, hl, ll = self.ctx.pk_info(self.pk_h)
            if ni != r1cs.num_instance or m != r1cs.num_variables or hl + 1 != r1cs.domain_size:
                raise ValueError("proving key does not belong to this program")
        except BaseException:
            self.close()          # a failed load must not leave the matrices / key shard resident in the shared context
            raise

    def prove_raw(self, z: np.ndarray, r: int, s: int) -> bytes:
        return self.ctx.prove(self.pk_h, self.r1cs_h, z, r, s)

    def prove_partial(self, z: Optional[np.ndarray]) -> np.ndarray:
        return self.ctx.prove_partial(self.pk_h, self.r1cs_h, z)

    def finalize(self, partials: np.ndarray, world: int, r: int, s: int) -> bytes:
        return self.ctx.finalize(self.pk_h, partials, world, r, s)

    def close(self):
        for name, fn in (("pk_h", self.ctx.pk_free), ("r1cs_h", self.ctx.r1cs_free)):
            h = getattr(self, name, None)
            if h:
                fn(h)
                setattr(self, name, None)


class B200:
    """`impl<T: Field + ArkFieldExtensions> Backend<T, G16> for B200`."""

    NAME = "b200"

    @staticmethod
    def generate_proof(program: Prog, witness: Witness, proving_key, rng: StdRng, device: int = 0,
                       lib: Optional[_lib.Library] = None) -> Proof:
        c = _curve(program.curve)
        pk_bytes = proving_key.read() if hasattr(proving_key, "read") else bytes(proving_key)
        inputs = program.public_inputs_values(witness)           # groth16.rs:34-38
        r = fr_rand(c, rng)                                       # create_random_proof: r then s, before synthesis
        s = fr_rand(c, rng)
        r1cs = synthesize(program)
        try:
            z = r1cs.assignment(witness)
        except KeyError as e:
            raise RuntimeError(f"AssignmentMissing: {e}")         # SynthesisError::AssignmentMissing -> unwrap panic
        sess = ProverSession(c, r1cs, pk_bytes, device, lib=lib)
        try:
            raw = sess.prove_raw(z, r, s)
        finally:
            sess.close()
        return Proof.from_raw(c, raw, inputs)

    @staticmethod
    def generate_proof_files(out_bytes: bytes, witness_bytes: bytes, proving_key, rng: StdRng, curve="bn128", device: int = 0,
                             lib: Optional[_lib.Library] = None, timings: Optional[dict] = None) -> Proof:
        """`generate_proof` for the three FILES the CLI hands over (zokrates_cli/src/ops/generate_proof.rs:152-202): the
        compiled program, the binary witness and `proving.key`.  Nothing is interpreted in Python: the library parses the
        program and the witness natively (`zkb_prog_load`, `zkb_prog_set_witness`), synthesises the R1CS in ark order and
        proves from the resident assignment.  Repeated calls with the same key bytes reuse the resident key and its window
        tables (ZKB_OPT_PK_CACHE).  Same proof as `generate_proof(read_prog(out), Witness.read(witness), ...)`."""
        import time
        c = _curve(curve)
        ctx = context(c, device, lib)
        pk_bytes = proving_key.read() if hasattr(proving_key, "read") else proving_key
        r = fr_rand(c, rng)
        s = fr_rand(c, rng)
        t0 = time.perf_counter()
        with ctx.lock:
            prog = ctx.prog_load(out_bytes)
            pk_h = None
            try:
                info = ctx.prog_info(prog)
                t1 = time.perf_counter()
                ctx.prog_set_witness(prog, witness_bytes)
                inputs = ctx.prog_public_inputs(prog)
                t2 = time.perf_counter()
                pk_h = ctx.pk_load(pk_bytes, 0, 1)
                t3 = time.perf_counter()
                raw = ctx.prove_resident(pk_h, info["r1cs"], r, s)
                t4 = time.perf_counter()
            finally:
                if pk_h:
                    ctx.pk_free(pk_h)
                ctx.prog_free(prog)
        if timings is not None:
            timings.update(prog_load_s=t1 - t0, witness_s=t2 - t1, pk_load_s=t3 - t2, prove_s=t4 - t3)
        return Proof.from_raw(c, raw, inputs)

    @staticmethod
    def generate_proofs(program: Prog, witnesses, proving_key, rng: StdRng, device: int = 0,
                        lib: Optional[_lib.Library] = None) -> list:
        """Proofs of several witnesses of ONE program under one key, proved as one batch on the GPU (zkb_groth16_prove_batch).
        (r, s) are drawn for the first witness, then the second, and so on, so with the same rng state the result equals
        `[B200.generate_proof(program, w, proving_key, rng) for w in witnesses]`.  An addition beside the trait, which has
        no batch method."""
        c = _curve(program.curve)
        pk_bytes = proving_key.read() if hasattr(proving_key, "read") else bytes(proving_key)
        r1cs = synthesize(program)
        inputs, zs, rs, ss = [], [], [], []
        for w in witnesses:
            inputs.append(program.public_inputs_values(w))
            rs.append(fr_rand(c, rng))
            ss.append(fr_rand(c, rng))
            try:
                zs.append(r1cs.assignment(w))
            except KeyError as e:
                raise RuntimeError(f"AssignmentMissing: {e}")
        if not zs:
            return []
        sess = ProverSession(c, r1cs, pk_bytes, device, lib=lib)
        try:
            raws = sess.ctx.prove_batch(sess.pk_h, sess.r1cs_h, zs, rs, ss)
        finally:
            sess.close()
        return [Proof.from_raw(c, raw, inp) for raw, inp in zip(raws, inputs)]

    @staticmethod
    def generate_proofs_files(out_bytes: bytes, witness_bytes_list, proving_key, rng: StdRng, curve="bn128", device: int = 0,
                              lib: Optional[_lib.Library] = None) -> list:
        """`generate_proof_files` for several witness FILES of one program: every witness is read natively
        (`zkb_prog_set_witness`, `zkb_prog_assignment`, `zkb_prog_public_inputs`) and all of them are proved in one batch.
        (r, s) are drawn in witness order, so the proofs equal sequential `generate_proof_files` calls on the same rng."""
        c = _curve(curve)
        ctx = context(c, device, lib)
        pk_bytes = proving_key.read() if hasattr(proving_key, "read") else proving_key
        rs, ss = [], []
        for _ in witness_bytes_list:
            rs.append(fr_rand(c, rng))
            ss.append(fr_rand(c, rng))
        if not rs:
            return []
        with ctx.lock:
            prog = ctx.prog_load(out_bytes)
            pk_h = None
            try:
                info = ctx.prog_info(prog)
                zs, inputs = [], []
                for wb in witness_bytes_list:
                    ctx.prog_set_witness(prog, wb)
                    zs.append(ctx.prog_assignment(prog))
                    inputs.append(ctx.prog_public_inputs(prog))
                pk_h = ctx.pk_load(pk_bytes, 0, 1)
                raws = ctx.prove_batch(pk_h, info["r1cs"], zs, rs, ss)
            finally:
                if pk_h:
                    ctx.pk_free(pk_h)
                ctx.prog_free(prog)
        return [Proof.from_raw(c, raw, inp) for raw, inp in zip(raws, inputs)]

    @staticmethod
    def setup_gm17(program: Prog, trapdoor, device: int = 0, lib: Optional[_lib.Library] = None) -> bytes:
        """`impl NonUniversalBackend<T, GM17> for Ark`::setup (zokrates_ark/src/gm17.rs:19-41) on the GPU.  `trapdoor`: an `StdRng`
        (alpha, beta, gamma, tau and the two generator scalars are drawn with `fr_rand`, in that order) or 6 explicit integers.
        Returns ark-gm17's `ProvingKey::serialize_unchecked` bytes (the verifying key is their head)."""
        c = _curve(program.curve)
        td = [fr_rand(c, trapdoor) for _ in range(6)] if isinstance(trapdoor, StdRng) else [int(v) % c.r for v in trapdoor]
        if len(td) != 6 or any(v == 0 for v in td[:3] + td[4:]):
            raise ValueError("trapdoor needs 6 scalars; alpha, beta, gamma and the generator scalars must be non-zero")
        r1cs = synthesize(program)
        ctx = context(c, device, lib)
        with ctx.lock:
            h = ctx.r1cs_load(r1cs.num_constraints, r1cs.num_instance, r1cs.num_witness, r1cs.matrices())
            try:
                return ctx.gm17_setup(h, td)
            finally:
                ctx.r1cs_free(h)

    @staticmethod
    def generate_proof_gm17(program: Prog, witness: Witness, proving_key, rng: StdRng, device: int = 0,
                            lib: Optional[_lib.Library] = None) -> Proof:
        """`impl Backend<T, GM17> for Ark`::generate_proof (zokrates_ark/src/gm17.rs:43-75) on the GPU: the proving key is ark-gm17's
        `ProvingKey::serialize_unchecked`; `create_random_proof` draws d1, d2, r in that order.  Same R1CS synthesis and
        public-input order as Groth16; the proof JSON carries scheme "gm17"."""
        c = _curve(program.curve)
        pk_bytes = proving_key.read() if hasattr(proving_key, "read") else bytes(proving_key)
        inputs = program.public_inputs_values(witness)
        d1 = fr_rand(c, rng)
        d2 = fr_rand(c, rng)
        r = fr_rand(c, rng)
        r1cs = synthesize(program)
        try:
            z = r1cs.assignment(witness)
        except KeyError as e:
            raise RuntimeError(f"AssignmentMissing: {e}")
        ctx = context(c, device, lib)
        with ctx.lock:
            rh = ctx.r1cs_load(r1cs.num_constraints, r1cs.num_instance, r1cs.num_witness, r1cs.matrices())
            pkh = None
            try:
                pkh = ctx.gm17_pk_load(pk_bytes)
                raw = ctx.gm17_prove(pkh, rh, z, d1, d2, r)
            finally:
                if pkh:
                    ctx.gm17_pk_free(pkh)
                ctx.r1cs_free(rh)
        return Proof.from_raw(c, raw, inputs, scheme="gm17")

    @staticmethod
    def compute_witness_files(out_bytes: bytes, inputs, curve="bn128", try_out_of_range: bool = False, device: int = 0,
                              lib: Optional[_lib.Library] = None) -> bytes:
        """`zokrates compute-witness` on the device: program file + argument values -> witness file bytes
        (`Interpreter::execute`, zokrates_interpreter/src/lib.rs:40-138, with the solver kernels of csrc/solvers.cuh)."""
        ctx = context(_curve(curve), device, lib)
        with ctx.lock:
            prog = ctx.prog_load(out_bytes)
            try:
                return ctx.prog_compute_witness(prog, inputs, try_out_of_range)
            finally:
                ctx.prog_free(prog)

    @staticmethod
    def setup(program: Prog, trapdoor, device: int = 0, lib: Optional[_lib.Library] = None) -> SetupKeypair:
        """`NonUniversalBackend::setup`.  `trapdoor` is either an `StdRng` (alpha, beta, gamma, delta, tau and
        the two generator scalars are drawn from it with `fr_rand`, in that order) or 7 explicit integers."""
        c = _curve(program.curve)
        if isinstance(trapdoor, StdRng):
            td = [fr_rand(c, trapdoor) for _ in range(7)]
        else:
            td = [int(v) % c.r for v in trapdoor]
        if len(td) != 7 or any(v == 0 for v in td[:4] + td[5:]):
            raise ValueError("trapdoor needs 7 scalars; alpha..delta and the generator scalars must be non-zero")
        r1cs = synthesize(program)
        ctx = context(c, device, lib)
        h = ctx.r1cs_load(r1cs.num_constraints, r1cs.num_instance, r1cs.num_witness, r1cs.matrices())
        try:
            pk = ctx.setup(h, td)
        finally:
            ctx.r1cs_free(h)
        return SetupKeypair(vk_from_pk_bytes(c, pk), pk)

    @staticmethod
    def verify_gm17(vk, proof: Proof) -> bool:
        """`impl Backend<T, GM17> for Ark`::verify (gm17.rs:77-117): both GM17 pairing equations, on the host."""
        from .verify import verify_proof_gm17
        return verify_proof_gm17(vk, proof)

    @staticmethod
    def verify(vk, proof: Proof) -> bool:
        """Pairing check on the host (SURVEY.md §8 row a13: verification is not a GPU path)."""
        from .verify import verify_proof
        return verify_proof(vk, proof)
