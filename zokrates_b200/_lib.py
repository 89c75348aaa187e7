"""ctypes binding of the C ABI in include/zkb.h (libzkb200.so).

The product library is the in-tree `zokrates_b200/libzkb200.so` built by `__graft_entry__.build()`
(nvcc, sm_90a).  There is NO CPU fallback: if the library is missing or no CUDA device is usable
every entry point raises `ZkbError`.  Tests may pass an explicit path (the host-emulation build of
the same sources under tests/host_emu) — the product never does.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(HERE, "libzkb200.so")

STATUS = {0: "ZKB_OK", 1: "ZKB_E_ARG", 2: "ZKB_E_FORMAT", 3: "ZKB_E_CUDA", 4: "ZKB_E_OOM", 5: "ZKB_E_UNSAT",
          6: "ZKB_E_INTERNAL"}

# every symbol include/zkb.h declares (tests check that the built library exports all of them)
SYMBOLS = [
    "zkb_last_error", "zkb_abi_version", "zkb_device_count", "zkb_ctx_create", "zkb_ctx_destroy", "zkb_curve_sizes",
    "zkb_pk_load", "zkb_pk_info", "zkb_pk_free", "zkb_r1cs_load", "zkb_r1cs_free", "zkb_groth16_prove",
    "zkb_r1cs_set_assignment", "zkb_groth16_prove_resident", "zkb_groth16_prove_partial", "zkb_groth16_finalize",
    "zkb_msm_g1", "zkb_msm_g2", "zkb_ntt", "zkb_witness_map", "zkb_field_op", "zkb_groth16_setup",
    "zkb_groth16_setup_size", "zkb_last_timings", "zkb_launch_count", "zkb_peak_probe", "zkb_groth16_prove_begin",
    "zkb_groth16_prove_end", "zkb_groth16_finalize_prepare", "zkb_r1cs_check", "zkb_witness_eval",
    "zkb_pk_table_info", "zkb_ctx_set_option", "zkb_groth16_prove_submit", "zkb_groth16_prove_collect",
    "zkb_groth16_prove_collect_partial", "zkb_groth16_prove_begin_async", "zkb_groth16_prove_end_async",
    "zkb_groth16_prove_chains_to_stream", "zkb_groth16_prove_stream_to_finish",
    "zkb_prog_load", "zkb_prog_info", "zkb_prog_free", "zkb_prog_compute_witness", "zkb_prog_set_witness",
    "zkb_prog_public_inputs", "zkb_gm17_pk_load", "zkb_gm17_pk_free", "zkb_gm17_prove", "zkb_gm17_setup", "zkb_gm17_setup_size",
    "zkb_groth16_prove_batch", "zkb_prog_assignment", "zkb_prog_compute_witness_batch", "zkb_prog_prove_batch",
]

OPT_TABLES, OPT_TABLE_MIN_LOG, OPT_TABLE_C, OPT_Z_MODE, OPT_NTT_TILE_MIN, OPT_NTT_MAX_S, OPT_BITSUM_RADIX, OPT_PK_CACHE, OPT_NTT_KERNEL, OPT_BATCH_AFFINE, OPT_BATCH_AFFINE_MIN_LOG = 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11
OPT_BATCH_PASS_MAX = 15
TABLE_STATUS = {0: "none", 1: "built", 2: "below-min-size", 3: "no-memory", 4: "disabled", 5: "no-window"}


class ZkbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"{STATUS.get(code, code)}: {msg}")
        self.code = code


_u8p = C.POINTER(C.c_uint8)
_u32p = C.POINTER(C.c_uint32)
_u64p = C.POINTER(C.c_uint64)


def _p(arr, typ):
    return arr.ctypes.data_as(typ)


class Library:
    def __init__(self, path: str | None = None):
        path = path or os.environ.get("ZKB200_LIB") or DEFAULT_LIB
        if not os.path.exists(path):
            raise ZkbError(3, f"{path} not found — build it with `python -c 'import __graft_entry__ as g; g.build()'`; "
                              "zokrates_b200 has no CPU fallback")
        self.path = path
        self.dll = C.CDLL(path)
        d = self.dll
        d.zkb_last_error.restype = C.c_char_p
        d.zkb_abi_version.restype = C.c_uint32
        d.zkb_device_count.restype = C.c_int32
        d.zkb_ctx_create.argtypes = [C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
        d.zkb_ctx_destroy.argtypes = [C.c_void_p]
        d.zkb_ctx_destroy.restype = None
        d.zkb_curve_sizes.argtypes = [C.c_int32, _u64p]
        d.zkb_pk_load.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, _u64p]
        d.zkb_pk_info.argtypes = [C.c_void_p, C.c_uint64, _u64p]
        d.zkb_pk_free.argtypes = [C.c_void_p, C.c_uint64]
        d.zkb_pk_table_info.argtypes = [C.c_void_p, C.c_uint64, _u64p]
        d.zkb_ctx_set_option.argtypes = [C.c_void_p, C.c_int32, C.c_int64]
        d.zkb_r1cs_load.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64] + [C.c_void_p] * 9 + [_u64p]
        d.zkb_r1cs_free.argtypes = [C.c_void_p, C.c_uint64]
        d.zkb_r1cs_set_assignment.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
        d.zkb_groth16_prove.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_size_t]
        d.zkb_groth16_prove_batch.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_size_t]
        d.zkb_prog_assignment.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]
        d.zkb_groth16_prove_resident.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p,
                                                 C.c_void_p, C.c_size_t]
        d.zkb_groth16_prove_partial.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t]
        d.zkb_groth16_finalize.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_size_t]
        d.zkb_groth16_prove_begin.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint32,
                                              C.POINTER(C.c_void_p), _u64p]
        d.zkb_groth16_prove_end.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_size_t]
        d.zkb_groth16_prove_submit.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, _u64p]
        d.zkb_groth16_prove_collect.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_size_t]
        d.zkb_groth16_prove_collect_partial.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_size_t]
        d.zkb_groth16_prove_begin_async.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint32,
                                                    C.POINTER(C.c_void_p), _u64p, _u64p]
        d.zkb_groth16_prove_end_async.argtypes = [C.c_void_p, C.c_uint64]
        d.zkb_groth16_prove_chains_to_stream.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
        d.zkb_groth16_prove_stream_to_finish.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
        d.zkb_groth16_finalize_prepare.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
        d.zkb_r1cs_check.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, _u64p]
        d.zkb_witness_eval.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, _u64p]
        d.zkb_gm17_setup_size.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_size_t)]
        d.zkb_gm17_setup.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        d.zkb_gm17_pk_load.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, _u64p]
        d.zkb_gm17_pk_free.argtypes = [C.c_void_p, C.c_uint64]
        d.zkb_gm17_prove.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        d.zkb_prog_load.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, _u64p]
        d.zkb_prog_info.argtypes = [C.c_void_p, C.c_uint64, _u64p]
        d.zkb_prog_free.argtypes = [C.c_void_p, C.c_uint64]
        d.zkb_prog_compute_witness.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_size_t,
                                               C.POINTER(C.c_size_t), _u64p]
        d.zkb_prog_compute_witness_batch.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.c_uint32,
                                                     C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p]
        d.zkb_prog_prove_batch.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.c_uint32,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint64, C.c_void_p]
        d.zkb_prog_set_witness.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_size_t]
        d.zkb_prog_public_inputs.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, _u64p]
        d.zkb_msm_g1.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        d.zkb_msm_g2.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        d.zkb_ntt.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int32, C.c_int32]
        d.zkb_witness_map.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64]
        d.zkb_field_op.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
        d.zkb_groth16_setup.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t,
                                        C.POINTER(C.c_size_t)]
        d.zkb_groth16_setup_size.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_size_t)]
        d.zkb_last_timings.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_char_p), C.c_int32]
        d.zkb_last_timings.restype = C.c_int32
        d.zkb_launch_count.argtypes = [C.c_void_p]
        d.zkb_launch_count.restype = C.c_uint64
        d.zkb_peak_probe.argtypes = [C.c_void_p, C.c_int32, C.c_uint32, C.POINTER(C.c_double)]

    def check(self, status: int):
        if status != 0:
            raise ZkbError(status, (self.dll.zkb_last_error() or b"").decode(errors="replace"))

    def curve_sizes(self, curve: int):
        out = (C.c_uint64 * 4)()
        self.check(self.dll.zkb_curve_sizes(curve, out))
        return [int(x) for x in out]


_default = None


def default_library() -> Library:
    global _default
    if _default is None:
        _default = Library()
    return _default


def fr_array(values, n_limbs64=4) -> np.ndarray:
    """list of ints -> (len, n_limbs64) uint64 little-endian limb array (canonical form)."""
    out = np.zeros((len(values), n_limbs64), dtype=np.uint64)
    mask = (1 << 64) - 1
    for i, v in enumerate(values):
        v = int(v)
        for k in range(n_limbs64):
            out[i, k] = (v >> (64 * k)) & mask
    return out


def fr_from_array(arr) -> list:
    arr = np.asarray(arr, dtype=np.uint64)
    return [sum(int(x) << (64 * k) for k, x in enumerate(row)) for row in arr.reshape(arr.shape[0], -1)]


class Context:
    """One GPU, one curve (zkb_ctx)."""

    def __init__(self, curve: int, device: int = 0, lib: Library | None = None):
        self.lib = lib or default_library()
        self.curve = curve
        # every C-ABI call is serialised per context inside the library; multi-call sequences on shared per-context state
        # (prove_begin .. prove_end, finalize_prepare .. finalize) take this lock on top
        import threading
        self.lock = threading.RLock()
        h = C.c_void_p()
        self.lib.check(self.lib.dll.zkb_ctx_create(curve, device, C.byref(h)))
        self.h = h
        self.fr_bytes, self.fq_bytes, self.proof_bytes, self.partial_bytes = self.lib.curve_sizes(curve)

    def close(self):
        if getattr(self, "h", None):
            self.lib.dll.zkb_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- proving key / r1cs
    def pk_load(self, pk_bytes: bytes, rank=0, world=1) -> int:
        buf = np.frombuffer(pk_bytes, dtype=np.uint8)
        h = C.c_uint64()
        self.lib.check(self.lib.dll.zkb_pk_load(self.h, buf.ctypes.data, len(buf), rank, world, C.byref(h)))
        return h.value

    def pk_info(self, h):
        out = (C.c_uint64 * 4)()
        self.lib.check(self.lib.dll.zkb_pk_info(self.h, h, out))
        return [int(x) for x in out]

    def pk_free(self, h):
        self.lib.check(self.lib.dll.zkb_pk_free(self.h, h))

    def pk_table_info(self, h) -> dict:
        out = (C.c_uint64 * 8)()
        self.lib.check(self.lib.dll.zkb_pk_table_info(self.h, h, out))
        v = [int(x) for x in out]
        return {"c_z": v[0], "W_z": v[1], "c_h": v[2], "W_h": v[3], "table_bytes": v[4], "resident_bytes": v[5],
                "z_tables": TABLE_STATUS.get(v[6], v[6]), "h_table": TABLE_STATUS.get(v[7], v[7])}

    def set_option(self, option: int, value: int):
        self.lib.check(self.lib.dll.zkb_ctx_set_option(self.h, option, value))

    def r1cs_load(self, n_constraints, n_instance, n_witness, mats) -> int:
        """mats: three (rowptr uint64[N+1], col uint32[nnz], val uint64[nnz,4]) tuples."""
        args = []
        keep = []
        for rowptr, col, val in mats:
            rowptr = np.ascontiguousarray(rowptr, dtype=np.uint64)
            col = np.ascontiguousarray(col, dtype=np.uint32)
            val = np.ascontiguousarray(val, dtype=np.uint64).reshape(-1, 4)
            if len(rowptr) != n_constraints + 1 or len(col) != int(rowptr[-1]) or len(val) != len(col):
                raise ValueError("malformed CSR matrix")
            keep += [rowptr, col, val]
            args += [rowptr.ctypes.data, col.ctypes.data, val.ctypes.data]
        h = C.c_uint64()
        self.lib.check(self.lib.dll.zkb_r1cs_load(self.h, n_constraints, n_instance, n_witness, *args, C.byref(h)))
        return h.value

    def r1cs_free(self, h):
        self.lib.check(self.lib.dll.zkb_r1cs_free(self.h, h))

    def set_assignment(self, r1cs, z: np.ndarray):
        z = np.ascontiguousarray(z, dtype=np.uint64)
        self.lib.check(self.lib.dll.zkb_r1cs_set_assignment(self.h, r1cs, z.ctypes.data))

    # -- prover
    def prove(self, pk, r1cs, z: np.ndarray, r: int, s: int) -> bytes:
        z = np.ascontiguousarray(z, dtype=np.uint64)
        ra, sa = fr_array([r]), fr_array([s])
        out = np.zeros(self.proof_bytes, dtype=np.uint8)
        self.lib.check(self.lib.dll.zkb_groth16_prove(self.h, pk, r1cs, z.ctypes.data, ra.ctypes.data, sa.ctypes.data,
                                                      out.ctypes.data, len(out)))
        return out.tobytes()

    def prove_batch(self, pk, r1cs, zs, rs, ss) -> list:
        """K proofs of one circuit in one call (zkb_groth16_prove_batch): zs holds K assignments (a (K, m, 4) array or a list
        of (m, 4) arrays), rs / ss K scalars each.  Proof k is byte-identical to prove(pk, r1cs, zs[k], rs[k], ss[k])."""
        if isinstance(zs, np.ndarray) and zs.dtype == np.uint64 and zs.ndim == 3 and zs.flags.c_contiguous:
            z = zs                    # already K assignments back to back: no copy
        else:
            z = np.ascontiguousarray(np.stack([np.asarray(x, dtype=np.uint64).reshape(-1, 4) for x in zs]) if len(zs) else
                                     np.zeros((0, 4), dtype=np.uint64), dtype=np.uint64)
        k = len(zs)
        if len(rs) != k or len(ss) != k:
            raise ValueError("zs, rs and ss must have the same length")
        ra, sa = fr_array(list(rs)), fr_array(list(ss))
        out = np.zeros(max(k, 1) * self.proof_bytes, dtype=np.uint8)
        self.lib.check(self.lib.dll.zkb_groth16_prove_batch(self.h, pk, r1cs, k, z.ctypes.data, ra.ctypes.data, sa.ctypes.data,
                                                            out.ctypes.data, k * self.proof_bytes))
        return [out[i * self.proof_bytes:(i + 1) * self.proof_bytes].tobytes() for i in range(k)]

    def prove_resident(self, pk, r1cs, r: int, s: int) -> bytes:
        ra, sa = fr_array([r]), fr_array([s])
        out = np.zeros(self.proof_bytes, dtype=np.uint8)
        self.lib.check(self.lib.dll.zkb_groth16_prove_resident(self.h, pk, r1cs, ra.ctypes.data, sa.ctypes.data,
                                                               out.ctypes.data, len(out)))
        return out.tobytes()

    def prove_partial(self, pk, r1cs, z) -> np.ndarray:
        out = np.zeros(self.partial_bytes, dtype=np.uint8)
        zp = None
        if z is not None:
            z = np.ascontiguousarray(z, dtype=np.uint64)
            zp = z.ctypes.data
        self.lib.check(self.lib.dll.zkb_groth16_prove_partial(self.h, pk, r1cs, zp, out.ctypes.data, len(out)))
        return out

    def prove_begin(self, pk, r1cs, z, chain_mask: int):
        """Start a proof and compute the witness-map chains in `chain_mask`; returns ([3 device addresses], bytes each)."""
        zp = None
        if z is not None:
            z = np.ascontiguousarray(z, dtype=np.uint64)
            zp = z.ctypes.data
        ptrs = (C.c_void_p * 3)()
        nbytes = C.c_uint64(0)
        self.lib.check(self.lib.dll.zkb_groth16_prove_begin(self.h, pk, r1cs, zp, chain_mask, ptrs, C.byref(nbytes)))
        return [int(p or 0) for p in ptrs], int(nbytes.value)

    def prove_end(self, pk, r1cs) -> np.ndarray:
        out = np.zeros(self.partial_bytes, dtype=np.uint8)
        self.lib.check(self.lib.dll.zkb_groth16_prove_end(self.h, pk, r1cs, out.ctypes.data, len(out)))
        return out

    # -- pipelined form: two proofs may be in flight
    def prove_submit(self, pk, r1cs, z, r: int | None = None, s: int | None = None) -> int:
        """Enqueue one proof (z None: the resident assignment); returns a ticket.  With r and s the ticket collects to a
        finished proof (`prove_collect`), without to the partial sums (`prove_collect_partial`)."""
        zp = None
        if z is not None:
            z = np.ascontiguousarray(z, dtype=np.uint64)
            zp = z.ctypes.data
        rp = sp = None
        keep = None
        if r is not None:
            keep = (fr_array([r]), fr_array([s]))
            rp, sp = keep[0].ctypes.data, keep[1].ctypes.data
        t = C.c_uint64(0)
        self.lib.check(self.lib.dll.zkb_groth16_prove_submit(self.h, pk, r1cs, zp, rp, sp, C.byref(t)))
        return int(t.value)

    def prove_collect(self, ticket: int) -> bytes:
        out = np.zeros(self.proof_bytes, dtype=np.uint8)
        self.lib.check(self.lib.dll.zkb_groth16_prove_collect(self.h, ticket, out.ctypes.data, len(out)))
        return out.tobytes()

    def prove_collect_partial(self, ticket: int) -> np.ndarray:
        out = np.zeros(self.partial_bytes, dtype=np.uint8)
        self.lib.check(self.lib.dll.zkb_groth16_prove_collect_partial(self.h, ticket, out.ctypes.data, len(out)))
        return out

    def prove_begin_async(self, pk, r1cs, z, chain_mask: int):
        zp = None
        if z is not None:
            z = np.ascontiguousarray(z, dtype=np.uint64)
            zp = z.ctypes.data
        ptrs = (C.c_void_p * 3)()
        nbytes = C.c_uint64(0)
        t = C.c_uint64(0)
        self.lib.check(self.lib.dll.zkb_groth16_prove_begin_async(self.h, pk, r1cs, zp, chain_mask, ptrs, C.byref(nbytes), C.byref(t)))
        return int(t.value), [int(p or 0) for p in ptrs], int(nbytes.value)

    def prove_chains_to_stream(self, ticket: int, cuda_stream: int):
        self.lib.check(self.lib.dll.zkb_groth16_prove_chains_to_stream(self.h, ticket, C.c_void_p(cuda_stream)))

    def prove_stream_to_finish(self, ticket: int, cuda_stream: int):
        self.lib.check(self.lib.dll.zkb_groth16_prove_stream_to_finish(self.h, ticket, C.c_void_p(cuda_stream)))

    def prove_end_async(self, ticket: int):
        self.lib.check(self.lib.dll.zkb_groth16_prove_end_async(self.h, ticket))

    def finalize_prepare(self, pk, r: int, s: int):
        ra, sa = fr_array([r]), fr_array([s])
        self.lib.check(self.lib.dll.zkb_groth16_finalize_prepare(self.h, pk, ra.ctypes.data, sa.ctypes.data))

    def finalize(self, pk, partials: np.ndarray, world: int, r: int, s: int) -> bytes:
        partials = np.ascontiguousarray(partials, dtype=np.uint8)
        assert partials.size == world * self.partial_bytes
        ra, sa = fr_array([r]), fr_array([s])
        out = np.zeros(self.proof_bytes, dtype=np.uint8)
        self.lib.check(self.lib.dll.zkb_groth16_finalize(self.h, pk, partials.ctypes.data, world, ra.ctypes.data,
                                                         sa.ctypes.data, out.ctypes.data, len(out)))
        return out.tobytes()

    # -- witness side
    def r1cs_check(self, r1cs, z=None):
        """None if (A z) o (B z) == C z; else the index of the first violated constraint (status ZKB_E_UNSAT)."""
        zp = None
        if z is not None:
            z = np.ascontiguousarray(z, dtype=np.uint64)
            zp = z.ctypes.data
        first = C.c_uint64(0)
        st = self.lib.dll.zkb_r1cs_check(self.h, r1cs, zp, C.byref(first))
        if st == 5:
            return int(first.value)
        self.lib.check(st)
        return None

    def witness_eval(self, r1cs, z: np.ndarray, level_ptr, rows, out_var) -> np.ndarray:
        """Fill the assignment level by level on the device; raises ZkbError(ZKB_E_UNSAT) if a checked constraint fails."""
        z = np.ascontiguousarray(z, dtype=np.uint64).copy()
        level_ptr = np.ascontiguousarray(level_ptr, dtype=np.uint32)
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        out_var = np.ascontiguousarray(out_var, dtype=np.uint32)
        first = C.c_uint64(0)
        self.lib.check(self.lib.dll.zkb_witness_eval(self.h, r1cs, z.ctypes.data, len(level_ptr) - 1, level_ptr.ctypes.data,
                                                     rows.ctypes.data, out_var.ctypes.data, C.byref(first)))
        return z

    # -- compiled programs (native `out` / witness-file front door)
    PROG_INFO = ("constraints", "instance", "witness", "arguments", "returns", "directives", "levels", "r1cs", "extra_variables",
                 "unsupported_directives", "public_arguments", "schedulable")

    def prog_load(self, out_bytes: bytes) -> int:
        buf = np.frombuffer(out_bytes, dtype=np.uint8)
        h = C.c_uint64(0)
        self.lib.check(self.lib.dll.zkb_prog_load(self.h, buf.ctypes.data, len(buf), C.byref(h)))
        return h.value

    def prog_info(self, prog: int) -> dict:
        out = (C.c_uint64 * 12)()
        self.lib.check(self.lib.dll.zkb_prog_info(self.h, prog, out))
        return dict(zip(self.PROG_INFO, [int(x) for x in out]))

    def prog_free(self, prog: int):
        self.lib.check(self.lib.dll.zkb_prog_free(self.h, prog))

    def prog_compute_witness(self, prog: int, inputs, try_out_of_range: bool = False) -> bytes:
        """`Interpreter::execute` on the device; returns the witness FILE bytes.  ZkbError(ZKB_E_UNSAT) on a violated constraint."""
        arr = fr_array([int(x) for x in inputs]) if len(inputs) else np.zeros((0, 4), dtype=np.uint64)
        info = self.prog_info(prog)
        cap = 8 + 40 * (info["instance"] + info["witness"] + info["extra_variables"])
        out = np.zeros(cap, dtype=np.uint8)
        n = C.c_size_t(0)
        first = C.c_uint64(0)
        self.lib.check(self.lib.dll.zkb_prog_compute_witness(self.h, prog, arr.ctypes.data if len(arr) else None, len(arr),
                                                             1 if try_out_of_range else 0, out.ctypes.data, cap, C.byref(n), C.byref(first)))
        return out[:n.value].tobytes()

    def _input_sets(self, prog: int, inputs_list):
        """K input sets -> (K, n, 4) uint64 array; every set must have the program's argument count (else the library refuses)"""
        n = len(inputs_list[0]) if len(inputs_list) else 0
        if any(len(x) != n for x in inputs_list):
            raise ValueError("all input sets must have the same length")
        arr = np.zeros((len(inputs_list), n, 4), dtype=np.uint64)
        for k, x in enumerate(inputs_list):
            if n:
                arr[k] = fr_array([int(v) for v in x])
        return arr, n

    def prog_compute_witness_batch(self, prog: int, inputs_list, try_out_of_range: bool = False):
        """K input sets in one level sweep (zkb_prog_compute_witness_batch).  Returns (witnesses, first_unsatisfied): entry k is
        set k's witness FILE bytes and None, or None and the index of its first violated constraint."""
        arr, n = self._input_sets(prog, inputs_list)
        k = len(inputs_list)
        info = self.prog_info(prog)
        cap = 8 + 40 * (info["instance"] + info["witness"] + info["extra_variables"])
        out = np.zeros(max(k, 1) * cap, dtype=np.uint8)
        ln = C.c_size_t(0)
        first = np.zeros(max(k, 1), dtype=np.uint64)
        st = self.lib.dll.zkb_prog_compute_witness_batch(self.h, prog, k, arr.ctypes.data if arr.size else None, n,
                                                         1 if try_out_of_range else 0, out.ctypes.data, k * cap, C.byref(ln),
                                                         first.ctypes.data)
        if st != 5:
            self.lib.check(st)
        size = ln.value
        sat = [int(f) == (1 << 64) - 1 for f in first[:k]]
        return ([out[i * size:(i + 1) * size].tobytes() if sat[i] else None for i in range(k)],
                [None if sat[i] else int(first[i]) for i in range(k)])

    def prog_prove_batch(self, prog: int, pk: int, inputs_list, rs, ss, try_out_of_range: bool = False):
        """Inputs -> K proofs (zkb_prog_prove_batch), the assignments resident on the device.  Returns (proofs,
        first_unsatisfied): entry k is (proof bytes, public inputs) and None, or None and set k's first violated constraint.
        Proof k equals prog_compute_witness(prog, inputs_list[k]) + prove_resident(pk, r1cs, rs[k], ss[k])."""
        arr, n = self._input_sets(prog, inputs_list)
        k = len(inputs_list)
        if len(rs) != k or len(ss) != k:
            raise ValueError("inputs_list, rs and ss must have the same length")
        info = self.prog_info(prog)
        npub = info["public_arguments"] + info["returns"]
        ra, sa = fr_array(list(rs)), fr_array(list(ss))
        out = np.zeros(max(k, 1) * self.proof_bytes, dtype=np.uint8)
        pub = np.zeros((max(k * npub, 1), 4), dtype=np.uint64)
        first = np.zeros(max(k, 1), dtype=np.uint64)
        st = self.lib.dll.zkb_prog_prove_batch(self.h, prog, pk, k, arr.ctypes.data if arr.size else None, n,
                                               1 if try_out_of_range else 0, ra.ctypes.data, sa.ctypes.data, out.ctypes.data,
                                               k * self.proof_bytes, pub.ctypes.data, k * npub, first.ctypes.data)
        if st != 5:
            self.lib.check(st)
        res, bad = [], []
        for i in range(k):
            if int(first[i]) == (1 << 64) - 1:
                res.append((out[i * self.proof_bytes:(i + 1) * self.proof_bytes].tobytes(), fr_from_array(pub[i * npub:(i + 1) * npub]) if npub else []))
                bad.append(None)
            else:
                res.append(None)
                bad.append(int(first[i]))
        return res, bad

    def prog_set_witness(self, prog: int, witness_bytes: bytes):
        buf = np.frombuffer(witness_bytes, dtype=np.uint8)
        self.lib.check(self.lib.dll.zkb_prog_set_witness(self.h, prog, buf.ctypes.data, len(buf)))

    def prog_public_inputs(self, prog: int):
        n = C.c_uint64(0)
        self.lib.check(self.lib.dll.zkb_prog_public_inputs(self.h, prog, None, 0, C.byref(n)))
        if n.value == 0:
            return []
        out = np.zeros((max(n.value, 1), 4), dtype=np.uint64)
        self.lib.check(self.lib.dll.zkb_prog_public_inputs(self.h, prog, out.ctypes.data, n.value, C.byref(n)))
        return fr_from_array(out[:n.value])

    def prog_assignment(self, prog: int) -> np.ndarray:
        """The program's current assignment (after prog_set_witness / prog_compute_witness), ark column order, (m, 4) uint64."""
        info = self.prog_info(prog)
        m = info["instance"] + info["witness"]
        out = np.zeros((m, 4), dtype=np.uint64)
        self.lib.check(self.lib.dll.zkb_prog_assignment(self.h, prog, out.ctypes.data, m))
        return out

    # -- GM17
    def gm17_setup(self, r1cs: int, trapdoor6) -> bytes:
        td = fr_array([int(v) for v in trapdoor6])
        assert td.shape == (6, 4)
        n = C.c_size_t(0)
        self.lib.check(self.lib.dll.zkb_gm17_setup_size(self.h, r1cs, C.byref(n)))
        out = np.zeros(n.value, dtype=np.uint8)
        ln = C.c_size_t(0)
        self.lib.check(self.lib.dll.zkb_gm17_setup(self.h, r1cs, td.ctypes.data, out.ctypes.data, len(out), C.byref(ln)))
        return out[:ln.value].tobytes()

    def gm17_pk_load(self, pk_bytes: bytes) -> int:
        buf = np.frombuffer(pk_bytes, dtype=np.uint8)
        h = C.c_uint64(0)
        self.lib.check(self.lib.dll.zkb_gm17_pk_load(self.h, buf.ctypes.data, len(buf), C.byref(h)))
        return h.value

    def gm17_pk_free(self, h: int):
        self.lib.check(self.lib.dll.zkb_gm17_pk_free(self.h, h))

    def gm17_prove(self, pk: int, r1cs: int, z, d1: int, d2: int, r: int) -> bytes:
        zz = None if z is None else np.ascontiguousarray(z, dtype=np.uint64)
        m = fr_array([d1, d2, r])
        out = np.zeros(8 * self.fq_bytes, dtype=np.uint8)
        self.lib.check(self.lib.dll.zkb_gm17_prove(self.h, pk, r1cs, None if zz is None else zz.ctypes.data, m[0].ctypes.data,
                                                   m[1].ctypes.data, m[2].ctypes.data, out.ctypes.data, len(out)))
        return out.tobytes()

    # -- building blocks
    def msm(self, group: int, points: bytes, scalars: np.ndarray) -> bytes:
        pts = np.frombuffer(points, dtype=np.uint8)
        scalars = np.ascontiguousarray(scalars, dtype=np.uint64).reshape(-1, 4)
        n = len(scalars)
        size = (2 if group == 1 else 4) * self.fq_bytes
        assert len(pts) == n * size
        out = np.zeros(size, dtype=np.uint8)
        fn = self.lib.dll.zkb_msm_g1 if group == 1 else self.lib.dll.zkb_msm_g2
        self.lib.check(fn(self.h, pts.ctypes.data if n else None, scalars.ctypes.data if n else None, n, out.ctypes.data))
        return out.tobytes()

    def ntt(self, data: np.ndarray, inverse=False, coset=False) -> np.ndarray:
        data = np.array(data, dtype=np.uint64).reshape(-1, 4)
        n = len(data)
        log_n = n.bit_length() - 1
        assert 1 << log_n == n
        self.lib.check(self.lib.dll.zkb_ntt(self.h, data.ctypes.data, log_n, int(inverse), int(coset)))
        return data

    def witness_map(self, r1cs, z: np.ndarray, n: int) -> np.ndarray:
        z = np.ascontiguousarray(z, dtype=np.uint64)
        out = np.zeros((n, 4), dtype=np.uint64)
        self.lib.check(self.lib.dll.zkb_witness_map(self.h, r1cs, z.ctypes.data, out.ctypes.data, n))
        return out

    def field_op(self, field: int, op: int, a: np.ndarray, b: np.ndarray | None) -> np.ndarray:
        a = np.ascontiguousarray(a, dtype=np.uint64)
        out = np.zeros_like(a)
        bp = None
        if b is not None:
            b = np.ascontiguousarray(b, dtype=np.uint64)
            bp = b.ctypes.data
        self.lib.check(self.lib.dll.zkb_field_op(self.h, field, op, a.ctypes.data, bp, out.ctypes.data, a.shape[0]))
        return out

    def setup(self, r1cs, trapdoor7: list) -> bytes:
        size = C.c_size_t()
        self.lib.check(self.lib.dll.zkb_groth16_setup_size(self.h, r1cs, C.byref(size)))
        out = np.zeros(size.value, dtype=np.uint8)
        td = fr_array(trapdoor7)
        got = C.c_size_t()
        self.lib.check(self.lib.dll.zkb_groth16_setup(self.h, r1cs, td.ctypes.data, out.ctypes.data, len(out), C.byref(got)))
        return out[:got.value].tobytes()

    # -- measurement
    def timings(self) -> dict:
        ms = (C.c_double * 64)()
        names = (C.c_char_p * 64)()
        k = self.lib.dll.zkb_last_timings(self.h, ms, names, 64)
        out = {}
        for i in range(k):
            key = names[i].decode()
            out[key] = out.get(key, 0.0) + ms[i]
        return out

    def launch_count(self) -> int:
        return int(self.lib.dll.zkb_launch_count(self.h))

    def peak_probe(self, kind: int, iters: int = 20000) -> float:
        out = C.c_double()
        self.lib.check(self.lib.dll.zkb_peak_probe(self.h, kind, iters, C.byref(out)))
        return out.value
