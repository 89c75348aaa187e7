"""ctypes wrapper of oracle/libzkoracle.so (the C restatement) — test infrastructure."""
import ctypes as C

import numpy as np


class OracleC:
    def __init__(self, path):
        self.dll = C.CDLL(path)
        self.dll.zko_threads.restype = C.c_int

    def threads(self):
        return self.dll.zko_threads()

    def set_threads(self, n: int):
        self.dll.zko_set_threads(int(n))

    def field_op(self, curve, field, op, a, b):
        a = np.ascontiguousarray(a, dtype=np.uint64)
        out = np.zeros_like(a)
        bp = None
        if b is not None:
            b = np.ascontiguousarray(b, dtype=np.uint64)
            bp = C.c_void_p(b.ctypes.data)
        self.dll.zko_field_op(curve, field, op, C.c_void_p(a.ctypes.data), bp, C.c_void_p(out.ctypes.data), C.c_uint64(a.shape[0]))
        return out

    def ntt(self, curve, data, inverse=False, coset=False):
        data = np.array(data, dtype=np.uint64).reshape(-1, 4)
        log_n = len(data).bit_length() - 1
        self.dll.zko_ntt(curve, C.c_void_p(data.ctypes.data), C.c_uint32(log_n), int(inverse), int(coset))
        return data

    def msm(self, curve, group, points: bytes, scalars, fq_bytes):
        pts = np.frombuffer(points, dtype=np.uint8)
        scalars = np.ascontiguousarray(scalars, dtype=np.uint64).reshape(-1, 4)
        out = np.zeros((2 if group == 1 else 4) * fq_bytes, dtype=np.uint8)
        self.dll.zko_msm(curve, group, C.c_void_p(pts.ctypes.data), C.c_void_p(scalars.ctypes.data), C.c_uint64(len(scalars)),
                         C.c_void_p(out.ctypes.data))
        return out.tobytes()

    @staticmethod
    def _mats(r1cs):
        args, keep = [], []
        for rowptr, col, val in r1cs.matrices():
            rowptr = np.ascontiguousarray(rowptr, dtype=np.uint64); col = np.ascontiguousarray(col, dtype=np.uint32)
            val = np.ascontiguousarray(val, dtype=np.uint64)
            keep += [rowptr, col, val]
            args += [C.c_void_p(rowptr.ctypes.data), C.c_void_p(col.ctypes.data), C.c_void_p(val.ctypes.data)]
        return args, keep

    def witness_map(self, curve, r1cs, z):
        z = np.ascontiguousarray(z, dtype=np.uint64)
        out = np.zeros((r1cs.domain_size, 4), dtype=np.uint64)
        args, keep = self._mats(r1cs)
        self.dll.zko_witness_map(curve, C.c_uint64(r1cs.num_constraints), C.c_uint64(r1cs.num_instance),
                                 C.c_uint64(r1cs.num_witness), *args, C.c_void_p(z.ctypes.data), C.c_void_p(out.ctypes.data))
        return out

    def prove(self, curve, pk: bytes, r1cs, z, r: int, s: int, fq_bytes):
        from zokrates_b200._lib import fr_array
        z = np.ascontiguousarray(z, dtype=np.uint64)
        pkb = np.frombuffer(pk, dtype=np.uint8)
        out = np.zeros(8 * fq_bytes, dtype=np.uint8)
        times = np.zeros(5, dtype=np.float64)
        ra, sa = fr_array([r]), fr_array([s])
        args, keep = self._mats(r1cs)
        rc = self.dll.zko_groth16_prove(curve, C.c_void_p(pkb.ctypes.data), C.c_uint64(len(pkb)), C.c_uint64(r1cs.num_constraints),
                                        C.c_uint64(r1cs.num_instance), C.c_uint64(r1cs.num_witness), *args,
                                        C.c_void_p(z.ctypes.data), C.c_void_p(ra.ctypes.data), C.c_void_p(sa.ctypes.data),
                                        C.c_void_p(out.ctypes.data), C.c_void_p(times.ctypes.data))
        if rc != 0:
            raise RuntimeError(f"zko_groth16_prove rc={rc}")
        return out.tobytes(), times

    def setup(self, curve, r1cs, trapdoor7):
        from zokrates_b200._lib import fr_array
        td = fr_array(trapdoor7)
        args, keep = self._mats(r1cs)
        n = C.c_uint64()
        cap = 1 << 16
        while True:
            out = np.zeros(cap, dtype=np.uint8)
            rc = self.dll.zko_groth16_setup(curve, C.c_uint64(r1cs.num_constraints), C.c_uint64(r1cs.num_instance),
                                            C.c_uint64(r1cs.num_witness), *args, C.c_void_p(td.ctypes.data),
                                            C.c_void_p(out.ctypes.data), C.c_uint64(cap), C.byref(n))
            if rc == 0:
                return out[:n.value].tobytes()
            if rc != 2:
                raise RuntimeError(f"zko_groth16_setup rc={rc}")
            cap = int(n.value)

    def trapdoor_expected(self, curve, r1cs, trapdoor7, z, r: int, s: int, fq_bytes):
        """Expected proof bytes from the trapdoor (Fr arithmetic + three generator multiplications; no NTT / MSM / key)."""
        from zokrates_b200._lib import fr_array
        td = fr_array(trapdoor7)
        z = np.ascontiguousarray(z, dtype=np.uint64)
        ra, sa = fr_array([r]), fr_array([s])
        out = np.zeros(8 * fq_bytes, dtype=np.uint8)
        args, keep = self._mats(r1cs)
        rc = self.dll.zko_trapdoor_expected(curve, C.c_uint64(r1cs.num_constraints), C.c_uint64(r1cs.num_instance),
                                            C.c_uint64(r1cs.num_witness), *args, C.c_void_p(td.ctypes.data), C.c_void_p(z.ctypes.data),
                                            C.c_void_p(ra.ctypes.data), C.c_void_p(sa.ctypes.data), C.c_void_p(out.ctypes.data))
        if rc != 0:
            raise RuntimeError(f"zko_trapdoor_expected rc={rc}")
        return out.tobytes()

    @staticmethod
    def _sizes(r1cs):
        return C.c_uint64(r1cs.num_constraints), C.c_uint64(r1cs.num_instance), C.c_uint64(r1cs.num_witness)

    def gm17_trapdoor_expected(self, curve, r1cs, trapdoor6, z, d1: int, d2: int, r: int, fq_bytes):
        """Expected GM17 proof bytes from the trapdoor (alpha, beta, gamma, tau, g1_k, g2_k) and the masks d1, d2, r: Fr
        arithmetic + three generator multiplications (no NTT / MSM / key)."""
        from zokrates_b200._lib import fr_array
        td = fr_array(trapdoor6)
        z = np.ascontiguousarray(z, dtype=np.uint64)
        masks = fr_array([d1, d2, r])
        out = np.zeros(8 * fq_bytes, dtype=np.uint8)
        args, keep = self._mats(r1cs)
        rc = self.dll.zko_gm17_trapdoor_expected(curve, *self._sizes(r1cs), *args, C.c_void_p(td.ctypes.data),
                                                 C.c_void_p(z.ctypes.data), C.c_void_p(masks[0].ctypes.data),
                                                 C.c_void_p(masks[1].ctypes.data), C.c_void_p(masks[2].ctypes.data),
                                                 C.c_void_p(out.ctypes.data))
        if rc != 0:
            raise RuntimeError(f"zko_gm17_trapdoor_expected rc={rc}")
        return out.tobytes()

    def gm17_sap_at_tau(self, curve, r1cs, tau: int):
        """(u_i(tau), w_i(tau)) of every SAP variable as two (nv, 4) canonical limb arrays, and Z(tau) as an int."""
        from zokrates_b200._lib import fr_array, fr_from_array
        nv = r1cs.num_instance + r1cs.num_witness + r1cs.num_constraints + r1cs.num_instance - 1
        a = np.zeros((nv, 4), dtype=np.uint64)
        cc = np.zeros((nv, 4), dtype=np.uint64)
        zt = np.zeros((1, 4), dtype=np.uint64)
        ta = fr_array([tau])
        args, keep = self._mats(r1cs)
        rc = self.dll.zko_gm17_sap_at_tau(curve, *self._sizes(r1cs), *args, C.c_void_p(ta.ctypes.data), C.c_void_p(a.ctypes.data),
                                          C.c_void_p(cc.ctypes.data), C.c_void_p(zt.ctypes.data))
        if rc != 0:
            raise RuntimeError(f"zko_gm17_sap_at_tau rc={rc}")
        return a, cc, fr_from_array(zt)[0]
