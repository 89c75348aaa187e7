"""iden3 `.r1cs` (v1) and `.wtns` (v2) export / import — the alternate front door of SURVEY.md §8(f) row 4.

Mirrors /root/reference/zokrates_circom/src/r1cs.rs:53-234 (`r1cs_program`, `write_r1cs`) and
src/witness.rs:27-104 (`write_witness`): wire order = one, outputs, public inputs, then every other variable
in increasing id order (which differs from the ark order used by `proving.key`, r1cs.rs:54-92), sections in
the order the reference writes them (constraints, header, wire map).  The readers accept what the writers emit
and produce an `R1CS` / assignment in THAT wire order, so a key made by `B200.setup` on the imported system
proves it.  Byte layout pinned by the reference's golden tests (r1cs.rs:242-430, witness.rs:113-230).
"""
from __future__ import annotations

import struct
from typing import Dict, List, Tuple

import numpy as np

from ._lib import fr_array
from .curves import curve as _curve
from .ir import Constraint, Prog, Variable, Witness
from .r1cs import R1CS


def r1cs_program(prog: Prog):
    """(variables in wire order, private_inputs_offset, constraints as term lists of (wire, coeff))."""
    index: Dict[Variable, int] = {}

    def provide(v):
        return index.setdefault(v, len(index))

    provide(Variable.one())
    for i in range(prog.return_count):
        provide(Variable.public(i))
    for p in prog.arguments:
        if not p.private:
            provide(p.id)
    private_offset = len(index)
    seen = set()
    cons = [s for s in prog.statements if isinstance(s, Constraint)]
    for s in cons:
        for lc in (s.quad.left, s.quad.right, s.lin):
            for v, _ in lc.value:
                seen.add(v)
    for v in sorted(seen):
        provide(v)
    rows = [tuple([(index[v], k) for v, k in lc.value] for lc in (s.quad.left, s.quad.right, s.lin)) for s in cons]
    variables = [None] * len(index)
    for v, i in index.items():
        variables[i] = v
    return variables, private_offset, rows


# the fields snarkjs / iden3 know; BLS12-377 is not one of them
CIRCOM_CURVES = ("bn128", "bls12_381")


def _circom_curve(curve):
    c = _curve(curve)
    if c.name not in CIRCOM_CURVES:
        raise ValueError("circom export supports bn128 and bls12_381, not %s" % c.name)
    return c


def write_r1cs(prog: Prog) -> bytes:
    c = _circom_curve(prog.curve)
    n8 = (c.r.bit_length() + 7) // 8
    variables, _, rows = r1cs_program(prog)
    n_pub_in = sum(not p.private for p in prog.arguments)
    n_prv_in = sum(p.private for p in prog.arguments)
    body = bytearray()
    for row in rows:
        for lc in row:
            body += struct.pack("<I", len(lc))
            for wire, coeff in lc:
                body += struct.pack("<I", wire) + int(coeff % c.r).to_bytes(32, "little")
    out = bytearray(b"r1cs") + struct.pack("<II", 1, 3)
    out += struct.pack("<IQ", 2, len(body)) + body
    out += struct.pack("<IQ", 1, 32 + 32)
    out += struct.pack("<I", n8) + c.r.to_bytes(n8, "little")
    out += struct.pack("<IIIIQI", len(variables), prog.return_count, n_pub_in, n_prv_in, len(variables), len(rows))
    out += struct.pack("<IQ", 3, 8 * len(variables))
    for i in range(len(variables)):
        out += struct.pack("<Q", i)
    return bytes(out)


def read_r1cs(data: bytes) -> R1CS:
    """Parse an iden3 .r1cs file into an `R1CS` whose instance variables are wires 0..nPubOut+nPubIn."""
    if data[:4] != b"r1cs":
        raise ValueError("not an r1cs file")
    version, nsec = struct.unpack_from("<II", data, 4)
    if version != 1:
        raise ValueError("unsupported r1cs version")
    off = 12
    sections = {}
    for _ in range(nsec):
        typ, size = struct.unpack_from("<IQ", data, off)
        off += 12
        sections[typ] = (off, size)
        off += size
    if 1 not in sections or 2 not in sections:
        raise ValueError("missing r1cs section")
    ho, _ = sections[1]
    (n8,) = struct.unpack_from("<I", data, ho)
    prime = int.from_bytes(data[ho + 4:ho + 4 + n8], "little")
    n_wires, n_out, n_pub, n_prv, n_labels, n_cons = struct.unpack_from("<IIIIQI", data, ho + 4 + n8)
    cv = next((c for c in map(_curve, CIRCOM_CURVES) if c.r == prime), None)
    if cv is None:
        raise ValueError("unknown field modulus")
    co, csize = sections[2]
    p = co
    mats = ([], [], [])
    ptrs = ([0], [0], [0])
    vals = ([], [], [])
    for _ in range(n_cons):
        for k in range(3):
            (nt,) = struct.unpack_from("<I", data, p)
            p += 4
            for _ in range(nt):
                (wire,) = struct.unpack_from("<I", data, p)
                coeff = int.from_bytes(data[p + 4:p + 4 + n8], "little")
                if wire >= n_wires or coeff >= prime:
                    raise ValueError("malformed constraint")
                mats[k].append(wire)
                vals[k].append(coeff)
                p += 4 + n8
            ptrs[k].append(len(mats[k]))
    if p != co + csize:
        raise ValueError("constraint section size mismatch")
    ni = 1 + n_out + n_pub
    csr = [(np.array(ptrs[k], dtype=np.uint64), np.array(mats[k], dtype=np.uint32), fr_array(vals[k])) for k in range(3)]
    return R1CS(cv.name, n_cons, ni, n_wires - ni, *csr)


def write_witness(witness: Witness, public_inputs: List[Variable]) -> bytes:
    """witness.rs:27-104: one, outputs in index order, public inputs (BTreeSet order), then the rest in map order."""
    c = _circom_curve(witness.curve)
    n8 = (c.r.bit_length() + 7) // 8
    w = dict(witness.values)
    vals = []
    if Variable.one() in w:
        vals.append(w.pop(Variable.one()))
    n_out = sum(v.is_output() for v in w)
    for i in range(n_out):
        vals.append(w.pop(Variable.public(i)))
    for v in sorted(set(public_inputs)):
        vals.append(w.pop(v))
    for v in sorted(w):
        vals.append(w[v])
    out = bytearray(b"wtns") + struct.pack("<II", 2, 2)
    out += struct.pack("<IQ", 1, 8 + n8) + struct.pack("<I", n8) + c.r.to_bytes(n8, "little") + struct.pack("<I", len(witness.values))
    out += struct.pack("<IQ", 2, len(vals) * n8)
    for v in vals:
        out += int(v).to_bytes(n8, "little")
    return bytes(out)


def read_wtns(data: bytes) -> Tuple[str, np.ndarray]:
    """-> (curve name, assignment uint64[n,4]) in wire order."""
    if data[:4] != b"wtns":
        raise ValueError("not a wtns file")
    version, nsec = struct.unpack_from("<II", data, 4)
    if version != 2:
        raise ValueError("unsupported wtns version")
    off = 12
    sections = {}
    for _ in range(nsec):
        typ, size = struct.unpack_from("<IQ", data, off)
        off += 12
        sections[typ] = (off, size)
        off += size
    ho, _ = sections[1]
    (n8,) = struct.unpack_from("<I", data, ho)
    prime = int.from_bytes(data[ho + 4:ho + 4 + n8], "little")
    (n,) = struct.unpack_from("<I", data, ho + 4 + n8)
    cv = next((c for c in map(_curve, CIRCOM_CURVES) if c.r == prime), None)
    if cv is None:
        raise ValueError("unknown field modulus")
    do, dsize = sections[2]
    if dsize != n * n8:
        raise ValueError("witness section size mismatch")
    vals = [int.from_bytes(data[do + i * n8:do + (i + 1) * n8], "little") for i in range(n)]
    if any(v >= prime for v in vals):
        raise ValueError("non-canonical witness value")
    return cv.name, fr_array(vals)
