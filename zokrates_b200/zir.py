"""Reader / writer of the compiled-program file (`out`) that `zokrates generate-proof -i out` consumes.

Restates /root/reference/zokrates_ast/src/ir/serialize.rs:
  * header (`ProgHeader::write/read`, :124-189): magic `ZOK\\0`, version 3.0.0.0, 4-byte curve id, u32 constraint count,
    u32 return count, then four (u32 type, u64 offset, u64 length) section records — parameters, constraints, solvers,
    module map.  The writer reserves `size_of::<ProgHeader>()` = 120 bytes (:195) although only 100 are used, and labels
    the module-map section with type 3 (`SectionType::Solvers`, :252) — both quirks are reproduced so files made here
    have the reference's layout; the reader relies on the offsets only, as `ProgEnum::read` does (:295-391).
  * sections are serde_cbor (0.11, default = structs as maps with text keys, externally tagged enums, `Option::None` as
    null, no self-describe tag): parameters = `Vec<Parameter>` (common/flat/parameter.rs:9-16), constraints = a stream
    of `Statement` values back to back (ir/mod.rs:118-128), solvers = `Vec<Solver>`, module map = `ModuleMap`.
  * field elements are CBOR byte strings holding ark's canonical little-endian encoding (zokrates_field/src/lib.rs:547-560);
    the visitor also accepts an array of small integers (:585-596) and so does this reader.

Only what the proving backend consumes is interpreted (parameters, return count, `Constraint` statements — ark's
synthesis skips directives and logs, zokrates_ark/src/lib.rs:116); everything else is decoded generically and kept
as plain Python values.  The reference ships no golden `out` file, so this layout is pinned only to the source text
above and to the curve ids of zokrates_book/src/toolbox/ir.md (tests/test_zir_format.py).
"""
from __future__ import annotations

import io
import struct
from typing import Any, List, Tuple

from .curves import curve as _curve
from .ir import Constraint, Directive, LinComb, Log, Parameter, Prog, QuadComb, Variable

MAGIC = b"ZOK\x00"
VERSION = bytes([3, 0, 0, 0])
CURVE_IDS = {"bn128": bytes.fromhex("b4f7b5bd"), "bls12_381": bytes.fromhex("40d8c1f9"), "bls12_377": bytes.fromhex("c2955ab5")}
HEADER_RESERVED = 120          # size_of::<ProgHeader>() on a 64-bit target: 20 + 4 * 24, rounded up to 8
SECTION_TYPES = (1, 2, 3, 3)   # the module map is (mis)labelled Solvers by the reference writer


class ZirFormatError(ValueError):
    pass


# ------------------------------------------------------------------------------------------------ CBOR (RFC 8949 subset)
class _Break:
    pass


_BREAK = _Break()


class CborReader:
    def __init__(self, data: bytes, pos: int = 0, end: int | None = None):
        self.d, self.p, self.end = data, pos, len(data) if end is None else end

    def _take(self, n: int) -> bytes:
        if self.p + n > self.end:
            raise ZirFormatError("CBOR item runs past the end of its section")
        b = self.d[self.p:self.p + n]
        self.p += n
        return b

    def _arg(self, info: int) -> int | None:
        if info < 24:
            return info
        if info == 24:
            return self._take(1)[0]
        if info == 25:
            return struct.unpack(">H", self._take(2))[0]
        if info == 26:
            return struct.unpack(">I", self._take(4))[0]
        if info == 27:
            return struct.unpack(">Q", self._take(8))[0]
        if info == 31:
            return None                    # indefinite length
        raise ZirFormatError("reserved CBOR additional information")

    def value(self) -> Any:
        ib = self._take(1)[0]
        major, info = ib >> 5, ib & 31
        if major == 7:
            if info == 20:
                return False
            if info == 21:
                return True
            if info in (22, 23):
                return None
            if info == 25:
                return float(struct.unpack(">e", self._take(2))[0])
            if info == 26:
                return struct.unpack(">f", self._take(4))[0]
            if info == 27:
                return struct.unpack(">d", self._take(8))[0]
            if info == 31:
                return _BREAK
            if info == 24:
                return self._take(1)[0]
            return info
        arg = self._arg(info)
        if major == 0:
            return arg
        if major == 1:
            return -1 - arg
        if major in (2, 3):
            if arg is None:                # indefinite: concatenation of definite chunks
                parts = []
                while True:
                    v = self.value()
                    if v is _BREAK:
                        break
                    parts.append(v)
                return (b"" if major == 2 else "").join(parts)
            raw = self._take(arg)
            return raw if major == 2 else raw.decode("utf-8")
        if major == 4:
            out = []
            if arg is None:
                while True:
                    v = self.value()
                    if v is _BREAK:
                        break
                    out.append(v)
            else:
                for _ in range(arg):
                    out.append(self.value())
            return out
        if major == 5:
            out = {}
            if arg is None:
                while True:
                    k = self.value()
                    if k is _BREAK:
                        break
                    out[k] = self.value()
            else:
                for _ in range(arg):
                    k = self.value()
                    out[k] = self.value()
            return out
        return self.value()                # major 6: tag — serde_cbor ignores tags


def cbor_encode(v: Any, out: io.BytesIO) -> None:
    """serde_cbor's choices: shortest-form heads, definite lengths, maps in insertion order."""
    def head(major: int, n: int):
        if n < 24:
            out.write(bytes([major << 5 | n]))
        elif n < 1 << 8:
            out.write(bytes([major << 5 | 24, n]))
        elif n < 1 << 16:
            out.write(bytes([major << 5 | 25]) + struct.pack(">H", n))
        elif n < 1 << 32:
            out.write(bytes([major << 5 | 26]) + struct.pack(">I", n))
        else:
            out.write(bytes([major << 5 | 27]) + struct.pack(">Q", n))
    if v is None:
        out.write(b"\xf6")
    elif v is True:
        out.write(b"\xf5")
    elif v is False:
        out.write(b"\xf4")
    elif isinstance(v, int):
        head(0, v) if v >= 0 else head(1, -1 - v)
    elif isinstance(v, (bytes, bytearray)):
        head(2, len(v)); out.write(bytes(v))
    elif isinstance(v, str):
        b = v.encode("utf-8"); head(3, len(b)); out.write(b)
    elif isinstance(v, (list, tuple)):
        head(4, len(v))
        for x in v:
            cbor_encode(x, out)
    elif isinstance(v, dict):
        head(5, len(v))
        for k, x in v.items():
            cbor_encode(k, out); cbor_encode(x, out)
    else:
        raise TypeError(f"cannot CBOR-encode {type(v).__name__}")


# ------------------------------------------------------------------------------------------------ serde model <-> ir.py
def _field(v, c) -> int:
    if isinstance(v, list):
        v = bytes(v)
    if not isinstance(v, (bytes, bytearray)) or len(v) != c.fr_bytes:
        raise ZirFormatError("field element is not a %d-byte string" % c.fr_bytes)
    x = int.from_bytes(v, "little")
    if x >= c.r:
        raise ZirFormatError("non-canonical field element")
    return x


def _lincomb(m, c) -> LinComb:
    try:
        return LinComb([(Variable(int(var["id"])), _field(coeff, c)) for var, coeff in m["value"]])
    except (KeyError, TypeError) as e:
        raise ZirFormatError(f"malformed LinComb: {e}")


def _quadcomb(m, c) -> QuadComb:
    return QuadComb(_lincomb(m["left"], c), _lincomb(m["right"], c))


def _solver(s) -> Tuple[str, Any]:
    """`Solver` (common/solvers.rs:11-27): unit variants are text, `Bits(n)` / `Ref(RefCall)` / `Zir(f)` are 1-entry maps."""
    if isinstance(s, str):
        return s, None
    if isinstance(s, dict) and len(s) == 1:
        (name, arg), = s.items()
        return name, arg
    raise ZirFormatError("malformed Solver")


def _statement(v, c, solvers):
    if not (isinstance(v, dict) and len(v) == 1):
        raise ZirFormatError("a Statement must be a one-entry map (externally tagged enum)")
    (kind, body), = v.items()
    if kind == "Constraint":
        err = body.get("error")
        if isinstance(err, dict):
            err = next(iter(err))
        return Constraint(_quadcomb(body["quad"], c), _lincomb(body["lin"], c), err)
    if kind == "Directive":
        name, arg = _solver(body["solver"])
        if name == "Ref":                  # SolverIndexer (serialize.rs:211-228) replaced the solver by its index
            idx = int(arg["index"])
            if idx < len(solvers):
                name, arg = _solver(solvers[idx])
        return Directive([_quadcomb(q, c) for q in body["inputs"]], [Variable(int(o["id"])) for o in body["outputs"]],
                         name, arg if isinstance(arg, int) else None)
    if kind == "Log":
        return Log(str(body.get("format_string")), [])
    raise ZirFormatError(f"unknown Statement variant {kind!r}")


def read_header(data: bytes):
    if len(data) < 100:
        raise ZirFormatError("Invalid header")
    if data[0:4] != MAGIC:
        raise ZirFormatError("Invalid magic number")
    if data[4:8] != VERSION:
        raise ZirFormatError("Invalid file version")
    cid = bytes(data[8:12])
    names = [k for k, v in CURVE_IDS.items() if v == cid]
    if not names:
        raise ZirFormatError("Unknown curve identifier")
    n_cons, n_ret = struct.unpack_from("<II", data, 12)
    sections = []
    for k in range(4):
        ty, off, ln = struct.unpack_from("<IQQ", data, 20 + 20 * k)
        if ty not in (1, 2, 3, 4):
            raise ZirFormatError("invalid section type")
        if off + ln > len(data):
            raise ZirFormatError("section out of bounds")
        sections.append((ty, off, ln))
    return names[0], n_cons, n_ret, sections


def read_prog(data: bytes) -> Prog:
    """`ProgEnum::deserialize` + `collect()` (serialize.rs:361-391): the statements in file order."""
    name, n_cons, n_ret, sec = read_header(data)
    c = _curve(name)
    params = CborReader(data, sec[0][1], sec[0][1] + sec[0][2]).value()
    if not isinstance(params, list):
        raise ZirFormatError("Cannot read parameters")
    try:
        arguments = [Parameter(Variable(int(p["id"]["id"])), bool(p["private"])) for p in params]
    except (KeyError, TypeError):
        raise ZirFormatError("Cannot read parameters")
    solvers = CborReader(data, sec[2][1], sec[2][1] + sec[2][2]).value() if sec[2][2] else []
    if not isinstance(solvers, list):
        raise ZirFormatError("Cannot read solvers")
    rd = CborReader(data, sec[1][1], sec[1][1] + sec[1][2])
    statements = []
    while rd.p < rd.end:
        statements.append(_statement(rd.value(), c, solvers))
    prog = Prog(arguments, n_ret, statements, name)
    if prog.constraint_count() != n_cons:
        raise ZirFormatError("constraint count in the header does not match the constraints section")
    return prog


def _lc_model(l: LinComb, c):
    return {"span": None, "value": [[{"id": v.id}, int(k % c.r).to_bytes(c.fr_bytes, "little")] for v, k in l.value]}


def _qc_model(q: QuadComb, c):
    return {"span": None, "left": _lc_model(q.left, c), "right": _lc_model(q.right, c)}


def write_prog(prog: Prog) -> bytes:
    """`ProgIterator::serialize` (serialize.rs:191-281) for programs built with ir.py (simple solvers only)."""
    c = _curve(prog.curve)
    body = io.BytesIO()
    body.write(b"\x00" * HEADER_RESERVED)
    spans: List[Tuple[int, int]] = []

    def section(write):
        a = body.tell(); write(); spans.append((a, body.tell() - a))

    section(lambda: cbor_encode([{"span": None, "id": {"id": p.id.id}, "private": bool(p.private)} for p in prog.arguments], body))
    solvers: list = []

    def solver_ref(d: Directive):
        model = d.solver if d.arg is None else {d.solver: d.arg}
        if model not in solvers:
            solvers.append(model)
        sig = (len(d.inputs), len(d.outputs))
        return {"Ref": {"index": solvers.index(model), "signature": [sig[0], sig[1]]}}

    def statements():
        for s in prog.statements:
            if isinstance(s, Constraint):
                cbor_encode({"Constraint": {"span": None, "quad": _qc_model(s.quad, c), "lin": _lc_model(s.lin, c),
                                            "error": s.error}}, body)
            elif isinstance(s, Directive):
                cbor_encode({"Directive": {"span": None, "inputs": [_qc_model(q, c) for q in s.inputs],
                                           "outputs": [{"id": o.id} for o in s.outputs], "solver": solver_ref(s)}}, body)
            # logs carry typed expressions the backend never reads: not emitted
    section(statements)
    section(lambda: cbor_encode(solvers, body))
    section(lambda: cbor_encode({"modules": {}}, body))
    head = MAGIC + VERSION + CURVE_IDS[prog.curve] + struct.pack("<II", prog.constraint_count(), prog.return_count)
    for ty, (off, ln) in zip(SECTION_TYPES, spans):
        head += struct.pack("<IQQ", ty, off, ln)
    out = bytearray(body.getvalue())
    out[:len(head)] = head
    return bytes(out)
