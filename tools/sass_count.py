"""Static multiply-add counts of the MSM bucket-accumulation kernels, read from the built library's SASS.

    python tools/sass_count.py [path/to/libzkb200.so]

For every `k_msm_accum1` instantiation it splits the kernel's SASS at the targets of its CALL instructions
into the kernel body and the out-of-line callees (fp2.cuh's mul_v / sqr_v / mul_sub_v for G2, the cold
doubling fallback ec.cuh mdbl_ni), and prints for each part the IMAD.WIDE* count and the IMAD-pipe count
(IMAD*, IMUL*; IMAD.MOV is listed apart since ptxas uses it as a plain move).  `per_add` is one pass of the
accumulate loop, i.e. one mixed addition: the body, plus for G2 the Fq2 arithmetic callees weighted by how
often the body calls them.  The G1 addition is inlined in the body, and the doubling fallback (G1: the
only callee; G2: the callee that itself makes calls) runs only when a bucket meets its own point, so it is
left out.  Needs only cuobjdump, no GPU.
"""
from __future__ import annotations

import collections
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "zokrates_b200", "libzkb200.so")

_FUNC = re.compile(r"^\s*Function : (\S+)")
_INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)(.*?);")
_CALL = re.compile(r"CALL\.REL(?:\.NOINC)?\s+(0x[0-9a-f]+)")


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("cuobjdump not found")


def _demangle(names):
    cf = shutil.which("c++filt")
    if not cf:
        return {n: n for n in names}
    out = subprocess.run([cf], input="\n".join(names), capture_output=True, text=True, check=True).stdout.split("\n")
    return dict(zip(names, out))


def functions(lib):
    """{mangled name: [(address, opcode, operands)]} for every kernel in the library."""
    sass = subprocess.run([_cuobjdump(), "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, cur = collections.OrderedDict(), None
    for line in sass.splitlines():
        m = _FUNC.match(line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = _INSN.match(line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(2), m.group(3)))
    return funcs


def count(insns):
    c = collections.Counter()
    for _, op, _ in insns:
        if op.startswith("IMAD.WIDE"):
            c["imad_wide"] += 1
        if op.startswith("IMAD.MOV"):
            c["imad_mov"] += 1
        elif op.startswith(("IMAD", "IMUL")):
            c["imad_pipe"] += 1
    return c


def split(insns):
    """Kernel body and callee regions (split at CALL targets); calls made from the body per callee."""
    targets = sorted({int(m.group(1), 16) for _, op, rest in insns if op.startswith("CALL")
                      for m in [_CALL.search(op + " " + rest)] if m})
    bounds = targets + [float("inf")]
    body = [i for i in insns if i[0] < bounds[0]]
    callees = collections.OrderedDict()
    for k, t in enumerate(targets):
        callees[t] = [i for i in insns if t <= i[0] < bounds[k + 1]]
    calls = collections.Counter()
    for _, op, rest in body:
        m = _CALL.search(op + " " + rest) if op.startswith("CALL") else None
        if m:
            calls[int(m.group(1), 16)] += 1
    return body, callees, calls


def report(lib):
    funcs = functions(lib)
    names = _demangle(list(funcs))
    rows = []
    for mangled, insns in funcs.items():
        name = names[mangled]
        if "k_msm_accum1" not in name:
            continue
        m = re.search(r"k_msm_accum1, (\d+), (\d+),.*?msm_accumulate<(.*?)>\(", name)
        field = m.group(3) if m else "?"
        body, callees, calls = split(insns)
        b = count(body)
        per_add = collections.Counter(b)
        parts = []
        for t, ins in callees.items():
            c = count(ins)
            n = calls.get(t, 0)
            leaf = not any(op.startswith("CALL") for _, op, _ in ins)
            if field.startswith("zkb::Fp2T") and leaf:
                for k in ("imad_wide", "imad_pipe"):
                    per_add[k] += n * c[k]
            parts.append({"addr": hex(t), "calls_from_body": n, "imad_wide": c["imad_wide"],
                          "imad_pipe": c["imad_pipe"], "makes_calls": not leaf})
        rows.append({"kernel": "k_msm_accum1<%s> block=%s minb=%s" % (field.replace("zkb::", ""), m.group(1), m.group(2)) if m else name,
                     "body": {"imad_wide": b["imad_wide"], "imad_pipe": b["imad_pipe"], "imad_mov": b["imad_mov"]},
                     "callees": parts,
                     "per_add": {"imad_wide": per_add["imad_wide"], "imad_pipe": per_add["imad_pipe"]}})
    return rows


def main(argv):
    lib = argv[1] if len(argv) > 1 else LIB
    for r in report(lib):
        print(r["kernel"])
        print("  per_add  imad_wide=%-6d imad_pipe=%d" % (r["per_add"]["imad_wide"], r["per_add"]["imad_pipe"]))
        print("  body     imad_wide=%-6d imad_pipe=%-6d imad_mov=%d" % (r["body"]["imad_wide"], r["body"]["imad_pipe"], r["body"]["imad_mov"]))
        for p in r["callees"]:
            print("  callee %-8s x%-3d imad_wide=%-6d imad_pipe=%-6d%s" % (p["addr"], p["calls_from_body"], p["imad_wide"], p["imad_pipe"],
                                                                       "  (makes calls)" if p["makes_calls"] else ""))


if __name__ == "__main__":
    main(sys.argv)
