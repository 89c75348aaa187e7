#!/usr/bin/env python3
"""zkb-compute-witness: the file-level face of the witness side, options and defaults of `zokrates compute-witness`
(/root/reference/zokrates_cli/src/ops/compute_witness.rs:16-75; raw `-a` / `--stdin` arguments — the ABI (JSON) input
format belongs to the compiler front end and is out of scope).  Reads the compiled program (`out`), evaluates it on the GPU level by
level (`zkb_prog_compute_witness`: constraints assign or check, solver directives run the kernels of csrc/solvers.cuh) and writes the binary `witness` (ir/witness.rs:44-53), optionally its JSON form and the
circom `.wtns` file.

    python tools/zkb_compute_witness.py -i out -o witness -a 337 113569 [--json] [--circom-witness out.wtns]

Many input sets of one program in one level sweep on the GPU (`zkb_prog_compute_witness_batch`): one space-separated argument
list per line of FILE, witness k written to DIR/witness_<k> (and DIR/witness_<k>.json with --json):

    python tools/zkb_compute_witness.py -i out --arguments-file args.txt --witness-dir witnesses [--json]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="zkb-compute-witness", description="Calculates a witness for a given constraint system")
    ap.add_argument("-i", "--input", default="out", metavar="FILE", help="Path of the binary")
    ap.add_argument("-o", "--output", default="witness", metavar="FILE", help="Path of the output witness file")
    ap.add_argument("--circom-witness", default=None, metavar="FILE", help="Path of the output circom witness file")
    ap.add_argument("-a", "--arguments", nargs="*", default=None, help="Arguments for the program's main function: a space-separated list of field elements like `-a 1 2 3`")
    ap.add_argument("--stdin", action="store_true", help="Read arguments from stdin")
    ap.add_argument("--json", action="store_true", help="Write witness in a json format for debugging purposes")
    ap.add_argument("--host", action="store_true", help="Force the host interpreter (Python mirror of the reference interpreter)")
    ap.add_argument("--try-out-of-range", action="store_true", help="Interpreter::try_out_of_range: second Bits decomposition")
    ap.add_argument("--arguments-file", default=None, metavar="FILE", help="Input sets of a batch, one space-separated argument list per line (needs --witness-dir)")
    ap.add_argument("--witness-dir", default=None, metavar="DIR", help="Directory of the batch's witness files witness_<k>")
    ap.add_argument("--verbose", action="store_true")
    args = ap.parse_args(argv)
    if (args.arguments_file is None) != (args.witness_dir is None):
        ap.error("--arguments-file and --witness-dir go together")

    from zokrates_b200 import circom, ir, witness_gpu, zir
    from zokrates_b200.curves import curve

    try:
        with open(args.input, "rb") as f:
            data = f.read()
        prog = zir.read_prog(data)
    except OSError as why:
        raise SystemExit(f"Could not open {args.input}: {why.strerror}")
    except zir.ZirFormatError as why:
        raise SystemExit(str(why))
    c = curve(prog.curve)

    def parse(raw, where=""):
        try:
            inputs = []
            for x in raw:
                v = int(x, 10)
                if v < 0 or v >= c.r:
                    raise ValueError(x)
                inputs.append(v)
            return inputs
        except ValueError as why:
            raise SystemExit(f"Could not parse argument{where}: {why}")

    if args.arguments_file is not None:
        return _batch(args, data, prog, parse)
    print("Computing witness...")
    raw = args.arguments
    if args.stdin:
        raw = sys.stdin.read().replace("\n", "").split(" ") if prog.arguments else []
    inputs = parse(raw or [])
    from zokrates_b200 import backend
    from zokrates_b200._lib import ZkbError
    try:
        if args.host:
            witness = ir.Interpreter(args.try_out_of_range).execute(prog, inputs)
        else:   # the library runs the statements level by level on the GPU, solver directives included
            witness = ir.Witness.read(backend.B200.compute_witness_files(data, inputs, prog.curve, args.try_out_of_range), prog.curve)
    except (ValueError, ir.UnsatisfiedConstraint, NotImplementedError, ZkbError) as why:
        raise SystemExit(f"Execution failed: {why}")
    if args.verbose:
        print(f"\nWitness: \n{[str(v) for v in witness.return_values()]}\n")
    try:
        with open(args.output, "wb") as f:
            f.write(witness.write())
        if args.json:
            with open(os.path.splitext(args.output)[0] + ".json", "w") as f:
                f.write(witness.write_json())
        if args.circom_witness:
            with open(args.circom_witness, "wb") as f:
                f.write(circom.write_witness(witness, [p.id for p in prog.arguments if not p.private]))
    except OSError as why:
        raise SystemExit(f"Could not create {why.filename}: {why.strerror}")
    print(f"Witness file written to '{args.output}'")
    return 0


def _batch(args, data, prog, parse) -> int:
    """--arguments-file: every line's witness from one zkb_prog_compute_witness_batch call"""
    from zokrates_b200 import backend, ir
    from zokrates_b200._lib import ZkbError
    try:
        with open(args.arguments_file) as f:
            lines = [ln.split() for ln in f.read().splitlines()]
    except OSError as why:
        raise SystemExit(f"Could not open {args.arguments_file}: {why.strerror}")
    while lines and not lines[-1]:
        lines.pop()
    sets = [parse(ln, f" on line {i + 1}") for i, ln in enumerate(lines)]
    print(f"Computing {len(sets)} witnesses...")
    if len(prog.arguments) and any(len(x) != len(prog.arguments) for x in sets):
        bad = next(i for i, x in enumerate(sets) if len(x) != len(prog.arguments))
        raise SystemExit(f"Execution failed on line {bad + 1}: WrongInputCount: expected {len(prog.arguments)}, received {len(sets[bad])}")
    ctx = backend.context(prog.curve)
    try:
        with ctx.lock:
            h = ctx.prog_load(data)
            try:
                wits, first = ctx.prog_compute_witness_batch(h, sets, args.try_out_of_range)
            finally:
                ctx.prog_free(h)
    except ZkbError as why:
        raise SystemExit(f"Execution failed: {why}")
    for i, f in enumerate(first):
        if f is not None:
            raise SystemExit(f"Execution failed on line {i + 1}: UnsatisfiedConstraint: constraint {f} is not satisfied")
    try:
        os.makedirs(args.witness_dir, exist_ok=True)
        for k, w in enumerate(wits):
            path = os.path.join(args.witness_dir, f"witness_{k}")
            with open(path, "wb") as f:
                f.write(w)
            if args.json:
                with open(path + ".json", "w") as f:
                    f.write(ir.Witness.read(w, prog.curve).write_json())
    except OSError as why:
        raise SystemExit(f"Could not create {why.filename}: {why.strerror}")
    print(f"{len(wits)} witness files written to '{args.witness_dir}'")
    return 0


if __name__ == "__main__":
    sys.exit(main())
