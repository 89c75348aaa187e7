#!/usr/bin/env python3
"""zkb-generate-proof: the file-level face of the B200 backend, same options and defaults as
`zokrates generate-proof` (/root/reference/zokrates_cli/src/ops/generate_proof.rs:21-93, defaults from
zokrates_cli/src/cli_constants.rs): reads the compiled program (`out`), the binary witness and `proving.key`,
proves on the GPU (libzkb200.so — no CPU path) and writes `proof.json` in the reference's TaggedProof layout.

    python tools/zkb_generate_proof.py -i out -w witness -p proving.key -j proof.json [-e entropy] [--verbose]
    python tools/zkb_generate_proof.py -i out --witnesses w0 w1 .. -p proving.key --proof-dir DIR [-e entropy]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="zkb-generate-proof", description="Calculates a proof for a given constraint system and witness")
    ap.add_argument("-w", "--witness", default="witness", metavar="FILE", help="Path of the witness file")
    ap.add_argument("-p", "--proving-key-path", default="proving.key", metavar="FILE", help="Path of the proving key file")
    ap.add_argument("-j", "--proof-path", default="proof.json", metavar="FILE", help="Path of the JSON proof file")
    ap.add_argument("-i", "--input", default="out", metavar="FILE", help="Path of the binary")
    ap.add_argument("-b", "--backend", default="b200", choices=["b200"], help="Backend to use")
    ap.add_argument("-s", "--proving-scheme", default="g16", choices=["g16"], help="Proving scheme to use to generate the proof")
    ap.add_argument("-e", "--entropy", default=None, help="User provided randomness")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--tables", type=int, default=0, choices=[0, 1],
                    help="build the HBM window tables for this key (pays off from about a hundred proofs per key on; a one-shot process proves without)")
    ap.add_argument("--witnesses", nargs="+", default=None, metavar="FILE",
                    help="prove several witness files of the program in one GPU batch (with --proof-dir; replaces -w / -j)")
    ap.add_argument("--proof-dir", default=None, metavar="DIR",
                    help="with --witnesses: write DIR/proof_<i>.json for the i-th witness (i from 0, in the order given)")
    ap.add_argument("--verbose", action="store_true")
    args = ap.parse_args(argv)
    if (args.witnesses is None) != (args.proof_dir is None):
        ap.error("--witnesses and --proof-dir go together")

    from zokrates_b200 import backend, rng, zir
    from zokrates_b200._lib import ZkbError

    def slurp(path):
        try:
            with open(path, "rb") as f:
                return f.read()
        except OSError as why:
            raise SystemExit(f"Could not open {path}: {why.strerror}")

    out_bytes = slurp(args.input)
    try:
        curve_name = zir.read_header(out_bytes)[0]          # only the header is read here; the library parses the rest
    except zir.ZirFormatError as why:
        raise SystemExit(str(why))
    if args.witnesses is not None:
        print(f"Generating {len(args.witnesses)} proofs...")
        witnesses = [slurp(p) for p in args.witnesses]
        pk = slurp(args.proving_key_path)
        r = rng.get_rng_from_entropy(args.entropy) if args.entropy is not None else rng.StdRng.from_entropy()
        try:
            from zokrates_b200._lib import OPT_TABLES
            backend.context(curve_name, args.device).set_option(OPT_TABLES, args.tables)
            proofs = backend.B200.generate_proofs_files(out_bytes, witnesses, pk, r, curve=curve_name, device=args.device)
        except ZkbError as why:
            raise SystemExit(f"Could not generate the proofs: {why}")
        try:
            os.makedirs(args.proof_dir, exist_ok=True)
            for i, proof in enumerate(proofs):
                with open(os.path.join(args.proof_dir, f"proof_{i}.json"), "w") as f:
                    f.write(proof.to_tagged_json())
        except OSError as why:
            raise SystemExit(f"Could not write to {args.proof_dir}: {why.strerror}")
        print(f"{len(proofs)} proofs written to '{args.proof_dir}'")
        return 0
    print("Generating proof...")
    witness_bytes = slurp(args.witness)
    pk = slurp(args.proving_key_path)
    r = rng.get_rng_from_entropy(args.entropy) if args.entropy is not None else rng.StdRng.from_entropy()
    timings = {}
    try:
        from zokrates_b200._lib import OPT_TABLES
        backend.context(curve_name, args.device).set_option(OPT_TABLES, args.tables)
        proof = backend.B200.generate_proof_files(out_bytes, witness_bytes, pk, r, curve=curve_name, device=args.device, timings=timings)
    except ZkbError as why:
        raise SystemExit(f"Could not generate the proof: {why}")
    text = proof.to_tagged_json()
    try:
        with open(args.proof_path, "w") as f:
            f.write(text)
    except OSError as why:
        raise SystemExit(f"Could not write to {args.proof_path}: {why.strerror}")
    if args.verbose:
        print("Proof:\n" + text)
        print("timings: " + ", ".join(f"{k} {v:.3f}" for k, v in timings.items()))
    print(f"Proof written to '{args.proof_path}'")
    return 0


if __name__ == "__main__":
    sys.exit(main())
