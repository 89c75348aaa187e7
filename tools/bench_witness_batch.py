#!/usr/bin/env python3
"""Throughput of batched witness generation (zkb_prog_compute_witness_batch) and of proving from inputs
(zkb_prog_prove_batch) against per-set calls, on one GPU.

For every (program, K) one JSON line with five arms, alternated after a warm-up of each, `--reps` times (medians count):
  a_witness_per_s   K x zkb_prog_compute_witness;
  b_witness_per_s   one zkb_prog_compute_witness_batch of the K sets;
  c_proofs_per_s    K x (zkb_prog_compute_witness + zkb_groth16_prove_resident);
  d_proofs_per_s    K x zkb_prog_compute_witness (+ zkb_prog_assignment), then one zkb_groth16_prove_batch;
  e_proofs_per_s    one zkb_prog_prove_batch;
  launches_b / launches_e   kernels one call of arm b / e launches (zkb_launch_count);
  gpu, power_limit_w        the card, read in the same run.
The bytes of arms a and b (witness files) and c, d and e (proofs) are compared; any mismatch exits with status 1.  Without a
CUDA device the script fails (status 2).

Programs: the sha256packed program (tests/test_sha256_program.py: ~35 k directives over 386 levels), and chained programs of
2^10, 2^14 and 2^16 constraints: 256 levels deep (t <- t * (t + b) per level), as wide as the size asks, so that the level
count stays that of a real program instead of growing with the size.  K in {1, 8, 64, 256}.

--parent-tree DIR also times the single zkb_prog_compute_witness of the sha256 program in a built checkout of another commit
(the parent), alternated with this tree, and checks that both give the same bytes.

    python tools/bench_witness_batch.py [--programs sha256 chain10 chain14 chain16] [--ks 1 8 64 256] [--reps 3] [--out FILE] [--parent-tree DIR]
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
TD = [5, 6, 7, 8, 99, 2, 3]
DEPTH = 256
SINGLE_SHA = """
import hashlib, json, sys, time
sys.path.insert(0, ".")
from zokrates_b200 import sha256_circuit, zir
from zokrates_b200._lib import Context
ctx = Context(0, 0)
h = ctx.prog_load(zir.write_prog(sha256_circuit.make_prog("bn128")))
w = ctx.prog_compute_witness(h, [0, 0, 0, 5])
ms = []
for _ in range(5):
    t0 = time.perf_counter(); ctx.prog_compute_witness(h, [0, 0, 0, 5]); ms.append(1e3 * (time.perf_counter() - t0))
print(json.dumps({"ms": ms, "sha": hashlib.sha256(w).hexdigest()}))
"""


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip().split(",")
    return out[0].strip(), float(out[1])


def chained(log_n):
    """W = 2^log_n / 256 chains of 256 levels: chain j starts at a_j * a_j and runs t <- t * (t + b); ~out_0 is their sum"""
    from zokrates_b200.ir import Constraint, LinComb, Parameter, Prog, QuadComb, Variable as V
    width = max(1, ((1 << log_n) - 8) // DEPTH)
    args = [V.new(j) for j in range(width)] + [V.new(width)]
    b = args[-1]
    nxt = width + 1
    st, ends = [], []
    for j in range(width):
        t = V.new(nxt); nxt += 1
        st.append(Constraint(QuadComb(LinComb.from_var(args[j]), LinComb.from_var(args[j])), LinComb.from_var(t)))
        for _ in range(DEPTH - 2):
            u = V.new(nxt); nxt += 1
            st.append(Constraint(QuadComb(LinComb.from_var(t), LinComb([(t, 1), (b, 1)])), LinComb.from_var(u)))
            t = u
        ends.append(t)
    st.append(Constraint(QuadComb(LinComb([(t, 1) for t in ends]), LinComb.one()), LinComb.from_var(V.public(0))))
    return Prog([Parameter.private_(a) for a in args[:-1]] + [Parameter.public(b)], 1, st, "bn128")


def program(name):
    from zokrates_b200 import sha256_circuit
    if name == "sha256":
        return sha256_circuit.make_prog("bn128")
    return chained(int(name[len("chain"):]))


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--programs", nargs="+", default=["sha256", "chain10", "chain14", "chain16"])
    ap.add_argument("--ks", nargs="+", type=int, default=[1, 8, 64, 256])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-prove", action="store_true", help="witness arms only")
    ap.add_argument("--parent-tree", default=None, metavar="DIR", help="a built checkout of the parent commit")
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)

    from zokrates_b200 import zir
    from zokrates_b200._lib import Context, Library, DEFAULT_LIB
    from zokrates_b200.curves import curve
    lib = Library(DEFAULT_LIB)
    if lib.dll.zkb_device_count() <= 0:
        print("bench_witness_batch.py needs a CUDA device", file=sys.stderr)
        return 2
    gpu, power = card()
    r = curve("bn128").r
    ctx = Context(0, 0, lib)
    lines, bad = [], False
    rnd = random.Random(1)

    def emit(line):
        line.update(gpu=gpu, power_limit_w=power)
        print(json.dumps(line), flush=True)
        lines.append(line)

    if args.parent_tree:
        # each tree times its own single call in its own process (the parent's binding lacks the batch entry points),
        # the two trees alternated
        times, outs = {"parent": [], "branch": []}, {}
        trees = {"parent": os.path.abspath(args.parent_tree), "branch": ROOT}
        for _ in range(3):
            for k in ("parent", "branch"):
                res = json.loads(subprocess.run([sys.executable, "-c", SINGLE_SHA], cwd=trees[k], capture_output=True, text=True,
                                                check=True).stdout.strip().splitlines()[-1])
                times[k] += res["ms"]
                outs[k] = res["sha"]
        same = outs["parent"] == outs["branch"]
        bad |= not same
        emit({"program": "sha256", "single_witness_ms_median": {k: round(statistics.median(v), 3) for k, v in times.items()},
              "single_witness_ms": times, "identical": same})

    for name in args.programs:
        prog = program(name)
        h = ctx.prog_load(zir.write_prog(prog))
        info = ctx.prog_info(h)
        n_args = info["arguments"]
        pk = None
        if not args.no_prove:
            pk = ctx.pk_load(ctx.setup(info["r1cs"], TD))
        for K in args.ks:
            if name == "sha256":
                sets = [[rnd.randrange(1 << 128) for _ in range(4)] for _ in range(K)]
            else:
                sets = [[rnd.randrange(r) for _ in range(n_args)] for _ in range(K)]
            rs = [1000 + k for k in range(K)]
            ss = [2000 + k for k in range(K)]
            arms = {
                "a": lambda: [ctx.prog_compute_witness(h, x) for x in sets],
                "b": lambda: ctx.prog_compute_witness_batch(h, sets)[0],
            }
            if pk:
                def arm_c():
                    out = []
                    for k, x in enumerate(sets):
                        ctx.prog_compute_witness(h, x)
                        out.append(ctx.prove_resident(pk, info["r1cs"], rs[k], ss[k]))
                    return out

                def arm_d():
                    zs = []
                    for x in sets:
                        ctx.prog_compute_witness(h, x)
                        zs.append(ctx.prog_assignment(h))
                    return ctx.prove_batch(pk, info["r1cs"], zs, rs, ss)
                arms.update(c=arm_c, d=arm_d, e=lambda: [p[0] for p in ctx.prog_prove_batch(h, pk, sets, rs, ss)[0]])
            res = {k: fn() for k, fn in arms.items()}          # warm-up of every arm, and their outputs
            launches = {}
            for k in ("b", "e"):
                if k in arms:
                    before = ctx.launch_count()
                    arms[k]()
                    launches[k] = ctx.launch_count() - before
            times = {k: [] for k in arms}
            for _ in range(args.reps):
                for k, fn in arms.items():
                    times[k].append(timed(fn)[0])
            med = {k: statistics.median(v) for k, v in times.items()}
            ok_w = res["a"] == res["b"]
            ok_p = (res["c"] == res["d"] == res["e"]) if pk else True
            bad |= not (ok_w and ok_p)
            line = {"program": name, "constraints": info["constraints"], "levels": info["levels"], "K": K,
                    "a_witness_per_s": round(K / med["a"], 2), "b_witness_per_s": round(K / med["b"], 2),
                    "witness_gain": round(med["a"] / med["b"], 2), "launches_b": launches["b"], "witness_identical": ok_w}
            if pk:
                line.update({f"{k}_proofs_per_s": round(K / med[k], 2) for k in "cde"})
                line.update(e_over_c=round(med["c"] / med["e"], 2), e_over_d=round(med["d"] / med["e"], 2),
                            launches_e=launches["e"], proofs_identical=ok_p)
            emit(line)
        if pk:
            ctx.pk_free(pk)
        ctx.prog_free(h)
    if args.out:
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
