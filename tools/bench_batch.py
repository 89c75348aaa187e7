#!/usr/bin/env python3
"""Throughput of batched proving (zkb_groth16_prove_batch) against the two-in-flight pipeline, on one GPU.

For every (curve, log_n, K, witness distribution) one JSON line:
  batch_proofs_per_s  K proofs by one zkb_groth16_prove_batch call;
  loop_proofs_per_s   the same K assignments and (r, s) through zkb_groth16_prove_submit / _collect with two proofs in flight
                      (submit k + 1, then collect k): what a caller can do without the batch entry point;
  launches_per_batch  kernels one batch call launches (zkb_launch_count);
  stages_ms           the batch call's per-stage times (zkb_last_timings);
  gpu, power_limit_w  the card, read in the same run.
The two arms alternate after a warm-up of each, `--reps` times; the median time counts.  The proof bytes of the two arms
are compared and any mismatch exits with status 1.  Without a CUDA device the script fails (status 2).

Sizes: BN254 at 2^10 .. 2^20 with K in {1, 8, 64, 256}, BLS12-381 at 2^12 and 2^16, uniform and 90 %-bits witnesses.
K * 2^log_n is capped at 2^24 (--max-work) so that one run stays within minutes; prove_batch itself splits a batch that does
not fit in HBM into passes.  From 2^18 on, and for K = 1, prove_batch drives the same two-slot pipeline as the loop arm
(engine.cuh, BATCH_SLOTS_MIN_LOG), so both arms there measure the same work; --lib runs another build of the library,
e.g. one with that threshold raised, to see the batch path itself at those sizes (how the threshold was set).

    python tools/bench_batch.py [--curves bn128 bls12_381] [--sizes 10 12] [--ks 1 8] [--reps 3] [--out FILE] [--lib PATH]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZES = {"bn128": [10, 12, 14, 16, 18, 20], "bls12_381": [12, 16]}
TD = [5, 6, 7, 8, 99, 2, 3]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return out[0].strip(), float(out[1])
    except Exception:
        return "unknown", None


def assignments(m, ni, K, dist, seed):
    """uniform: full-width values; bits: 90 % of the values 0 / 1 (hash-like witnesses).  z[0] = 1."""
    rnd = np.random.RandomState(seed)
    zs = np.zeros((K, m, 4), dtype=np.uint64)
    if dist == "uniform":
        zs[:] = rnd.randint(0, 1 << 62, size=(K, m, 4), dtype=np.int64).astype(np.uint64)
        zs[:, :, 3] &= np.uint64((1 << 60) - 1)
    else:
        zs[:, :, 0] = (rnd.rand(K, m) < 0.5).astype(np.uint64)
        big = rnd.rand(K, m) >= 0.9
        zs[big, 0] = rnd.randint(0, 1 << 62, size=int(big.sum()), dtype=np.int64).astype(np.uint64)
    zs[:, 0] = [1, 0, 0, 0]
    return zs


def loop_arm(ctx, pk, h, zs, rs, ss):
    out, prev = [], None
    for k in range(len(zs)):
        t = ctx.prove_submit(pk, h, zs[k], rs[k], ss[k])
        if prev is not None:
            out.append(ctx.prove_collect(prev))
        prev = t
    out.append(ctx.prove_collect(prev))
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--curves", nargs="+", default=list(SIZES))
    ap.add_argument("--sizes", nargs="+", type=int, default=None, help="log2 domain sizes (default: per curve, see above)")
    ap.add_argument("--ks", nargs="+", type=int, default=[1, 8, 64, 256])
    ap.add_argument("--dists", nargs="+", default=["uniform", "bits"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-work", type=int, default=24, help="largest log2(K * domain size) measured")
    ap.add_argument("--lib", default=None, help="library to load (default: the in-tree libzkb200.so)")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args(argv)

    from zokrates_b200 import synthetic
    from zokrates_b200._lib import Context, Library
    from zokrates_b200.curves import curve as get_curve

    lib = Library(args.lib) if args.lib else Library()
    if lib.dll.zkb_device_count() <= 0:
        print("bench_batch: no CUDA device (the prover has no CPU path)", file=sys.stderr)
        return 2
    gpu, power = card()
    mismatches = 0
    for curve in args.curves:
        c = get_curve(curve)
        ctx = Context(c.id, 0, lib)
        for log_n in (args.sizes or SIZES[curve]):
            ks = [k for k in args.ks if k.bit_length() - 1 + log_n <= args.max_work]
            if not ks:
                continue
            r1, _ = synthetic.make_layered(ctx, curve, (1 << log_n) - 2)
            h = ctx.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())
            pk = ctx.pk_load(ctx.setup(h, TD))
            tables = ctx.pk_table_info(pk)["z_tables"]
            for dist in args.dists:
                for K in ks:
                    zs = assignments(r1.num_variables, r1.num_instance, K, dist, 1000 * log_n + K)
                    rs = [1 + 3 * k for k in range(K)]
                    ss = [2 + 5 * k for k in range(K)]
                    ctx.prove_batch(pk, h, zs, rs, ss)          # warm-up of both arms (allocations, module loads)
                    loop_arm(ctx, pk, h, zs, rs, ss)
                    tb, tl = [], []
                    for _ in range(args.reps):
                        l0 = ctx.launch_count()
                        t0 = time.perf_counter()
                        got_b = ctx.prove_batch(pk, h, zs, rs, ss)
                        tb.append(time.perf_counter() - t0)
                        launches = ctx.launch_count() - l0
                        stages = ctx.timings()
                        t0 = time.perf_counter()
                        got_l = loop_arm(ctx, pk, h, zs, rs, ss)
                        tl.append(time.perf_counter() - t0)
                        if got_b != got_l:
                            mismatches += 1
                    rec = {"curve": curve, "log_n": log_n, "K": K, "witness": dist, "z_tables": tables,
                           "batch_proofs_per_s": round(K / statistics.median(tb), 2),
                           "loop_proofs_per_s": round(K / statistics.median(tl), 2),
                           "batch_ms": [round(1e3 * t, 3) for t in tb], "loop_ms": [round(1e3 * t, 3) for t in tl],
                           "launches_per_batch": launches, "stages_ms": {k: round(v, 3) for k, v in stages.items()},
                           "proofs_equal": got_b == got_l, "gpu": gpu, "power_limit_w": power,
                           "lib": os.path.basename(lib.path)}
                    line = json.dumps(rec)
                    print(line, flush=True)
                    if args.out:
                        with open(args.out, "a") as f:
                            f.write(line + "\n")
            ctx.pk_free(pk)
            ctx.r1cs_free(h)
    if mismatches:
        print(f"bench_batch: {mismatches} runs where the batch and the pipeline gave different proofs", file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
