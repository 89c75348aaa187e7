#!/usr/bin/env python3
"""Groth16 proving time per curve on one GPU, with bench.py's protocol, for curves bench.py does not offer.

    python tools/bench_curve.py --curve bls12_377 --curve bls12_381 --witness uniform --witness bits --log-n 20

Every (curve, witness) pair gets bench.py's workload: the synthetic circuit of 2^k - 2 constraints (one public input, domain
2^k), bench.py's trapdoor, r and s, the key and the assignment resident on the device, and proofs pipelined two in flight
(submit proof i + 1 before collecting proof i).  After --warmup proofs per pair, --rounds rounds time --steps proofs of
every pair in turn, so the pairs alternate under the same clocks; each pair reports the median ms/proof over its rounds.
One JSON line on stdout, with the device name and its power limit read in the same call.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TRAPDOOR = [0x1111, 0x2222, 0x3333, 0x4444, 0x123456789ABCDEF, 3, 7]   # bench.py's
R_S = (1234567, 7654321)


def power_limit_w():
    """Enforced power limit of GPU 0 (a read-only nvidia-smi query), or None."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        return None


class Pair:
    def __init__(self, lib, curve, witness, log_n):
        from zokrates_b200 import synthetic
        from zokrates_b200._lib import Context
        from zokrates_b200.curves import curve as _curve
        self.curve, self.witness = curve, witness
        self.ctx = Context(_curve(curve).id, 0, lib)
        r1, z = synthetic.make_layered(self.ctx, curve, (1 << log_n) - 2, distribution=witness)
        self.r1 = self.ctx.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())
        self.pk = self.ctx.pk_load(self.ctx.setup(self.r1, TRAPDOOR))
        self.ctx.set_assignment(self.r1, z)
        self.ms = []

    def run(self, steps):
        """`steps` proofs, two in flight; returns the last proof."""
        pending, proof = [], None
        for _ in range(steps):
            pending.append(self.ctx.prove_submit(self.pk, self.r1, None, *R_S))
            if len(pending) >= 2:
                proof = self.ctx.prove_collect(pending.pop(0))
        while pending:
            proof = self.ctx.prove_collect(pending.pop(0))
        return proof

    def timed(self, steps):
        import torch
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        self.run(steps)
        torch.cuda.synchronize()
        self.ms.append(1e3 * (time.perf_counter() - t0) / steps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curve", action="append", choices=["bn128", "bls12_381", "bls12_377"])
    ap.add_argument("--witness", action="append", choices=["uniform", "bits"])
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    curves, witnesses = args.curve or ["bls12_377"], args.witness or ["uniform"]
    sys.stdout.flush()
    stdout_fd = os.dup(1)
    os.dup2(2, 1)                        # one JSON line on stdout; anything a library prints goes to stderr

    import torch
    from zokrates_b200._lib import Library
    if not torch.cuda.is_available():
        raise SystemExit("bench_curve.py needs a CUDA device")
    lib = Library()
    pairs = [Pair(lib, c, w, args.log_n) for c in curves for w in witnesses]
    for p in pairs:
        p.run(max(args.warmup, 3))
    for _ in range(args.rounds):
        for p in pairs:
            p.timed(args.steps)
    n_cons = (1 << args.log_n) - 2
    line = {"metric": "groth16_ms_per_proof", "log_n": args.log_n, "constraints": n_cons, "steps": args.steps,
            "warmup": max(args.warmup, 3), "rounds": args.rounds, "pipeline": 2,
            "device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
            "results": [{"curve": p.curve, "witness": p.witness, "ms_per_proof": round(statistics.median(p.ms), 2),
                         "ms_rounds": [round(v, 2) for v in p.ms],
                         "constraints_per_sec": round(n_cons / statistics.median(p.ms) * 1e3)} for p in pairs]}
    for p in pairs:
        p.ctx.close()
    os.dup2(stdout_fd, 1)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
