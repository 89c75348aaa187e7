"""Pins of the prover's orchestration: the kernels a single Groth16 proof, a batch pass of three proofs, a standalone G1 MSM
and a GM17 proof launch (zkb_launch_count), and the stage names their calls report (zkb_last_timings).  bench.py reads
`accum1_g1_h` and writes every stage into its output, tools/microbench.py reads `msm_plan`, `msm_exec` and `accum1`, and
tools/bench_batch.py reports the `*_batch` stages, so a change of either is a change of what those tools measure.  The CPU
tier pins the launch counts through the host emulation; the stage names need the GPU, because the stage timer records CUDA
events and the emulation build has none."""
import random

import pytest

from oracle import ark
from oracle.ff import BN254, g1_group
from zokrates_b200 import synthetic
from zokrates_b200._lib import Context, fr_array

TD = [5, 6, 7, 8, 99, 2, 3]
GM17_TD = [3, 5, 7, 1234567, 11, 13]
N_CONSTRAINTS = 1000    # Groth16 domain 2^10 (tile passes of the transforms), GM17 domain 2^11

# the emulation counts the kernels it steps through; the device build also counts the scan and view-compaction launches,
# which the emulation runs as host loops
LAUNCHES_EMU = {"single": 87, "batch3": 86, "msm_g1": 17, "gm17": 102}
LAUNCHES_GPU = {"single": 95, "batch3": 98, "msm_g1": 18, "gm17": 105}

# `host_*` stages are timed on the host clock
STAGES = {
    "single": {"h2d_z", "witness_map_chains", "msm_plan_z", "accum1_g2_b2", "tail_g2_b2", "accum1_g1_l", "tail_g1_l", "accum1_g1_a",
               "tail_g1_a", "accum1_g1_b1", "tail_g1_b1", "witness_map_finish", "msm_plan_h", "wait_h", "accum1_g1_h", "tail_g1_h",
               "tails_wait", "d2h_windows", "host_tree_finish", "host_final_combine"},
    "batch3": {"h2d_z_batch", "witness_map_batch", "witness_map_finish_batch", "msm_plan_z_batch", "msm_plan_h_batch",
               "accum1_g2_b2_batch", "tail_g2_b2_batch", "accum1_g1_l_batch", "tail_g1_l_batch", "accum1_g1_a_batch", "tail_g1_a_batch",
               "accum1_g1_b1_batch", "tail_g1_b1_batch", "accum1_g1_h_batch", "tail_g1_h_batch", "d2h_windows_batch", "host_tails_batch"},
    "msm_g1": {"msm_plan", "msm_exec", "accum1"},
    "gm17": {"gm17_witness_map", "gm17_msms"},
}


def run_cases(ctx):
    """case -> (kernels launched, stage names reported) of the four calls on one BN254 context"""
    r1, z = synthetic.make("bn128", N_CONSTRAINTS)
    h = ctx.r1cs_load(r1.num_constraints, r1.num_instance, r1.num_witness, r1.matrices())
    pk = ctx.pk_load(ctx.setup(h, TD))
    gpk = ctx.gm17_pk_load(ctx.gm17_setup(h, GM17_TD))
    rnd = random.Random(11)
    G1 = g1_group(BN254)
    base = [G1.mul(BN254.g1, rnd.randrange(1, BN254.r)) for _ in range(8)]
    n = 700
    points = b"".join(ark.ser_g1(BN254, base[i % 8]) for i in range(n))
    scalars = fr_array([rnd.randrange(BN254.r) for _ in range(n)])
    calls = {
        "single": lambda: ctx.prove(pk, h, z, 1234, 5678),
        "batch3": lambda: ctx.prove_batch(pk, h, [z, z, z], [11, 12, 13], [21, 22, 23]),
        "msm_g1": lambda: ctx.msm(1, points, scalars),
        "gm17": lambda: ctx.gm17_prove(gpk, h, z, 17, 19, 23),
    }
    out = {}
    for name, call in calls.items():
        before = ctx.launch_count()
        call()
        out[name] = (ctx.launch_count() - before, set(ctx.timings()))
    return out


def test_emu_launch_counts(emu_lib):
    got = run_cases(Context(0, 0, emu_lib))
    assert {k: v[0] for k, v in got.items()} == LAUNCHES_EMU


@pytest.mark.gpu
def test_gpu_stage_names(gpu_lib):
    got = run_cases(Context(0, 0, gpu_lib))
    assert {k: v[1] for k, v in got.items()} == STAGES
    assert {k: v[0] for k, v in got.items()} == LAUNCHES_GPU
