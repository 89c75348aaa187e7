"""Multi-GPU proving: one process per GPU, MSMs sharded by index range, one tiny exchange per proof.

The Groth16 prover's five MSMs are sums over independent (scalar, point) pairs, so every rank keeps the
[rank/world) slice of each query vector resident (`zkb_pk_load(rank, world)`) and produces five partial
sums.  Elliptic-curve addition is not an NCCL reduction op, so the partial blobs (a few hundred bytes per
rank) are all-gathered with `torch.distributed` (NCCL over NVLink on GPUs, gloo in the CPU tests) and the
final combination runs once (rank `dst`).

witness_map: every rank needs all of h for its h-query slice.  With one or two ranks it is simply replicated
(it hides under the MSM kernels).  With three or more ranks the MSM shards are so small that the replicated
witness map becomes the critical path, and its three chains coset_fft(ifft(M z)), M = A, B, C, are independent:
chain k is computed once, by rank k mod world, and broadcast as 32 n bytes over NVLink (`zkb_groth16_prove_begin`
/ `_end`).  The transforms themselves stay per-GPU: sharding an NTT would need all-to-all transposes
(SURVEY.md §8e).
"""
from __future__ import annotations

from typing import Optional

import numpy as np


def gather_partials(partial: np.ndarray, group=None, device=None) -> np.ndarray:
    """all_gather of the per-rank partial-sum blobs; returns the world * partial_bytes concatenation."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    mine = torch.from_numpy(np.ascontiguousarray(partial, dtype=np.uint8))
    if device is not None:
        mine = mine.to(device)
    out = torch.empty(world * mine.numel(), dtype=torch.uint8, device=mine.device)
    dist.all_gather_into_tensor(out, mine, group=group)
    return out.cpu().numpy()


class _DevBuf:
    """A device allocation owned by libzkb200 seen through __cuda_array_interface__ (torch.as_tensor shares it)."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}


def chain_tensor(ptr: int, nbytes: int, device=None):
    """uint8 tensor over a chain buffer returned by `zkb_groth16_prove_begin`: CUDA memory on a GPU context, host
    memory under the host-emulation test library (device=None)."""
    import torch
    if device is None or str(device) == "cpu":
        import ctypes
        return torch.frombuffer((ctypes.c_uint8 * nbytes).from_address(ptr), dtype=torch.uint8)
    return torch.as_tensor(_DevBuf(ptr, nbytes), device=device)


def wm_chain_mask(rank: int, world: int) -> int:
    """Chains this rank computes: chain k belongs to rank k mod world (all three when world < 3: replicated)."""
    if world < 3:
        return 7
    return sum(1 << k for k in range(3) if k % world == rank)


def prove_partial_shared_wm(ctx, pk_h, r1cs_h, z: Optional[np.ndarray], group=None, device=None) -> np.ndarray:
    """This rank's partial sums with the witness map shared between the ranks (see the module docstring)."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    mask = wm_chain_mask(rank, world)
    with ctx.lock:                                               # one open proof per context: begin .. end is one critical section
        ptrs, nbytes = ctx.prove_begin(pk_h, r1cs_h, z, mask)
        if mask != 7:
            for k in range(3):
                dist.broadcast(chain_tensor(ptrs[k], nbytes, device), src=dist.get_global_rank(group, k % world) if group else k % world,
                               group=group)
            if device is not None and str(device) != "cpu":
                torch.cuda.current_stream(device).synchronize()  # the chains must be in memory before prove_end reads them
        return ctx.prove_end(pk_h, r1cs_h)


def submit_shared_wm(ctx, pk_h, r1cs_h, z: Optional[np.ndarray], group=None, device=None) -> int:
    """Pipelined form of `prove_partial_shared_wm`: enqueue this rank's share of one proof (chains exchanged in the middle)
    and return its ticket without waiting for the result — `ctx.prove_collect_partial(ticket)` follows later, typically after
    the next proof has been submitted."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    mask = wm_chain_mask(rank, world)
    on_gpu = device is not None and str(device) != "cpu"
    with ctx.lock:
        if mask == 7 or not on_gpu:
            ticket, ptrs, nbytes = ctx.prove_begin_async(pk_h, r1cs_h, z, mask)
            if mask != 7:
                for k in range(3):
                    dist.broadcast(chain_tensor(ptrs[k], nbytes, device), src=dist.get_global_rank(group, k % world) if group else k % world,
                                   group=group)
        else:
            # stream-ordered exchange: torch's current stream waits for this rank's chains, the three NCCL broadcasts follow on
            # it (ProcessGroupNCCL orders its own stream against the current one), and the finish step waits for that stream —
            # the host enqueues and moves on, it never blocks between two proofs
            stream = torch.cuda.current_stream(device).cuda_stream
            ticket, ptrs, nbytes = ctx.prove_begin_async(pk_h, r1cs_h, z, mask | 0x80000000)
            ctx.prove_chains_to_stream(ticket, stream)
            for k in range(3):
                dist.broadcast(chain_tensor(ptrs[k], nbytes, device), src=dist.get_global_rank(group, k % world) if group else k % world,
                               group=group)
            ctx.prove_stream_to_finish(ticket, stream)
        ctx.prove_end_async(ticket)
    return ticket


def prove_sharded(session, z: Optional[np.ndarray], r: int, s: int, finalize_session=None, dst: int = 0, group=None,
                  device=None) -> Optional[bytes]:
    """One proof across all ranks of `group`.  `session` holds this rank's key shard; `finalize_session`
    (rank `dst` only) may be any session of the same key.  Returns the raw proof on rank `dst`, None elsewhere."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    if rank == dst:
        (finalize_session or session).ctx.finalize_prepare((finalize_session or session).pk_h, r, s)
    if world >= 3:
        partial = prove_partial_shared_wm(session.ctx, session.pk_h, session.r1cs_h, z, group, device)
    else:
        partial = session.prove_partial(z)
    allp = gather_partials(partial, group, device)
    if rank != dst:
        return None
    return (finalize_session or session).finalize(allp, world, r, s)


def msm_g1_sharded(ctx, points: bytes, scalars: np.ndarray, group=None, device=None) -> bytes:
    """BASELINE config 5 at N > 1: sum_i s_i P_i with the (scalar, point) pairs split by contiguous index range over the ranks
    (every rank passes the FULL vectors and computes only its slice with `zkb_msm_g1`), the per-rank affine results
    all-gathered (one point per rank) and added on the host.  Returns the point in ark's uncompressed encoding on every rank."""
    import torch
    import torch.distributed as dist
    from .curves import CURVES
    from .verify import _pairing
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    scalars = np.ascontiguousarray(scalars, dtype=np.uint64)
    n = scalars.shape[0]
    curve_name = next(c.name for c in CURVES.values() if c.id == ctx.curve)
    pr = _pairing(curve_name)
    nb = 2 * pr.c.fq_bytes
    lo, hi = n * rank // world, n * (rank + 1) // world
    mine = np.frombuffer(ctx.msm(1, points[lo * nb:hi * nb], scalars[lo:hi]), dtype=np.uint8).copy()
    t = torch.from_numpy(mine)
    if device is not None:
        t = t.to(device)
    out = torch.empty(world * nb, dtype=torch.uint8, device=t.device)
    dist.all_gather_into_tensor(out, t, group=group)
    raw = out.cpu().numpy().tobytes()
    acc = None
    for k in range(world):
        part = raw[k * nb:(k + 1) * nb]
        if part[-1] & 0x40:                      # infinity flag
            continue
        x = int.from_bytes(part[:nb // 2], "little")
        y = int.from_bytes(part[nb // 2:], "little")
        acc = pr.g1_add(acc, (x, y))
    if acc is None:
        res = bytearray(nb)
        res[-1] = 0x40
        return bytes(res)
    return acc[0].to_bytes(nb // 2, "little") + acc[1].to_bytes(nb // 2, "little")
