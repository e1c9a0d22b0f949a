"""Base-range sharding of one proof over several GPUs (SURVEY.md 8e): host-side logic shared by bench.py and the tests.

Rank r of R owns the r-th contiguous slice of every query (the C side applies the same split in b2g_pk_load), computes
five partial MSM results, and the 768-byte partials are exchanged with ONE all-gather (NCCL on GPUs, gloo in the CPU
tests).  Every rank then folds the partials in rank order (b2g_prove_finish) and obtains identical proof bytes.
"""
from __future__ import annotations

import numpy as np

from .groth16 import CircomReduction, Groth16

PARTIAL_BYTES = 768
# offsets inside a partial: [H, L, A, B1] as G1 XYZZ (128 B) then B2 as G2 XYZZ (256 B)
PARTIAL_LAYOUT = {'h': (0, 128), 'l': (128, 128), 'a': (256, 128), 'b1': (384, 128), 'b2': (512, 256)}


def shard_range(total: int, rank: int, count: int):
    """[lo, hi) of `total` items owned by `rank` (identical to the split in prover.cu:b2g_pk_load)."""
    return total * rank // count, total * (rank + 1) // count


def query_totals(n_vars: int, n_public: int, domain_size: int) -> dict:
    """Number of (base, scalar) pairs per query and the first scalar each pairs with.  L is re-indexed onto w[1..]
    (its first n_public bases are points at infinity) so that L, A, B1, B2 share one digit sort."""
    return {'h': (domain_size, 'h', 0), 'l': (n_vars - 1, 'w', 1), 'a': (n_vars - 1, 'w', 1), 'b1': (n_vars - 1, 'w', 1), 'b2': (n_vars - 1, 'w', 1)}


def all_gather_partials(partial: np.ndarray, dist, device=None, group=None) -> np.ndarray:
    """One all-gather of this rank's 768-byte partial; returns (world, 768) uint8 on the host."""
    import torch
    world = dist.get_world_size()
    mine = torch.from_numpy(np.ascontiguousarray(partial, dtype=np.uint8).reshape(PARTIAL_BYTES).copy())
    if device is not None:
        mine = mine.to(device, non_blocking=True)
    out = torch.empty(world * PARTIAL_BYTES, dtype=torch.uint8, device=mine.device)
    dist.all_gather_into_tensor(out, mine, group=group)
    return out.cpu().numpy().reshape(world, PARTIAL_BYTES)


def prove_sharded(ctx, pk, matrices, w_mont, r, s, dist, device=None, group=None, reduction=CircomReduction):
    """One proof on a sharded context: partial MSMs -> all-gather -> identical fold on every rank."""
    part = Groth16.prove_partial(pk, matrices, w_mont, ctx, r, s, reduction)
    allp = all_gather_partials(part, dist, device, group)
    return Groth16.prove_finish(pk, allp, r, s, ctx)


def connect_p2p(ctx, dist, group=None) -> None:
    """Exchange the CUDA-IPC handles of every rank's exchange arena (host-side, once) so that Groth16.prove_sharded_p2p
    can fold the partials - and, with >= 3 ranks, read the three transformed vectors of the split witness map - straight out
    of NVLink peer memory.  Call ctx.prepare(pk, matrices) first: the arena is sized for the prepared domain."""
    handles = [None] * dist.get_world_size()
    dist.all_gather_object(handles, ctx.p2p_export(), group=group)
    ctx.p2p_import(handles)


def connect_p2p_local(ctxs) -> None:
    """Same wiring for shard contexts living in one process, ONE CONTEXT PER GPU.  (Several shard contexts on the same
    device of one process can alias the same hardware work queue, where a rank waiting for its peer blocks that peer's
    kernels; separate processes - the deployment model, one per GPU - do not share queues.)"""
    import ctypes as C
    from . import _native as N
    arr = (C.c_void_p * len(ctxs))(*[c._h for c in ctxs])
    N.check(N.lib().b2g_p2p_connect_local(arr, len(ctxs)))
