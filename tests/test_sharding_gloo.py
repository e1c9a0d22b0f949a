"""world_size-2 gloo test of the multi-GPU path's host logic (no GPU): each rank computes the partial MSMs of its
base range with the CPU oracle, the 768-byte partials go through the same all_gather helper bench.py uses, and the
rank-ordered fold + proof assembly must give the golden proof on every rank."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, q):
    sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
    os.environ['MASTER_ADDR'] = '127.0.0.1'; os.environ['MASTER_PORT'] = str(port)
    import torch.distributed as dist
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from circom_compat_b200 import read_zkey, fr_to_mont, sharding
        from oracle import cref as c, pyref as o
        from proof_model import assemble, fold, partial_points, partial_record, rank_partials, shard_bases, shard_scalars
        g = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'golden_vectors.json')))['complex_zkey']
        data = open(os.path.join(ROOT, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'), 'rb').read()
        pk, cm = read_zkey(data)
        za = c.zkey_arrays(data)
        wm = fr_to_mont(o.chain_witness(pk.n_vars, g['a']))
        h = c.witness_map(cm.num_constraints, cm.num_instance_variables, pk.n_vars, za['a_csr'], za['b_csr'], wm, nthreads=2)
        part = partial_record(rank_partials(pk, shard_bases(pk), shard_scalars(wm, h), rank, world, nthreads=2))
        allp = sharding.all_gather_partials(part, dist)
        assert allp.shape == (world, sharding.PARTIAL_BYTES) and np.array_equal(allp[rank], part)
        # fold in rank order and assemble (ark-groth16 create_proof_with_assignment) with the big-int oracle
        proof = assemble(pk, fold([partial_points(p) for p in allp]), int(g['r']), int(g['s']))
        q.put((rank, proof.hex() == g['proof_hex']))
    finally:
        dist.destroy_process_group()


def test_shard_ranges_partition():
    from circom_compat_b200 import sharding
    for total in (0, 1, 5, 10001, 1 << 20):
        for count in (1, 2, 3, 8):
            rs = [sharding.shard_range(total, r, count) for r in range(count)]
            assert rs[0][0] == 0 and rs[-1][1] == total
            assert all(rs[i][1] == rs[i + 1][0] for i in range(count - 1))


def test_two_rank_sharded_proof_over_gloo():
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = [q.get(timeout=300) for _ in range(2)]
    [p.join(timeout=60) for p in procs]
    assert sorted(res) == [(0, True), (1, True)]
