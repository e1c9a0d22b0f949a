"""Base-range-sharded proofs at every witness-map shape, under both reductions, at 1 to 64 ranks, each rank's partial MSMs
checked on their own against a CPU model (tests/proof_model.py) and every folded proof against a CPU reference.

Rank r of R owns the r-th contiguous slice of every query's bases (b2g_pk_load) and computes five partial MSMs (H, L, A,
B1, B2); the partials are folded in rank order by b2g_prove_finish after a host exchange, or inside the proof graph over
peer memory by b2g_prove_sharded_p2p.  The case matrix reaches empty slices and slices of one base in every query, uneven
splits, the LibsnarkReduction key's H query of domain - 1 bases, and all three outcomes of the per-shard B compaction; the
CPU tests below assert that from sharding.shard_range instead of assuming it.

CPU tests: the model's rank partials fold to each query's whole MSM and assemble to the oracle's proof.  GPU tests (host
exchange, every rank a shard context on device 0): every rank's 768-byte partial equals the model's, prove_finish gives the
same bytes on every rank's context, and those equal the CPU reference and the unsharded proof, with (r, s) given to
prove_partial and without.  GPU test (peer memory, one process per rank): a sequence of keys on contexts wired once."""
import functools
import os
import random

import numpy as np
import pytest

from circom_compat_b200 import CircomReduction, LibsnarkReduction
from oracle import pyref as o
from proof_model import (EDGE_RS, CpuFixedBase, assemble, b_head_circuit, check_partial, expect_proofs, fold, libsnark_h,
                         libsnark_key_with_domain_h, perturbed, points, query_slices, ragged_circuit, rank_partials,
                         shape_case, shard_bases, shard_scalars, trapdoor_keys, witness_map_mont, QUERIES)

R = o.R_MOD
REDUCTIONS = {'circom': CircomReduction, 'libsnark': LibsnarkReduction}
# 2^1 / 2^2 hand-made circuits (w0 alone: every witness query empty; an empty L query), 2^5 / 2^11 / 2^13 chains, ragged rows,
# the circom-like 2^13 circuit (sparse B) and 8192 wires of which B touches 1..2047 (B compaction on some ranks only)
SHAPES = ['w0_only', 'private_w1', 'empty_l', 'chain5', 'chain11', 'chain13', 'ragged', 'circomlike13', 'b_head']
COUNTS = [1, 2, 3, 5, 7]
CASES = [(shape, red, count) for shape in SHAPES for red in REDUCTIONS for count in COUNTS + ([64] if shape in ('w0_only', 'chain11') else [])]
# (r, s) of the five proofs of a case: proof j proves assignment j % 3, with (r, s) handed to prove_partial when j is even
RS = EDGE_RS + [(random.Random(0x5A4D).randrange(R), random.Random(0x5A4E).randrange(R))]


def _case_id(case):
    return '%s-%s-%d' % case


def _circuit(shape):
    """(circuit, three assignments with the all-zero one in the middle)"""
    if shape == 'ragged':
        circ, ws = ragged_circuit()
        return circ, ws[:3]
    if shape == 'circomlike13':
        from circom_compat_b200 import synth
        circ, w = synth.circomlike_circuit(13)
        return circ, [w, [1] + [0] * (len(w) - 1), perturbed(w, random.Random(13))]
    if shape == 'b_head':
        return b_head_circuit()
    return shape_case(shape)


class _Setup:
    """a key of the shape and reduction, its three assignments and their scalars, and the CPU reference of the five proofs"""
    def __init__(self, fixed_base, shape, red, domain_h=False):
        from circom_compat_b200 import fr_to_mont
        self.red = REDUCTIONS[red]
        self.circ, self.ws = _circuit(shape)
        if domain_h:
            self.pk, self.td, self.cm = libsnark_key_with_domain_h(fixed_base, self.circ)
        else:
            self.pk, self.td, self.cm = trapdoor_keys(fixed_base, self.circ, self.red)
        self.wm = [fr_to_mont(w) for w in self.ws]
        self.bases = shard_bases(self.pk)
        self.scal = [shard_scalars(wm, witness_map_mont(self.pk, self.cm, wm, self.red)) for wm in self.wm]
        self.expect = expect_proofs(self.pk, self.td, self.cm, RS, [self.ws[j % 3] for j in range(len(RS))], self.red)

    def rank_rows(self, wi, count):
        return [rank_partials(self.pk, self.bases, self.scal[wi], k, count) for k in range(count)]


@functools.lru_cache(maxsize=None)
def _cpu_setup(shape, red, domain_h=False):
    """keys built on the CPU (the oracle's fixed-base multiplication gives the device's bytes), kept for the whole session"""
    return _Setup(CpuFixedBase(), shape, red, domain_h)


# ------------------------------------------------------------------------------------------------ the matrix's reach (CPU)
def _b_compaction(pk, rank, count):
    """b2g_pk_load's per-shard B compaction rule (prover.cu, the Q_B1 step of its query loop): a rank builds its B1 / B2
    tables over the real points only when its slice has at least 1024 bases and fewer than 80 % of them are real points in
    B1 or B2.  Returns b_compact (the number of real points kept), or None when the rank does not compact."""
    lo, hi, _ = query_slices(pk, rank, count)['b1']
    b1 = np.asarray(pk.b_g1_query).reshape(pk.n_vars, -1)[1 + lo:1 + hi]
    b2 = np.asarray(pk.b_g2_query).reshape(pk.n_vars, -1)[1 + lo:1 + hi]
    real = int(np.count_nonzero(b1.any(axis=1) | b2.any(axis=1)))
    return real if hi - lo >= 1024 and real * 5 < (hi - lo) * 4 else None


def test_case_matrix_reaches_every_edge():
    """over the GPU matrix: every query has a rank with an empty slice, a rank with exactly one base and an uneven split;
    the LibsnarkReduction H query of domain - 1 bases is split; B compaction happens with b_compact = 0 and > 0, and does
    not happen, and at least one key mixes compacting and non-compacting ranks"""
    reach = {q: set() for q in QUERIES}
    lib_h_split = False
    compaction, mixed = set(), []
    for shape, red, count in CASES:
        st = _cpu_setup(shape, red)
        if red == 'libsnark':
            assert len(st.pk.h_query) == st.pk.domain_size == st.circ.domain_size - 1
        slices = [query_slices(st.pk, k, count) for k in range(count)]
        for q in QUERIES:
            sizes = [sl[q][1] - sl[q][0] for sl in slices]
            reach[q] |= {'empty'} if 0 in sizes else set()
            reach[q] |= {'one'} if 1 in sizes else set()
            reach[q] |= {'uneven'} if len(set(sizes)) > 1 else set()
        lib_h_split |= red == 'libsnark' and sum(sl['h'][1] > sl['h'][0] for sl in slices) > 1
        outcome = [_b_compaction(st.pk, k, count) for k in range(count)]
        compaction |= {'none' if b is None else 'zero' if b == 0 else 'some' for b in outcome}
        if None in outcome and any(b is not None for b in outcome):
            mixed.append((shape, red, count))
    assert all(reach[q] == {'empty', 'one', 'uneven'} for q in QUERIES), reach
    assert lib_h_split
    assert compaction == {'none', 'zero', 'some'}, compaction
    assert ('b_head', 'circom', 5) in mixed, mixed


# ------------------------------------------------------------------------------------------------ the rank model (CPU)
@pytest.mark.parametrize('case', CASES, ids=_case_id)
def test_rank_partials_fold_to_the_oracle_proof(case):
    """the model's partials of every rank add up to each query's whole MSM, and folded in rank order and assembled they give
    the CPU reference proof of each (r, s)"""
    shape, red, count = case
    st = _cpu_setup(shape, red)
    for wi in range(3):
        whole = points(rank_partials(st.pk, st.bases, st.scal[wi], 0, 1))
        acc = fold([points(rows) for rows in st.rank_rows(wi, count)])
        assert acc == whole, [q for q in QUERIES if acc[q] != whole[q]]
        for j in range(wi, len(RS), 3):
            assert assemble(st.pk, acc, *RS[j]) == st.expect[j], (wi, RS[j])


def test_libsnark_domain_h_key_model():
    """a LibsnarkReduction key with domain H bases: h of a satisfying assignment has a zero top coefficient, so its proofs
    equal those of the arkworks key (domain - 1 H bases) of the same trapdoor, and the rank model folds to them"""
    st, ark = _cpu_setup('chain11', 'libsnark', True), _cpu_setup('chain11', 'libsnark')
    assert len(st.pk.h_query) == st.pk.domain_size == st.circ.domain_size
    for wi in (0, 1):                                                  # the satisfying assignments of the chain
        assert libsnark_h(st.cm, st.ws[wi])[-1] == 0
        acc = fold([points(rows) for rows in st.rank_rows(wi, 5)])
        for j in range(wi, len(RS), 3):
            assert st.expect[j] == ark.expect[j]
            assert assemble(st.pk, acc, *RS[j]) == st.expect[j]


# ------------------------------------------------------------------------------------------------ host exchange (GPU)
def _prove_host_exchange(ctx, st, count, witnesses):
    """one key at `count` shard contexts on device 0: every rank's partial against the model, then prove_finish on every
    rank's context and the unsharded proof against the CPU reference, with (r, s) given to prove_partial and without"""
    from circom_compat_b200 import Context, Groth16, release
    pk, cm, red = st.pk, st.cm, st.red
    ranks = [Context(0, k, count) for k in range(count)]
    try:
        rows = {wi: st.rank_rows(wi, count) for wi in witnesses}
        for j, (r, s) in enumerate(RS):
            wi = j % 3
            if wi not in witnesses:
                continue
            early = (r, s) if j % 2 == 0 else (None, None)
            parts = [Groth16.prove_partial(pk, cm, st.wm[wi], cx, *early, reduction=red) for cx in ranks]
            bad = [(k, q, err) for k, part in enumerate(parts) for q, err in check_partial(part, rows[wi][k])]
            assert not bad, ('(rank, query, error) of partials that differ from the model', j, bad)
            got = [Groth16.prove_finish(pk, np.stack(parts), r, s, cx).data for cx in ranks]
            assert [k for k, p in enumerate(got) if p != st.expect[j]] == [], ('ranks whose folded proof differs', j)
            whole = Groth16.create_proof_with_reduction_and_matrices(pk, r, s, cm, cm.num_instance_variables, cm.num_constraints,
                                                                     st.wm[wi], ctx, red).data
            assert whole == st.expect[j], ('unsharded proof differs from the CPU reference', j)
    finally:
        for cx in ranks:
            cx.close()
        release(pk); release(cm)


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=_case_id)
def test_host_exchange(ctx, case):
    shape, red, count = case
    _prove_host_exchange(ctx, _cpu_setup(shape, red), count, (0, 1, 2))


@pytest.mark.gpu
@pytest.mark.parametrize('count', [1, 3, 5])
def test_host_exchange_libsnark_domain_h_key(ctx, count):
    """a LibsnarkReduction key with domain H bases, which b2g_prove accepts as well: proved with the Circom witness map it
    would give a proof of the wrong h, so only the reduction's own map gives the reference bytes (satisfying assignments)"""
    _prove_host_exchange(ctx, _cpu_setup('chain11', 'libsnark', True), count, (0, 1))


# ------------------------------------------------------------------------------------------------ peer memory (GPU)
# the keys one set of wired contexts proves in turn, two epochs each: (shape, reduction, proofs j of the case: assignment
# j % 3 with RS[j]); the arena is sized for domain 8192 (circomlike13, prepared before the wiring)
P2P_SEQUENCE = [('chain11', 'circom', (0, 2)),        # split witness map, H of 2048 split unevenly
                ('w0_only', 'circom', (1, 4)),        # empty slices, H slices of 0 elements, no witness words on ranks >= 3
                ('circomlike13', 'circom', (3, 2)),   # sparse B
                ('chain11', 'libsnark', (0, 2)),      # replicated map over peer memory
                ('chain14', 'circom', (4, 1)),        # larger than the arena: replicated map
                ('chain11', 'circom', (1, 3))]        # back to the first key: the proof graph is captured again


def _p2p_worker(rank, world, port, q, arena_key, jobs):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    os.environ['MASTER_ADDR'] = '127.0.0.1'; os.environ['MASTER_PORT'] = str(port)
    os.environ['B2G_P2P_TIMEOUT_MS'] = '15000'                   # a broken exchange fails instead of spinning
    import torch
    import torch.distributed as dist
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from circom_compat_b200 import Groth16, Context, sharding
        ctx = Context(rank % torch.cuda.device_count(), rank, world)
        ctx.prepare(*arena_key)                                  # before the wiring: the exchange arena is sized for this domain
        sharding.connect_p2p(ctx, dist)
        dist.barrier()
        out = []
        for pk, cm, red, proofs in jobs:
            ctx.prepare(pk, cm, red.ID)
            out.append([Groth16.prove_sharded_p2p(pk, cm, r, s, wm, ctx, red).data.hex() for r, s, wm in proofs])
        q.put((rank, out))
        dist.barrier()
        ctx.close()
    except Exception as e:                                       # noqa: BLE001
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize('world', [3, 5])
def test_peer_memory_key_sequence(world):
    """b2g_prove_sharded_p2p, one process per rank (one GPU each if the box has them, else all on device 0), wired once and
    proving the keys of P2P_SEQUENCE in turn; the parent builds the keys and compares every rank's proofs with the CPU
    reference"""
    import torch.multiprocessing as mp
    from circom_compat_b200 import fr_to_mont, synth
    arena = _cpu_setup('circomlike13', 'circom')
    chain14 = synth.chain_circuit(1 << 14)
    setups = {}
    jobs, expect = [], []
    for shape, red, js in P2P_SEQUENCE:
        if shape == 'chain14':
            pk, td, cm = trapdoor_keys(CpuFixedBase(), chain14, CircomReduction)
            wl = [synth.chain_witness(1 << 14, 5), synth.chain_witness(1 << 14, 0)]
            exp = expect_proofs(pk, td, cm, [RS[j] for j in js], wl, CircomReduction)
            proofs = [(*RS[j], fr_to_mont(w)) for j, w in zip(js, wl)]
        else:
            st = setups.setdefault((shape, red), _cpu_setup(shape, red))
            pk, cm = st.pk, st.cm
            exp = [st.expect[j] for j in js]
            proofs = [(*RS[j], st.wm[j % 3]) for j in js]
        jobs.append((pk, cm, REDUCTIONS[red], proofs))
        expect.append([p.hex() for p in exp])
    mpc = mp.get_context('spawn')
    q = mpc.Queue()
    port = 30100 + (os.getpid() % 300) + world
    procs = [mpc.Process(target=_p2p_worker, args=(r, world, port, q, (arena.pk, arena.cm), jobs)) for r in range(world)]
    [p.start() for p in procs]
    res = dict(q.get(timeout=600) for _ in range(world))
    [p.join(timeout=60) for p in procs]
    for rank in range(world):
        assert not isinstance(res[rank], str), (rank, res[rank])
        bad = [(P2P_SEQUENCE[j][:2], e) for j in range(len(jobs)) for e in range(2) if res[rank][j][e] != expect[j][e]]
        assert not bad, ('rank', rank, '(key, epoch) whose proof differs from the CPU reference', bad)
