"""CPU model of whole and base-range-sharded Groth16 proofs, shared by tests/test_prove_many_shapes.py,
tests/test_sharded_shapes.py, tests/test_sharding_gloo.py and tests/test_host.py.  TEST INFRASTRUCTURE ONLY.

Circuits and trapdoor keys of every witness-map shape, the CPU references of a proof (the oracle's proof bytes, oracle/cref.c,
for CircomReduction; the trapdoor closed form for LibsnarkReduction), and the five partial MSMs one shard rank computes
(H, L, A, B1, B2 over the rank's slice of each query, as b2g_pk_load splits them), folded in rank order and assembled as
ark-groth16 0.5.0 create_proof_with_assignment does."""
import random

import numpy as np

from circom_compat_b200 import sharding
from oracle import cref as c
from oracle import pyref as o
from oracle import xyzz as X

R = o.R_MOD
EDGE_RS = [(0, 0), (0, 1), (1, 0), (R - 1, R - 1)]


class CpuFixedBase:
    """stands in for Context in synth.setup without a GPU: the group elements come from the oracle (the same bytes as the
    device's b2g_fixed_base_g1 / g2)"""
    def fixed_base_g1(self, s): return c.fixed_base_g1(s)
    def fixed_base_g2(self, s): return c.fixed_base_g2(s)


# ------------------------------------------------------------------------------------------------ circuits and keys
def oracle_key(pk, cm):
    za = dict(n_vars=pk.n_vars, n_public=pk.n_public, domain_size=pk.domain_size, num_constraints=cm.num_constraints, a_csr=cm.a, b_csr=cm.b)
    for name in ('alpha_g1', 'beta_g1', 'delta_g1', 'beta_g2', 'delta_g2', 'a_query', 'b_g1_query', 'b_g2_query', 'l_query', 'h_query'):
        za[name] = np.ascontiguousarray(getattr(pk, name), dtype=np.uint64)
    return za


def perturbed(w, rng, share=3):
    """w with w1 (the first public input) and a share of the private wires redrawn: a distinct, in general unsatisfying,
    assignment whose proof is still fully determined"""
    v = list(w)
    v[1] = rng.randrange(R)
    for i in rng.sample(range(2, len(v)), (len(v) - 2) // share):
        v[i] = rng.randrange(R) if i % 2 else rng.randrange(2)
    return v


def trapdoor_keys(ctx, circ, reduction, seed=0xB200):
    """(pk, td, cm) of a trapdoor key of the reduction's flavour; cm carries C for LibsnarkReduction.  ctx: a Context, or
    CpuFixedBase() to build the key on the CPU"""
    from circom_compat_b200 import LibsnarkReduction, synth
    lib = reduction is LibsnarkReduction
    pk, td = synth.setup(ctx, circ, seed=seed, flavour='libsnark' if lib else 'circom')
    return pk, td, circ.matrices(with_c=lib)


def shape_case(name):
    """(circuit, three distinct assignments with the all-zero one in the middle)"""
    from circom_compat_b200 import synth
    z, one = np.array([0]), [1]
    rng = random.Random(name)
    if name == 'w0_only':          # 1 * 1 = 1: the assignment is w0 alone, domain 2; the proofs differ by (r, s) only
        return synth.Circuit(1, 1, 1, (z, z, one), (z, z, one), (z, z, one)), [[1], [1], [1]]
    if name == 'private_w1':       # w1 * 1 = w1, w1 private: domain 2, one L base
        return synth.Circuit(2, 1, 1, (z, np.array([1]), one), (z, z, one), (z, np.array([1]), one)), [[1, 5], [1, 0], [1, R - 1]]
    if name == 'empty_l':          # the same with w1 public: n_vars == num_inputs, domain 4, the L query is empty
        return synth.Circuit(2, 2, 1, (z, np.array([1]), one), (z, z, one), (z, np.array([1]), one)), [[1, 5], [1, 0], [1, R - 1]]
    log_n = int(name[5:])          # 'chainK': squaring chain of domain 2^K
    n = 1 << log_n
    return synth.chain_circuit(n), [synth.chain_witness(n, 3 + log_n), synth.chain_witness(n, 0),
                                    perturbed(synth.chain_witness(n, 7 + log_n), rng)]


def ragged_circuit():
    """rows of 0 to 6 terms, repeated wires, explicit 0, 1 and r - 1 coefficients in A, B and C; w0 and two public inputs"""
    from circom_compat_b200 import synth
    rng = random.Random(31)
    n_vars, li, m = 40, 3, 29
    mats = []
    for terms in (lambda i: i % 7, lambda i: (i * 3) % 5, lambda i: (i * 5) % 4):
        rows, cols, vals = [], [], []
        for i in range(m):
            for _ in range(terms(i)):
                rows.append(i); cols.append(rng.randrange(n_vars)); vals.append(rng.choice([0, 1, R - 1, rng.randrange(R)]))
        mats.append((np.array(rows, dtype=np.int64), np.array(cols, dtype=np.int64), vals))
    circ = synth.Circuit(n_vars, li, m, *mats)
    ws = [[1] + [rng.randrange(R) for _ in range(n_vars - 1)] for _ in range(3)]
    return circ, [ws[0], [1] + [0] * (n_vars - 1), ws[1], ws[2]]


def b_head_circuit():
    """8192 wires, domain 8192, B touching only wires 1..2047: over five ranks, rank 0's B slice is all real points, rank 1's
    a quarter real and ranks 2..4 all at infinity.  Returns (circuit, three assignments with the all-zero one in the middle)."""
    from circom_compat_b200 import synth
    n_vars, m = 8192, 8190
    rows = np.arange(m, dtype=np.int64)
    circ = synth.Circuit(n_vars, 2, m, (rows, rows + 2, [1] * m), (rows, 1 + rows % 2047, [R - 1] * m),
                         (rows, (rows * 7 + 3) % n_vars, [1] * m))
    rng = random.Random(2047)
    w = [1] + [rng.randrange(R) if i % 3 else rng.randrange(2) for i in range(1, n_vars)]
    return circ, [w, [1] + [0] * (n_vars - 1), perturbed(w, rng)]


def libsnark_key_with_domain_h(ctx, circ, seed=0xB200):
    """(pk, td, cm) of a LibsnarkReduction key with domain H bases (tau^i Z(tau) / delta for i < domain) instead of
    arkworks' domain - 1: the other H length b2g_prove accepts for LibsnarkReduction.  Its proofs equal the arkworks key's
    for witnesses that satisfy the circuit, whose h has a zero top coefficient."""
    from circom_compat_b200 import LibsnarkReduction, synth
    pk, td, cm = trapdoor_keys(ctx, circ, LibsnarkReduction, seed)
    n = circ.domain_size
    top = pow(td.tau, n - 1, R) * (pow(td.tau, n, R) - 1) * pow(td.delta, -1, R) % R
    td.h_t = td.h_t + [top]
    pk.h_query = np.concatenate([np.asarray(pk.h_query, dtype=np.uint64), ctx.fixed_base_g1(c.ints_to_limbs([top]))])
    pk.domain_size = n
    return pk, td, cm


# ------------------------------------------------------------------------------------------------ whole-proof references
def proof_bytes(dlogs):
    """the 256-byte proofs ([da] G1, [db] G2, [dc] G1) of a list of (da, db, dc), by the oracle's fixed-base multiplication"""
    g1 = c.limbs_to_ints(c.fq_from_mont(c.fixed_base_g1(c.ints_to_limbs([x for da, _, dc in dlogs for x in (da, dc)]))))
    g2 = c.limbs_to_ints(c.fq_from_mont(c.fixed_base_g2(c.ints_to_limbs([db for _, db, _ in dlogs]))))
    return [b''.join(v.to_bytes(32, 'little') for v in g1[4 * j:4 * j + 2] + g2[4 * j:4 * j + 4] + g1[4 * j + 2:4 * j + 4])
            for j in range(len(dlogs))]


def expect_circom(pk, cm, rs, ws):
    """CircomReduction: the CPU oracle's proof of each (r, s, w) on the same key"""
    from circom_compat_b200 import fr_to_mont
    za = oracle_key(pk, cm)
    return [c.prove(za, r, s, fr_to_mont(w)) for (r, s), w in zip(rs, ws)]


def libsnark_h(cm3, w):
    """canonical ints of h = (a*b - c) / Z from the oracle's LibsnarkReduction witness map (domain_size coefficients)"""
    from circom_compat_b200 import fr_to_mont
    return c.limbs_to_ints(c.fr_from_mont(c.witness_map_libsnark(cm3.num_constraints, cm3.num_instance_variables, cm3.a, cm3.b, cm3.c, fr_to_mont(w))))


def expect_libsnark(td, cm3, rs, ws):
    """LibsnarkReduction on a trapdoor key: the closed form of each proof with h from the oracle's witness map (holds for
    assignments that do not satisfy the circuit too)"""
    from circom_compat_b200 import synth
    dl = []
    for (r, s), w in zip(rs, ws):
        dl.append(synth.expected_proof_dlogs(td, w, libsnark_h(cm3, w)[:len(td.h_t)], r, s, cm3.num_instance_variables))
    return proof_bytes(dl)


def expect_proofs(pk, td, cm, rs, ws, reduction):
    from circom_compat_b200 import LibsnarkReduction
    return expect_libsnark(td, cm, rs, ws) if reduction is LibsnarkReduction else expect_circom(pk, cm, rs, ws)


# ------------------------------------------------------------------------------------------------ shard ranks
QUERIES = tuple(sharding.PARTIAL_LAYOUT)                      # h, l, a, b1, b2: the order of a 768-byte partial


def shard_bases(pk):
    """every query's bases in the order the shards split them: L re-indexed onto w[1..] (its first n_public entries points at
    infinity), A / B1 / B2 without query[0], which the proof adds separately"""
    li = pk.n_public + 1
    l_padded = np.concatenate([np.zeros((li - 1, 8), dtype=np.uint64), np.asarray(pk.l_query, dtype=np.uint64).reshape(-1, 8)])
    return {'h': np.asarray(pk.h_query, dtype=np.uint64), 'l': l_padded, 'a': np.asarray(pk.a_query, dtype=np.uint64)[1:],
            'b1': np.asarray(pk.b_g1_query, dtype=np.uint64)[1:], 'b2': np.asarray(pk.b_g2_query, dtype=np.uint64)[1:]}


def shard_scalars(w_mont, h_mont):
    """the canonical scalar vectors the queries pair with: 'w' (the assignment) and 'h' (the witness map's output)"""
    return {'w': c.fr_from_mont(w_mont), 'h': c.fr_from_mont(h_mont)}


def witness_map_mont(pk, cm, w_mont, reduction):
    """h (Montgomery) from the oracle's witness map of the reduction"""
    from circom_compat_b200 import LibsnarkReduction
    if reduction is LibsnarkReduction:
        return c.witness_map_libsnark(cm.num_constraints, cm.num_instance_variables, cm.a, cm.b, cm.c, w_mont)
    return c.witness_map(cm.num_constraints, cm.num_instance_variables, pk.n_vars, cm.a, cm.b, w_mont)


def query_slices(pk, rank, count):
    """{query: (lo, hi, total)} of the rank's slice of every query (sharding.shard_range over sharding.query_totals)"""
    out = {}
    for q, (total, _, _) in sharding.query_totals(pk.n_vars, pk.n_public, pk.domain_size).items():
        out[q] = sharding.shard_range(total, rank, count) + (total,)
    return out


def rank_partials(pk, bases, scal, rank, count, nthreads=0):
    """{query: affine row (Montgomery words, all-zero = infinity)} of the rank's five partial MSMs, by the oracle's MSM"""
    out = {}
    for q, (total, sv, soff) in sharding.query_totals(pk.n_vars, pk.n_public, pk.domain_size).items():
        lo, hi = sharding.shard_range(total, rank, count)
        f = c.msm_g2 if q == 'b2' else c.msm_g1
        out[q] = f(bases[q][lo:hi], scal[sv][soff + lo:soff + hi], nthreads)
    return out


def partial_record(rows):
    """the 768-byte partial of a rank's affine rows, each as an XYZZ record with ZZ = ZZZ = 1"""
    part = np.zeros(sharding.PARTIAL_BYTES, dtype=np.uint8)
    for q, (off, size) in sharding.PARTIAL_LAYOUT.items():
        g2 = q == 'b2'
        part[off:off + size] = np.frombuffer(X.record(X.aff(rows[q], g2), (1, 0) if g2 else 1, g2).tobytes(), dtype=np.uint8)
    return part


def points(rows):
    """{query: affine point, canonical (None = infinity)} of a rank's affine rows"""
    return {q: X.aff(rows[q], q == 'b2') for q in QUERIES}


def partial_points(part):
    """{query: affine point, canonical (None = infinity)} of a 768-byte partial whose records have ZZ = ZZZ = 1 or 0"""
    out = {}
    for q, (off, size) in sharding.PARTIAL_LAYOUT.items():
        rec = np.frombuffer(np.ascontiguousarray(part[off:off + size]).tobytes(), dtype='<u8')
        out[q] = X.aff(rec[:len(rec) // 2], q == 'b2')
    return out


def check_partial(part, rows):
    """[(query, what is wrong)] of a device partial (768 bytes of unnormalised XYZZ Montgomery records) against the model's
    affine rows; empty = every query holds the model's point"""
    bad = []
    for q, (off, size) in sharding.PARTIAL_LAYOUT.items():
        words = np.frombuffer(np.ascontiguousarray(part[off:off + size], dtype=np.uint8).tobytes(), dtype='<u8')
        err = X.check_record(words, X.aff(rows[q], q == 'b2'), q == 'b2')
        if err:
            bad.append((q, err))
    return bad


def fold(points_per_rank):
    """rank-order sum of every query's partial points"""
    acc = {q: None for q in QUERIES}
    for pts in points_per_rank:
        for q in QUERIES:
            acc[q] = (o.G2 if q == 'b2' else o.G1).add(acc[q], pts[q])
    return acc


def assemble(pk, acc, r, s):
    """proof bytes from the folded MSMs (ark-groth16 0.5.0 create_proof_with_assignment, as b2g_prove_finish assembles it)"""
    def pt1(arr): return o._g1_from(np.ascontiguousarray(arr, dtype=np.uint64).tobytes())
    def pt2(arr): return o._g2_from(np.ascontiguousarray(arr, dtype=np.uint64).tobytes())
    delta1, delta2 = pt1(pk.delta_g1), pt2(pk.delta_g2)
    A = o.G1.sum([o.G1.mul(delta1, r), pt1(pk.a_query[0]), acc['a'], pt1(pk.alpha_g1)])
    B1 = o.G1.sum([o.G1.mul(delta1, s), pt1(pk.b_g1_query[0]), acc['b1'], pt1(pk.beta_g1)])
    B2 = o.G2.sum([o.G2.mul(delta2, s), pt2(pk.b_g2_query[0]), acc['b2'], pt2(pk.beta_g2)])
    C = o.G1.sum([o.G1.mul(A, s), o.G1.mul(B1, r), o.G1.neg(o.G1.mul(delta1, r * s % R)), acc['l'], acc['h']])
    return o.proof_to_bytes(A, B2, C)
