"""Groth16.create_proofs (b2g_prove_many) at every witness-map shape, under both reductions, each batched proof checked on
its own against a CPU reference: the oracle's proof bytes (oracle/cref.c) for CircomReduction, the trapdoor closed form for
LibsnarkReduction (with h from the oracle's witness map) and for the 2^21 batch (with no h at all).

The batch runs every kernel of the chain once, with the proof on an extra grid dimension (spmv / bit-reversing copy:
blockIdx.y, NTT passes: blockIdx.z, MSM sort and reduce: blockIdx.y, glue: one CTA per proof).  Each batch mixes witnesses
that differ in their public inputs and private wires with the all-zero witness (only w0 = 1) and the (r, s) edge pairs, so
a kernel that reads or writes another proof's slice changes some proof."""
import os
import random

import numpy as np
import pytest

from oracle import cref as c
from oracle import pyref as o

pytestmark = pytest.mark.gpu

R = o.R_MOD
EDGE_RS = [(0, 0), (0, 1), (1, 0), (R - 1, R - 1)]


def _oracle_key(pk, cm):
    za = dict(n_vars=pk.n_vars, n_public=pk.n_public, domain_size=pk.domain_size, num_constraints=cm.num_constraints, a_csr=cm.a, b_csr=cm.b)
    for name in ('alpha_g1', 'beta_g1', 'delta_g1', 'beta_g2', 'delta_g2', 'a_query', 'b_g1_query', 'b_g2_query', 'l_query', 'h_query'):
        za[name] = np.ascontiguousarray(getattr(pk, name), dtype=np.uint64)
    return za


def _many(pk, cm, rs, ws, ctx, reduction):
    from circom_compat_b200 import Groth16, fr_to_mont
    return [p.data for p in Groth16.create_proofs(pk, rs, cm, [fr_to_mont(w) for w in ws], ctx, reduction)]


def _proof_bytes(dlogs):
    """the 256-byte proofs ([da] G1, [db] G2, [dc] G1) of a list of (da, db, dc), by the oracle's fixed-base multiplication"""
    g1 = c.limbs_to_ints(c.fq_from_mont(c.fixed_base_g1(c.ints_to_limbs([x for da, _, dc in dlogs for x in (da, dc)]))))
    g2 = c.limbs_to_ints(c.fq_from_mont(c.fixed_base_g2(c.ints_to_limbs([db for _, db, _ in dlogs]))))
    return [b''.join(v.to_bytes(32, 'little') for v in g1[4 * j:4 * j + 2] + g2[4 * j:4 * j + 4] + g1[4 * j + 2:4 * j + 4])
            for j in range(len(dlogs))]


def _expect_circom(pk, cm, rs, ws):
    """CircomReduction: the CPU oracle's proof of each (r, s, w) on the same key"""
    from circom_compat_b200 import fr_to_mont
    za = _oracle_key(pk, cm)
    return [c.prove(za, r, s, fr_to_mont(w)) for (r, s), w in zip(rs, ws)]


def _expect_libsnark(td, cm3, rs, ws):
    """LibsnarkReduction on a trapdoor key: the closed form of each proof with h from the oracle's witness map (holds for
    assignments that do not satisfy the circuit too)"""
    from circom_compat_b200 import fr_to_mont, synth
    dl = []
    for (r, s), w in zip(rs, ws):
        h = c.limbs_to_ints(c.fr_from_mont(c.witness_map_libsnark(cm3.num_constraints, cm3.num_instance_variables, cm3.a, cm3.b, cm3.c, fr_to_mont(w))))
        dl.append(synth.expected_proof_dlogs(td, w, h[:len(td.h_t)], r, s, cm3.num_instance_variables))
    return _proof_bytes(dl)


def _assert_batch(got, expect):
    assert len(got) == len(expect)
    bad = [j for j, (g, e) in enumerate(zip(got, expect)) if g != e]
    assert not bad, 'proofs %s of %d differ from the CPU reference' % (bad, len(got))


def _perturbed(w, rng, share=3):
    """w with w1 (the first public input) and a share of the private wires redrawn: a distinct, in general unsatisfying,
    assignment whose proof is still fully determined"""
    v = list(w)
    v[1] = rng.randrange(R)
    for i in rng.sample(range(2, len(v)), (len(v) - 2) // share):
        v[i] = rng.randrange(R) if i % 2 else rng.randrange(2)
    return v


def _rs(rng, count, shift):
    """(r, s) of a batch: the edge pairs from EDGE_RS[shift] on, the last entry random"""
    return [EDGE_RS[(shift + j) % 4] if j < min(count - 1, 4) else (rng.randrange(R), rng.randrange(R)) for j in range(count)]


def _keys(ctx, circ, reduction, seed=0xB200):
    """(pk, td, cm) of a trapdoor key of the reduction's flavour; cm carries C for LibsnarkReduction"""
    from circom_compat_b200 import LibsnarkReduction, synth
    lib = reduction is LibsnarkReduction
    pk, td = synth.setup(ctx, circ, seed=seed, flavour='libsnark' if lib else 'circom')
    return pk, td, circ.matrices(with_c=lib)


def _expect(pk, td, cm, rs, ws, reduction):
    from circom_compat_b200 import LibsnarkReduction
    return _expect_libsnark(td, cm, rs, ws) if reduction is LibsnarkReduction else _expect_circom(pk, cm, rs, ws)


def _reductions():
    from circom_compat_b200 import CircomReduction, LibsnarkReduction
    return [pytest.param(CircomReduction, id='circom'), pytest.param(LibsnarkReduction, id='libsnark')]


# ------------------------------------------------------------------------------------------------ domain sizes
def _shape(name):
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
                                    _perturbed(synth.chain_witness(n, 7 + log_n), rng)]


# 2^1 / 2^2: hand-made circuits; below 2^5 the radix-2 pass kernel runs; 2^5, 2^9: one radix-8 pass; 2^11, 2^13: block pass
# plus strided passes
SHAPES = ['w0_only', 'private_w1', 'empty_l', 'chain2', 'chain3', 'chain4', 'chain5', 'chain9', 'chain11', 'chain13']


@pytest.mark.parametrize('reduction', _reductions())
@pytest.mark.parametrize('shape', SHAPES)
def test_domain_sizes(ctx, shape, reduction):
    from circom_compat_b200 import release
    circ, ws = _shape(shape)
    pk, td, cm = _keys(ctx, circ, reduction)
    rs = _rs(random.Random(shape), 3, SHAPES.index(shape))
    got = _many(pk, cm, rs, ws, ctx, reduction)
    _assert_batch(got, _expect(pk, td, cm, rs, ws, reduction))
    # the same batch rotated by one: every proof follows its own (r, s, w)
    assert _many(pk, cm, rs[1:] + rs[:1], ws[1:] + ws[:1], ctx, reduction) == got[1:] + got[:1]
    release(pk); release(cm)


# ------------------------------------------------------------------------------------------------ pass schedules
@pytest.fixture(scope='module')
def chain13_both(ctx):
    """2^13 squaring chain, a key of each flavour, one batch of three and its CPU expectation per reduction"""
    from circom_compat_b200 import CircomReduction, LibsnarkReduction, synth, release
    circ, ws = _shape('chain13')
    rs = _rs(random.Random(1313), 3, 3)
    out = {}
    for red in (CircomReduction, LibsnarkReduction):
        pk, td, cm = _keys(ctx, circ, red, seed=0x1313)
        out[red] = (pk, _expect(pk, td, cm, rs, ws, red))
        release(cm)
    yield circ, ws, rs, out
    for pk, _ in out.values():
        release(pk)


@pytest.mark.parametrize('env', [dict(B2G_NTT_RADIX2='1'), dict(B2G_NTT_TL='5'), dict(B2G_NTT_TL='6', B2G_NTT_MAXK='2'),
                                 dict(B2G_NTT_TL='7', B2G_NTT_MAXK='4'), dict(B2G_NTT_TL='11'), dict(B2G_NTT_MAXK='5'),
                                 dict(B2G_NTT_RADIX2='1', B2G_NTT_MAXK='5')],
                         ids=lambda e: ','.join('%s=%s' % (k[8:], v) for k, v in e.items()))
def test_pass_schedules(ctx, monkeypatch, chain13_both, env):
    """every NTT pass shape under a batch: the schedule is fixed when the matrices load, so fresh matrices per setting"""
    from circom_compat_b200 import LibsnarkReduction, release
    circ, ws, rs, out = chain13_both
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    for red, (pk, expect) in out.items():
        cm = circ.matrices(with_c=red is LibsnarkReduction)
        try:
            _assert_batch(_many(pk, cm, rs, ws, ctx, red), expect)
        finally:
            release(cm)


# ------------------------------------------------------------------------------------------------ >= 2^21 schedule
def test_2p21_batch_closed_form(ctx):
    """two 2^21 chain proofs in one pass: the block pass and the 2-D strided tiles of at most 7 index bits, against the
    trapdoor closed form that takes no h"""
    from circom_compat_b200 import CircomReduction, synth, release
    n = 1 << 21
    circ = synth.chain_circuit(n)
    pk, td = synth.setup(ctx, circ)
    cm = circ.matrices()
    ws = [synth.chain_witness(n, a) for a in (5, 13)]
    rs = [(R - 1, 0x1234567890abcdef), (0xfedcba0987654321, 1)]
    got = _many(pk, cm, rs, ws, ctx, CircomReduction)
    release(pk); release(cm)
    _assert_batch(got, _proof_bytes([synth.expected_proof_dlogs_independent(td, circ, w, r, s) for (r, s), w in zip(rs, ws)]))


# ------------------------------------------------------------------------------------------------ sparse B, LibsnarkReduction
@pytest.fixture(scope='module')
def sparse_b_libsnark(ctx):
    """circom-like 2^12 key of the libsnark flavour (most B bases at infinity): the real witness, the all-zero one and three
    perturbed copies"""
    from circom_compat_b200 import LibsnarkReduction, synth, release
    circ, w = synth.circomlike_circuit(12)
    pk, td, cm = _keys(ctx, circ, LibsnarkReduction)
    rng = random.Random(12)
    ws = [list(w), _perturbed(w, rng), [1] + [0] * (len(w) - 1), _perturbed(w, rng, 2), _perturbed(w, rng, 5)]
    rs = _rs(rng, 5, 0)
    yield pk, cm, rs, ws, _expect_libsnark(td, cm, rs, ws)
    release(pk); release(cm)


@pytest.mark.parametrize('compact', [True, False], ids=['b_compact', 'no_b_compact'])
def test_libsnark_sparse_b(ctx, monkeypatch, sparse_b_libsnark, compact):
    from circom_compat_b200 import LibsnarkReduction, release
    pk, cm, rs, ws, expect = sparse_b_libsnark
    if not compact:
        monkeypatch.setenv('B2G_NO_B_COMPACT', '1')
    release(pk)                                                        # B2G_NO_B_COMPACT is read when the key loads
    try:
        _assert_batch(_many(pk, cm, rs, ws, ctx, LibsnarkReduction), expect)
    finally:
        release(pk)


# ------------------------------------------------------------------------------------------------ ragged rows
def _ragged_circuit():
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


@pytest.mark.parametrize('reduction', _reductions())
def test_ragged_rows_and_repeated_columns(ctx, reduction):
    from circom_compat_b200 import release
    circ, ws = _ragged_circuit()
    assert circ.domain_size == 32
    pk, td, cm = _keys(ctx, circ, reduction, seed=0x31)
    rs = _rs(random.Random(31), 4, 1)
    _assert_batch(_many(pk, cm, rs, ws, ctx, reduction), _expect(pk, td, cm, rs, ws, reduction))
    release(pk); release(cm)


# ------------------------------------------------------------------------------------------------ R1CS fixture
def test_r1cs_fixture_batch(ctx):
    """mycircuit.r1cs (a * b = c, c public) with a LibsnarkReduction key of generate_random_parameters_with_reduction: the
    batched proofs of distinct valid witnesses equal their single proofs, verify, and fail with a wrong public input"""
    from circom_compat_b200 import R1CSFile, R1CS, Groth16, LibsnarkReduction, Proof, fr_to_mont, release
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'mycircuit.r1cs')
    r1 = R1CS.from_file(R1CSFile.new(open(path, 'rb').read()))
    circ = r1.to_circuit()
    cm = circ.matrices(with_c=True)
    pk = Groth16.generate_random_parameters_with_reduction(circ, random.Random(77), ctx, LibsnarkReduction)
    ws = [[1, a * b % R, a, b] for a, b in ((3, 11), (0, 9), (R - 1, 2), (123456789, R - 5), (1, 1))]
    rs = _rs(random.Random(77), len(ws), 2)
    got = _many(pk, cm, rs, ws, ctx, LibsnarkReduction)
    singles = [Groth16.create_proof_with_reduction_and_matrices(pk, r, s, cm, r1.num_inputs, len(r1.constraints), fr_to_mont(w), ctx,
                                                                LibsnarkReduction).data for (r, s), w in zip(rs, ws)]
    assert got == singles
    assert len(set(got)) == len(got)
    proofs = [Proof(d) for d in got]
    assert Groth16.verify_many(pk, [w[1:r1.num_inputs] for w in ws], proofs, ctx) == [True] * len(ws)
    assert Groth16.verify_many(pk, [[(w[1] + 1) % R] for w in ws], proofs, ctx) == [False] * len(ws)
    release(pk); release(cm)
