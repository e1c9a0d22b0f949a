"""Groth16.create_proofs (b2g_prove_many) at every witness-map shape, under both reductions, each batched proof checked on
its own against a CPU reference: the oracle's proof bytes (oracle/cref.c) for CircomReduction, the trapdoor closed form for
LibsnarkReduction (with h from the oracle's witness map) and for the 2^21 batch (with no h at all).

The batch runs every kernel of the chain once, with the proof on an extra grid dimension (spmv / bit-reversing copy:
blockIdx.y, NTT passes: blockIdx.z, MSM sort and reduce: blockIdx.y, glue: one CTA per proof).  Each batch mixes witnesses
that differ in their public inputs and private wires with the all-zero witness (only w0 = 1) and the (r, s) edge pairs, so
a kernel that reads or writes another proof's slice changes some proof."""
import os
import random

import pytest

from oracle import pyref as o
from proof_model import (EDGE_RS, expect_libsnark, expect_proofs, perturbed, proof_bytes, ragged_circuit, shape_case,
                         trapdoor_keys)

pytestmark = pytest.mark.gpu

R = o.R_MOD


def _many(pk, cm, rs, ws, ctx, reduction):
    from circom_compat_b200 import Groth16, fr_to_mont
    return [p.data for p in Groth16.create_proofs(pk, rs, cm, [fr_to_mont(w) for w in ws], ctx, reduction)]


def _assert_batch(got, expect):
    assert len(got) == len(expect)
    bad = [j for j, (g, e) in enumerate(zip(got, expect)) if g != e]
    assert not bad, 'proofs %s of %d differ from the CPU reference' % (bad, len(got))


def _rs(rng, count, shift):
    """(r, s) of a batch: the edge pairs from EDGE_RS[shift] on, the last entry random"""
    return [EDGE_RS[(shift + j) % 4] if j < min(count - 1, 4) else (rng.randrange(R), rng.randrange(R)) for j in range(count)]


def _reductions():
    from circom_compat_b200 import CircomReduction, LibsnarkReduction
    return [pytest.param(CircomReduction, id='circom'), pytest.param(LibsnarkReduction, id='libsnark')]


# ------------------------------------------------------------------------------------------------ domain sizes
# 2^1 / 2^2: hand-made circuits; below 2^5 the radix-2 pass kernel runs; 2^5, 2^9: one radix-8 pass; 2^11, 2^13: block pass
# plus strided passes
SHAPES = ['w0_only', 'private_w1', 'empty_l', 'chain2', 'chain3', 'chain4', 'chain5', 'chain9', 'chain11', 'chain13']


@pytest.mark.parametrize('reduction', _reductions())
@pytest.mark.parametrize('shape', SHAPES)
def test_domain_sizes(ctx, shape, reduction):
    from circom_compat_b200 import release
    circ, ws = shape_case(shape)
    pk, td, cm = trapdoor_keys(ctx, circ, reduction)
    rs = _rs(random.Random(shape), 3, SHAPES.index(shape))
    got = _many(pk, cm, rs, ws, ctx, reduction)
    _assert_batch(got, expect_proofs(pk, td, cm, rs, ws, reduction))
    # the same batch rotated by one: every proof follows its own (r, s, w)
    assert _many(pk, cm, rs[1:] + rs[:1], ws[1:] + ws[:1], ctx, reduction) == got[1:] + got[:1]
    release(pk); release(cm)


# ------------------------------------------------------------------------------------------------ pass schedules
@pytest.fixture(scope='module')
def chain13_both(ctx):
    """2^13 squaring chain, a key of each flavour, one batch of three and its CPU expectation per reduction"""
    from circom_compat_b200 import CircomReduction, LibsnarkReduction, synth, release
    circ, ws = shape_case('chain13')
    rs = _rs(random.Random(1313), 3, 3)
    out = {}
    for red in (CircomReduction, LibsnarkReduction):
        pk, td, cm = trapdoor_keys(ctx, circ, red, seed=0x1313)
        out[red] = (pk, expect_proofs(pk, td, cm, rs, ws, red))
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
    _assert_batch(got, proof_bytes([synth.expected_proof_dlogs_independent(td, circ, w, r, s) for (r, s), w in zip(rs, ws)]))


# ------------------------------------------------------------------------------------------------ sparse B, LibsnarkReduction
@pytest.fixture(scope='module')
def sparse_b_libsnark(ctx):
    """circom-like 2^12 key of the libsnark flavour (most B bases at infinity): the real witness, the all-zero one and three
    perturbed copies"""
    from circom_compat_b200 import LibsnarkReduction, synth, release
    circ, w = synth.circomlike_circuit(12)
    pk, td, cm = trapdoor_keys(ctx, circ, LibsnarkReduction)
    rng = random.Random(12)
    ws = [list(w), perturbed(w, rng), [1] + [0] * (len(w) - 1), perturbed(w, rng, 2), perturbed(w, rng, 5)]
    rs = _rs(rng, 5, 0)
    yield pk, cm, rs, ws, expect_libsnark(td, cm, rs, ws)
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
@pytest.mark.parametrize('reduction', _reductions())
def test_ragged_rows_and_repeated_columns(ctx, reduction):
    from circom_compat_b200 import release
    circ, ws = ragged_circuit()
    assert circ.domain_size == 32
    pk, td, cm = trapdoor_keys(ctx, circ, reduction, seed=0x31)
    rs = _rs(random.Random(31), 4, 1)
    _assert_batch(_many(pk, cm, rs, ws, ctx, reduction), expect_proofs(pk, td, cm, rs, ws, reduction))
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
