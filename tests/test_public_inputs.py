"""Setup, key checks, proofs and verification of circuits with many public inputs (tests/public_inputs_model.py).

The public-input count moves code on every stage: the input rows a[m + j] = w[j] of the witness map, the IC / L split and the
gamma / delta choice of the setup routes, the L query padded with n_public points at infinity in the prover (whole ranks of a
sharded proof pair such points with nonzero scalars), the public rows and the rho offset of the key check, and the per-input
work of the verifiers (one warp per (proof, input), the IC sums, a window table per input in a key batch).  The shapes cross
one 256-thread CTA of input rows, let the input rows fill or decide the domain, and reach n_public = 0, an empty L query and
2048 public inputs.

CPU: the circuit family and its witnesses, the setup model against synth and pyref, and the key-check equations for honest
and forged key scalars.  GPU: the three setup routes byte for byte, the key check on honest keys and forgeries, the
contribution check, the witness map and proofs of both reductions against the CPU oracle and the trapdoor closed form,
sharded proofs rank by rank, and every verifier with real keys."""
import ctypes as C
import random

import numpy as np
import pytest

from circom_compat_b200 import CircomReduction, LibsnarkReduction, synth
from circom_compat_b200.zkey import R_MOD
from oracle import pyref as o
import public_inputs_model as P
import setup_check_model as SC
import setup_model as SM

R = R_MOD
SHAPE_NAMES = list(P.SHAPES)
REDUCTIONS = {'circom': CircomReduction, 'libsnark': LibsnarkReduction}
KEY_FIELDS = ('alpha_g1', 'beta_g1', 'beta_g2', 'gamma_g2', 'delta_g1', 'delta_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query',
              'b_g2_query', 'l_query', 'h_query')


def _secrets(seed):
    rng = random.Random(seed)
    return [rng.randrange(1, R) for _ in range(5)]           # alpha, beta, gamma, delta, tau


def _mentions(mat, col):
    """the rows of a coordinate-list matrix holding column col"""
    rows, cols, _ = mat
    return set(np.asarray(rows)[np.asarray(cols) == col].tolist())


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_shapes_cross_their_boundaries():
    dom = {name: P.shape_circuit(name)[0].domain_size for name in SHAPE_NAMES}
    circ = {name: P.shape_circuit(name)[0] for name in SHAPE_NAMES}
    assert circ['p0'].num_inputs == 1
    assert [circ[k].num_inputs for k in ('p254', 'p255', 'p256')] == [255, 256, 257]
    assert circ['fill1024'].num_constraints + circ['fill1024'].num_inputs == dom['fill1024'] == 1024
    assert circ['over1024'].num_constraints + circ['over1024'].num_inputs == 1025 and dom['over1024'] == 2048
    assert dom['ordinary'] == 2048 and circ['ordinary'].num_inputs == 48
    assert circ['wide'].n_vars == dom['wide'] == 8192
    assert circ['most'].num_inputs == 2049
    assert circ['all_public'].n_vars == circ['all_public'].num_inputs == 300


@pytest.mark.parametrize('mode', P.MODES)
def test_each_mode_places_the_inputs(mode):
    m, ni = 7, 20
    circ, witness = P.public_circuit(m, ni, ni if mode == 'all_public' else 40, mode, seed=3)
    mats = {'in_a': circ.A, 'in_b': circ.B, 'in_c': circ.C}
    for j in range(1, ni):
        seen = [_mentions(mat, j) for mat in (circ.A, circ.B, circ.C)]
        if mode == 'unused':
            assert seen == [set(), set(), set()], j
        elif mode in mats:
            assert _mentions(mats[mode], j) and sum(map(bool, seen)) == 1, j
        elif mode == 'hot':
            assert seen == [set(range(m))] * 3 if j == ni - 1 else seen == [set(), set(), set()], j
    if mode == 'in_a':                       # coefficients 1, r - 1 and random on the input columns
        cols, vals = np.asarray(circ.A[1]), circ.A[2]
        got = {vals[k] for k in range(len(vals)) if 1 <= cols[k] < ni}
        assert 1 in got and R - 1 in got and len(got) > 2
    for pub in P.public_values(ni - 1):
        w = witness(pub)
        assert w[1:ni] == [v % R for v in pub] and not P.unsatisfied_rows(circ, w)


@pytest.mark.parametrize('name', SHAPE_NAMES)
def test_witnesses_satisfy_the_circuit(name):
    circ, witness = P.shape_circuit(name)
    for k, pub in enumerate(P.public_values(circ.num_inputs - 1)):
        w = witness(pub, wseed=k)
        assert len(w) == circ.n_vars and w[0] == 1 and w[1:circ.num_inputs] == pub
        assert P.unsatisfied_rows(circ, w) == [], (name, k)


@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('name', SHAPE_NAMES)
def test_setup_model_agrees_with_synth_and_pyref(name, flavour):
    circ, _ = P.shape_circuit(name)
    alpha, beta, gamma, delta, tau = _secrets(len(name) + circ.num_inputs)
    got = SM.setup_scalars(circ, tau, alpha, beta, gamma, delta, flavour)
    ref = synth.setup_scalars(circ, trapdoor=(tau, alpha, beta, gamma, delta), flavour=flavour)
    assert got['n'] == circ.domain_size and got['lagrange'] == ref.lagrange
    assert got['a'] == ref.a_t and got['b'] == ref.b_t
    assert got['ic'] == ref.ic_t and got['l'] == ref.l_t and got['h'] == ref.h_t
    assert len(got['ic']) == circ.num_inputs and len(got['l']) == circ.n_vars - circ.num_inputs
    if flavour == 'circom':                  # the oracle's closed form takes gamma = 1
        rows = [[[], [], []] for _ in range(circ.num_constraints)]
        for x, (rs, cs, vs) in enumerate((circ.A, circ.B, circ.C)):
            for r, c, v in zip(np.asarray(rs).tolist(), np.asarray(cs).tolist(), vs):
                rows[r][x].append((v, c))
        pr = o.trapdoor_setup_scalars([r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows], circ.n_vars,
                                      circ.num_inputs, tau, alpha, beta, delta)
        one = SM.setup_scalars(circ, tau, alpha, beta, 1, delta, 'circom')
        assert pr['n'] == one['n'] and pr['a'] == one['a'] and pr['b'] == one['b']
        assert pr['ic'] == one['ic'] and pr['l'] == one['l'] and pr['h'] == one['h']


CHECK_SHAPES = ['p0', 'p256', 'over1024', 'most', 'all_public']


@pytest.mark.parametrize('name', CHECK_SHAPES)
def test_key_check_model_on_honest_and_forged_keys(name):
    """E1-E5 hold for the honest key scalars, every forgery breaks E4 (the IC / L equation) and nothing before it, and a
    dropped or added IC point falls to the count rule with the circuit's num_inputs"""
    circ, _ = P.shape_circuit(name)
    ni, nv = circ.num_inputs, circ.n_vars
    for flavour in ('circom', 'libsnark'):
        tau, alpha, beta, delta, rho, sigma = _secrets(ni)[:5] + [1234567]
        key = SC.key_scalars(circ, tau, alpha, beta, delta, flavour)
        assert P.broken_equations(circ, key, tau, alpha, beta, delta, rho, sigma, flavour) == []
        forged = P.forgeries(ni, nv - ni)
        assert len(forged) == (1 if name == 'all_public' else 3)
        for what, edit in forged:
            broken = P.broken_equations(circ, P.edited(key, edit), tau, alpha, beta, delta, rho, sigma, flavour)
            assert broken == ['gamma_abc_g1 / l_query'], (what, broken)
        nh = circ.domain_size - (flavour == 'libsnark')
        assert P.count_rule(circ, nv, ni, nv - ni, nh, flavour) is None
        for n_ic in (ni - 1, ni + 1):
            assert P.count_rule(circ, nv, n_ic, nv - ni, nh, flavour) == ('gamma_abc_g1', ni)


def test_sharded_cases_reach_the_padding_and_the_b_compaction():
    """every sharded shape has a rank whose L slice lies inside the n_public points at infinity, and 'most' at two ranks
    compacts its B query, so that B2G_NO_B_COMPACT changes the path"""
    from proof_model import CpuFixedBase, query_slices, trapdoor_keys
    for name in SHARD_SHAPES:
        circ, _ = P.shape_circuit(name)
        pk = _FakeKey(circ)
        for count in SHARD_COUNTS:
            l_slices = [query_slices(pk, k, count)['l'] for k in range(count)]
            padded = [k for k, (lo, hi, _) in enumerate(l_slices) if hi > lo and hi <= circ.num_inputs - 1]
            assert padded, (name, count)
    circ, _ = P.shape_circuit('most')
    pk, _, _ = trapdoor_keys(CpuFixedBase(), circ, CircomReduction)
    lo, hi, _ = query_slices(pk, 0, 2)['b1']
    assert P.b_compaction(pk, lo, hi) is not None


class _FakeKey:
    """the sizes sharding.query_totals reads"""
    def __init__(self, circ):
        self.n_vars, self.n_public, self.domain_size = circ.n_vars, circ.num_inputs - 1, circ.domain_size


# ------------------------------------------------------------------------------------------------------------------ GPU
def _limbs(vals):
    return synth._ints_to_limbs([v % R for v in vals])


def _assert_same_key(pk, ref):
    for name in KEY_FIELDS:
        a, b = np.ascontiguousarray(getattr(pk, name)), np.ascontiguousarray(getattr(ref, name))
        assert a.shape == b.shape and a.tobytes() == b.tobytes(), name
    assert (pk.n_vars, pk.n_public, pk.domain_size) == (ref.n_vars, ref.n_public, ref.domain_size)


class _Ceremony:
    """a power-13 ceremony for known (tau, alpha, beta) on the standard generators, and its phase-2 preparation"""
    POWER = 13

    def __init__(self, ctx, seed=17):
        from circom_compat_b200 import Groth16, Powers
        rng = random.Random(seed)
        self.tau, self.alpha, self.beta = (rng.randrange(1, R) for _ in range(3))
        n = 1 << self.POWER
        t = [1] * (2 * n - 1)
        for i in range(1, 2 * n - 1):
            t[i] = t[i - 1] * self.tau % R
        self.powers = Powers(self.POWER, self.POWER, ctx.fixed_base_g1(_limbs(t)), ctx.fixed_base_g2(_limbs(t[:n])),
                             ctx.fixed_base_g1(_limbs([self.alpha * v for v in t[:n]])),
                             ctx.fixed_base_g1(_limbs([self.beta * v for v in t[:n]])), ctx.fixed_base_g2(_limbs([self.beta])))
        self.prepared = Groth16.prepare_powers_of_tau(self.powers, ctx=ctx)
        assert self.prepared.lagrange.power == self.POWER


_STATE = {}


def _ceremony(ctx):
    if 'cer' not in _STATE:
        _STATE['cer'] = _Ceremony(ctx)
    return _STATE['cer']


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('name', SHAPE_NAMES)
def test_setup_routes_agree(ctx, name, flavour):
    """generate_parameters_with_qap equals synth.setup; from the ceremony, the powers route and the prepared-Lagrange route
    equal the qap key with gamma = delta = 1, and it passes the key check before and after a contribution"""
    from circom_compat_b200 import Groth16
    circ, _ = P.shape_circuit(name)
    red = REDUCTIONS[flavour]
    alpha, beta, gamma, delta, tau = _secrets(circ.num_inputs * 3 + len(name))
    pk = Groth16.generate_parameters_with_qap(circ, alpha, beta, gamma, delta, tau=tau, ctx=ctx, reduction=red)
    ref, _ = synth.setup(ctx, circ, trapdoor=(tau, alpha, beta, gamma, delta), flavour=flavour)
    _assert_same_key(pk, ref)
    cer = _ceremony(ctx)
    qap = Groth16.generate_parameters_with_qap(circ, cer.alpha, cer.beta, 1, 1, tau=cer.tau, ctx=ctx, reduction=red)
    powers = Groth16.generate_parameters_from_powers_of_tau(circ, cer.powers, ctx, red)
    lagrange = Groth16.generate_parameters_from_powers_of_tau(circ, cer.prepared, ctx, red)
    _assert_same_key(powers, qap)
    _assert_same_key(lagrange, qap)
    for key in (pk, qap, powers, lagrange):
        assert key.gamma_abc_g1.shape == (circ.num_inputs, 8) and key.n_public == circ.num_inputs - 1
        assert np.asarray(key.l_query).shape == (circ.n_vars - circ.num_inputs, 8)
    if name == 'all_public':
        assert all(np.asarray(key.l_query).size == 0 for key in (pk, qap, powers, lagrange))
    r = Groth16.verify_proving_key(circ, cer.powers, powers, reduction=red, ctx=ctx)
    assert r and r.reason is None, r.reason
    after = Groth16.contribute(powers, random.Random(circ.num_inputs), ctx)
    r = Groth16.verify_proving_key(circ, cer.powers, after, reduction=red, ctx=ctx)
    assert r and r.reason is None, r.reason


def _with(pk, **fields):
    from circom_compat_b200 import ProvingKey
    arrs = {k: np.array(getattr(pk, k), copy=True) for k in KEY_FIELDS}
    arrs.update(fields)
    return ProvingKey(pk.n_vars, pk.n_public, pk.domain_size, *(arrs[k] for k in KEY_FIELDS))


def _raw_check(ctx, circ, powers, pk, red, challenges):
    """b2g_setup_check with the counts of the key's own arrays (the Python entry refuses a wrong count before the library)"""
    from circom_compat_b200 import _native as N
    from circom_compat_b200.groth16 import _circuit_desc, _powers_desc
    from circom_compat_b200.keycheck import KEY_FIELDS as ORDER
    d, keep, nv, ni, size, nh = _circuit_desc(circ, red)
    pd, arrays = _powers_desc(powers, size)
    arrs = {k: np.ascontiguousarray(getattr(pk, k), dtype=np.uint64) for k in ORDER}
    kd = N.KeyDesc()
    kd.n_vars, kd.n_ic = nv, arrs['gamma_abc_g1'].size // 8
    kd.n_l, kd.n_h = arrs['l_query'].size // 8, arrs['h_query'].size // 8
    for k, a in arrs.items():
        setattr(kd, k, a.ctypes.data if a.size else None)
    cb = np.frombuffer(b''.join(int(v).to_bytes(32, 'little') for v in challenges), dtype=np.uint8).copy()
    rep = N.SetupReport()
    assert N.lib().b2g_setup_check(ctx._h, C.byref(d), C.byref(pd), C.byref(kd), cb.ctypes.data, C.byref(rep)) == N.B2G_OK
    return rep


@pytest.mark.gpu
@pytest.mark.parametrize('name', CHECK_SHAPES)
def test_key_check_refuses_forgeries_as_the_model_predicts(ctx, name):
    """a contributed ceremony key (delta = x): IC[n_public] swapped with L[0], a middle IC point and L[0] moved by G fail with
    the equation the model names; one IC point dropped or added fails the count rule with the circuit's num_inputs"""
    from circom_compat_b200 import Groth16
    from circom_compat_b200.keycheck import KEY_FIELDS as ORDER, report_reason
    circ, _ = P.shape_circuit(name)
    ni, nv = circ.num_inputs, circ.n_vars
    cer, x, rho, sigma = _ceremony(ctx), 987654321, 1234567, 7654321
    pk = Groth16.contribute(Groth16.generate_parameters_from_powers_of_tau(circ, cer.powers, ctx), x=x, ctx=ctx)
    key = SC.key_scalars(circ, cer.tau, cer.alpha, cer.beta, x, 'circom')
    assert P.broken_equations(circ, key, cer.tau, cer.alpha, cer.beta, x, rho, sigma, 'circom') == []
    assert Groth16.verify_proving_key(circ, cer.powers, pk, ctx=ctx, challenges=[rho, sigma])
    g = ctx.fixed_base_g1(_limbs([1]))[0]
    ic, l = np.array(pk.gamma_abc_g1, copy=True), np.array(pk.l_query, copy=True)
    points = {'IC[middle] + G': dict(gamma_abc_g1=np.concatenate([ic[:ni // 2], ctx.test_op(8, ic[ni // 2], g), ic[ni // 2 + 1:]]))}
    if nv > ni:
        s_ic, s_l = ic.copy(), l.copy()
        s_ic[-1], s_l[0] = l[0], ic[-1]
        points['IC[n_public] <-> L[0]'] = dict(gamma_abc_g1=s_ic, l_query=s_l)
        points['L[0] + G'] = dict(l_query=np.concatenate([ctx.test_op(8, l[0], g), l[1:]]))
    forged = P.forgeries(ni, nv - ni)
    assert sorted(points) == sorted(what for what, _ in forged)
    for what, edit in forged:
        broken = P.broken_equations(circ, P.edited(key, edit), cer.tau, cer.alpha, cer.beta, x, rho, sigma, 'circom')
        fake = _with(pk, **points[what])
        for ch in ([rho, sigma], None):
            r = Groth16.verify_proving_key(circ, cer.powers, fake, ctx=ctx, challenges=ch)
            assert not r and r.reason == P.EQUATION_REASONS[broken[0]], (what, r.reason)
    nh = circ.domain_size
    for n_ic, arr in ((ni - 1, ic[:-1]), (ni + 1, np.concatenate([ic, g[None]]))):
        field, index = P.count_rule(circ, nv, n_ic, nv - ni, nh, 'circom')
        fake = _with(pk, gamma_abc_g1=arr)
        assert Groth16.verify_proving_key(circ, cer.powers, fake, ctx=ctx).reason == f"gamma_abc_g1 holds {n_ic} points; the circuit needs {ni}"
        rep = _raw_check(ctx, circ, cer.powers, fake, CircomReduction, [rho, sigma])
        assert (rep.ok, rep.rule, ORDER[rep.field], rep.index) == (0, 6, field, index)
        assert report_reason(rep) == f"gamma_abc_g1: the circuit needs {ni} points"


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['most', 'all_public'])
def test_contribution_check(ctx, name):
    """verify_contribution after contribute on a key of 2049 inputs and on one whose L query is empty (n_l = 0)"""
    from circom_compat_b200 import Groth16
    circ, _ = P.shape_circuit(name)
    cer = _ceremony(ctx)
    before = Groth16.generate_parameters_from_powers_of_tau(circ, cer.powers, ctx)
    after = Groth16.contribute(before, random.Random(5), ctx)
    assert np.asarray(after.l_query).shape == np.asarray(before.l_query).shape
    assert Groth16.verify_contribution(before, after, ctx)
    assert Groth16.verify_contribution(before, Groth16.contribute(after, x=3, ctx=ctx), ctx)
    assert not Groth16.verify_contribution(before, _with(after, h_query=before.h_query), ctx)
    assert not Groth16.verify_contribution(before, _with(after, gamma_abc_g1=after.gamma_abc_g1[::-1].copy()), ctx)
    assert Groth16.verify_proving_key(circ, cer.powers, after, ctx=ctx)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('name', SHAPE_NAMES)
def test_witness_map_matches_the_oracle(ctx, name, flavour):
    from circom_compat_b200 import fr_to_mont, release
    from oracle import cref as c
    circ, witness = P.shape_circuit(name)
    red = REDUCTIONS[flavour]
    cm = circ.matrices(with_c=flavour == 'libsnark')
    m, ni = circ.num_constraints, circ.num_inputs
    for k, pub in enumerate(P.public_values(ni - 1)):
        wm = fr_to_mont(witness(pub, wseed=k))
        got = red.witness_map_from_matrices(cm, ni, m, wm, ctx)
        want = (c.witness_map_libsnark(m, ni, cm.a, cm.b, cm.c, wm) if flavour == 'libsnark' else
                c.witness_map(m, ni, circ.n_vars, cm.a, cm.b, wm))
        assert got.shape == want.shape == (circ.domain_size, 4)
        diff = np.flatnonzero((got != want).any(axis=1))
        assert diff.size == 0, (k, diff[:8].tolist())
    release(cm)


def _proved(ctx, name, flavour='circom'):
    """(pk, td, cm, witnesses, proofs) of a trapdoor key of the shape: four witnesses with public inputs 0, 1, r - 1 and
    random, proved with the proof_model.EDGE_RS pairs"""
    from circom_compat_b200 import Groth16, fr_to_mont
    from proof_model import EDGE_RS, trapdoor_keys
    key = (name, flavour)
    if key not in _STATE:
        circ, witness = P.shape_circuit(name)
        pk, td, cm = trapdoor_keys(ctx, circ, REDUCTIONS[flavour], seed=0xB200 + circ.num_inputs)
        ws = [witness(pub, wseed=k) for k, pub in enumerate(P.public_values(circ.num_inputs - 1))]
        proofs = Groth16.create_proofs(pk, EDGE_RS, cm, [fr_to_mont(w) for w in ws], ctx, REDUCTIONS[flavour])
        _STATE[key] = (pk, td, cm, ws, proofs)
    return _STATE[key]


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('name', SHAPE_NAMES)
def test_proofs_match_the_cpu_references(ctx, name, flavour):
    """single proofs and one create_proofs batch against the oracle's bytes (CircomReduction) or the trapdoor closed form
    with the oracle's h (LibsnarkReduction), and against the closed form without any h"""
    from circom_compat_b200 import Groth16, fr_to_mont, release
    from proof_model import EDGE_RS, expect_proofs, proof_bytes
    circ, _ = P.shape_circuit(name)
    red = REDUCTIONS[flavour]
    pk, td, cm, ws, batch = _proved(ctx, name, flavour)
    single = [Groth16.create_proof_with_reduction_and_matrices(pk, r, s, cm, circ.num_inputs, circ.num_constraints,
                                                               fr_to_mont(w), ctx, red).data for (r, s), w in zip(EDGE_RS, ws)]
    want = expect_proofs(pk, td, cm, EDGE_RS, ws, red)
    closed = proof_bytes([P.proof_dlogs(td, circ, w, r, s) for (r, s), w in zip(EDGE_RS, ws)])
    assert want == closed
    assert [k for k in range(len(ws)) if single[k] != want[k]] == []
    assert [k for k in range(len(ws)) if batch[k].data != want[k]] == []
    release(pk); release(cm)
    if flavour == 'libsnark':
        del _STATE[(name, flavour)]


SHARD_SHAPES = ['over1024', 'most', 'all_public']
SHARD_COUNTS = [2, 3, 5, 8]


@pytest.mark.gpu
@pytest.mark.parametrize('compact', [True, False], ids=['b_compact', 'no_b_compact'])
@pytest.mark.parametrize('count', SHARD_COUNTS)
@pytest.mark.parametrize('name', SHARD_SHAPES)
def test_sharded_proofs_rank_by_rank(ctx, monkeypatch, name, count, compact):
    """every rank's partial against proof_model.rank_partials, the folded proof against the oracle's and the whole proof;
    ranks whose L slice lies inside the n_public padding pair points at infinity with nonzero scalars"""
    from circom_compat_b200 import Context, Groth16, fr_to_mont, release
    from proof_model import check_partial, expect_circom, rank_partials, shard_bases, shard_scalars, witness_map_mont
    if compact:
        monkeypatch.delenv('B2G_NO_B_COMPACT', raising=False)
    else:
        monkeypatch.setenv('B2G_NO_B_COMPACT', '1')
    pk, _, cm, ws, proofs = _proved(ctx, name)
    release(pk)                                        # the rank contexts load the key under this B2G_NO_B_COMPACT
    w = ws[3]
    wm = fr_to_mont(w)
    scal = shard_scalars(wm, witness_map_mont(pk, cm, wm, CircomReduction))
    bases = shard_bases(pk)
    rows = [rank_partials(pk, bases, scal, k, count) for k in range(count)]
    rs = [(5, 7), (R - 1, 1)]
    want = expect_circom(pk, cm, rs, [w, w])
    ranks = [Context(0, k, count) for k in range(count)]
    try:
        for j, (r, s) in enumerate(rs):
            early = (r, s) if j == 0 else (None, None)
            parts = [Groth16.prove_partial(pk, cm, wm, cx, *early) for cx in ranks]
            bad = [(k, q, err) for k, part in enumerate(parts) for q, err in check_partial(part, rows[k])]
            assert not bad, ('(rank, query, error) of partials that differ from the model', j, bad)
            got = [Groth16.prove_finish(pk, np.stack(parts), r, s, cx).data for cx in ranks]
            assert [k for k, p in enumerate(got) if p != want[j]] == [], j
            whole = Groth16.create_proof_with_reduction_and_matrices(pk, r, s, cm, cm.num_instance_variables,
                                                                     cm.num_constraints, wm, ctx).data
            assert whole == want[j], j
    finally:
        for cx in ranks:
            cx.close()
        release(pk)


def _mixed(p, q):
    """A and C of proof p with B of proof q: not a proof of p's statement"""
    from circom_compat_b200 import Proof
    return Proof(p.data[:64] + q.data[64:192] + p.data[192:])


@pytest.mark.gpu
@pytest.mark.parametrize('name', SHAPE_NAMES)
def test_verifiers_on_real_keys(ctx, name):
    from circom_compat_b200 import Groth16, release
    circ, _ = P.shape_circuit(name)
    pk, _, cm, ws, proofs = _proved(ctx, name)
    npub = circ.num_inputs - 1
    pubs = [w[1:circ.num_inputs] for w in ws]
    ok = [True] * len(proofs)
    assert Groth16.verify_many(pk, pubs, proofs, ctx) == ok
    assert Groth16.verify_batch(pk, pubs, proofs, ctx)
    assert Groth16.verify_batch_locate(pk, pubs, proofs, ctx) == ok
    rer = Groth16.rerandomize_proofs(pk, proofs, random.Random(npub), ctx)
    assert all(a.data != b.data for a, b in zip(rer, proofs))
    assert Groth16.verify_many(pk, pubs, rer, ctx) == ok
    assert Groth16.verify_batch(pk, pubs, rer, ctx)
    assert Groth16.verify_batch_locate(pk, pubs, rer, ctx) == ok
    # refusals: the last input, a middle input, two inputs swapped (proof 3's inputs are random, so a swap changes them)
    wrong = []
    if npub:
        for i in sorted({npub - 1, npub // 2}):
            v = list(pubs[3]); v[i] = (v[i] + 1) % R
            wrong.append(v)
    if npub >= 2:
        v = list(pubs[3]); v[0], v[npub - 1] = v[npub - 1], v[0]
        wrong.append(v)
    for v in wrong:
        bad_pubs = pubs[:3] + [v]
        assert Groth16.verify_many(pk, bad_pubs, proofs, ctx) == [True, True, True, False]
        assert not Groth16.verify_batch(pk, bad_pubs, proofs, ctx)
        assert Groth16.verify_batch_locate(pk, bad_pubs, proofs, ctx) == [True, True, True, False]
    # 70 proofs, proof 66 wrong: its last input changed, or (no inputs) its B taken from another proof
    pubs70, proofs70 = [pubs[j % 4] for j in range(70)], [proofs[j % 4] for j in range(70)]
    if npub:
        pubs70[66] = list(pubs70[66]); pubs70[66][-1] = (pubs70[66][-1] + 1) % R
    else:
        proofs70[66] = _mixed(proofs[2], proofs[3])
    assert Groth16.verify_batch_locate(pk, pubs70, proofs70, ctx) == [j != 66 for j in range(70)]
    assert not Groth16.verify_batch(pk, pubs70, proofs70, ctx)
    if name == 'p256':
        from circom_compat_b200 import ethereum as eth
        blobs = [eth.serialize_compressed(eth.Proof.from_proof(p)) for p in proofs]
        assert Groth16.verify_many_compressed(pk, pubs, blobs, ctx) == ok
        assert Groth16.verify_batch_compressed(pk, pubs, blobs, ctx)
        assert Groth16.verify_batch_locate_compressed(pk, pubs, blobs, ctx) == ok
        assert Groth16.verify_many_compressed(pk, pubs[:3] + [wrong[0]], blobs, ctx) == [True, True, True, False]
    # the pure-Python pairing on one proof
    def g1(a): return o._g1_from(np.ascontiguousarray(a).tobytes())
    def g2(a): return o._g2_from(np.ascontiguousarray(a).tobytes())
    z = o.ZKey()
    z.alpha_g1, z.beta_g2, z.gamma_g2, z.delta_g2 = g1(pk.alpha_g1), g2(pk.beta_g2), g2(pk.gamma_g2), g2(pk.delta_g2)
    z.ic = [g1(x) for x in pk.gamma_abc_g1]
    p = proofs[3]
    assert o.verify(z, pubs[3], (p.a, p.b, p.c))
    release(pk); release(cm)


@pytest.mark.gpu
def test_key_batches_mix_input_counts(ctx):
    """one verify_batch_keys / verify_batch_keys_locate call over keys with n_public 256, 0 and 2048 (the largest shape): the
    segment without inputs sits between the others and shares its public-input offset with its neighbour"""
    from circom_compat_b200 import Groth16, release, release_all
    sets = {}
    for name in ('p256', 'p0', 'most'):
        pk, _, _, ws, proofs = _proved(ctx, name)
        sets[name] = (pk, [w[1:pk.n_public + 1] for w in ws], list(proofs))
    assert [sets[k][0].n_public for k in ('p256', 'p0', 'most')] == [256, 0, 2048]
    order = ['p256', 'p0', 'most', 'p0']
    batches = [sets[k] for k in order]
    assert Groth16.verify_batch_keys(batches, ctx) == [True] * 4
    assert Groth16.verify_batch_keys_locate(batches, ctx) == [[True] * 4] * 4
    pk, pubs, proofs = sets['most']
    bad_most = (pk, pubs[:2] + [pubs[2][:-1] + [(pubs[2][-1] + 1) % R]] + pubs[3:], proofs)
    pk, pubs, proofs = sets['p256']
    bad_256 = (pk, [pubs[0][:128] + [(pubs[0][128] + 1) % R] + pubs[0][129:]] + pubs[1:], proofs)
    pk, pubs, proofs = sets['p0']
    bad_0 = (pk, pubs, proofs[:1] + [_mixed(proofs[1], proofs[2])] + proofs[2:])
    batches = [bad_256, sets['p0'], bad_most, bad_0, sets['most']]
    assert Groth16.verify_batch_keys(batches, ctx) == [False, True, False, False, True]
    t = [True] * 4
    assert Groth16.verify_batch_keys_locate(batches, ctx) == [[False] + t[1:], t, t[:2] + [False, True], [True, False, True, True], t]
    release_all()


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['p0', 'p256', 'over1024', 'most', 'all_public'])
def test_keys_round_trip_through_zkey_and_ark_serialize(ctx, tmp_path, name):
    from circom_compat_b200 import deserialize_proving_key, deserialize_verifying_key, read_zkey, serialize_proving_key, \
        serialize_verifying_key
    from circom_compat_b200.keycheck import matrices_reason
    from circom_compat_b200.verifier import VerifyingKey
    circ, _ = P.shape_circuit(name)
    pk, _, _, _, _ = _proved(ctx, name)
    path = str(tmp_path / f'{name}.zkey')
    synth.write_zkey(path, pk, circ)
    zk, mats = read_zkey(path)
    _assert_same_key(zk, pk)
    assert matrices_reason(circ.matrices(), mats) is None
    for compress in (True, False):
        back = deserialize_proving_key(serialize_proving_key(pk, compress, ctx), compress, ctx)
        _assert_same_key(back, pk)
        vk = deserialize_verifying_key(serialize_verifying_key(pk, compress, ctx), compress, ctx)
        assert vk.gamma_abc_g1 == VerifyingKey.from_proving_key(pk).gamma_abc_g1
        assert len(vk.gamma_abc_g1) == circ.num_inputs
