"""The proving-key check (b2g_setup_check, Groth16.verify_proving_key): a key against its circuit and powers-of-tau ceremony.
CPU: the big-int model of tests/setup_check_model.py (the scalar side of E1-E5 equals the weighted trapdoor scalars for a
known tau, and a forged scalar breaks it), and the host comparison of a .zkey's coefficient section with its circuit on the
reference's snarkjs keys.  GPU: honest keys after 0, 1 and 2 contributions pass under both reductions, on every circuit shape
the setup's tests use; each forgery fails with the expected reason; the verdict equals the rebuild recipe's; a forgery built
for known challenges passes only with them; the error codes; the C++ mode."""
import ctypes as C
import os
import random

import numpy as np
import pytest

from circom_compat_b200 import Groth16, R1CS, R1CSFile, read_ptau, read_zkey, synth
from circom_compat_b200.keycheck import matrices_reason
from circom_compat_b200.zkey import Q_MOD, R_MOD
import setup_check_model as M
from ptau_model import write_ptau

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
FIELDS = ('alpha_g1', 'beta_g1', 'beta_g2', 'gamma_g2', 'delta_g1', 'delta_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query',
          'b_g2_query', 'l_query', 'h_query')


def _circuit(n_vars, num_inputs, rows):
    mats = []
    for x in range(3):
        r = [k for k, row in enumerate(rows) for _ in row[x]]
        c = [col for row in rows for col, _ in row[x]]
        v = [val % R_MOD for row in rows for _, val in row[x]]
        mats.append((np.array(r, dtype=np.int64), np.array(c, dtype=np.int64), v))
    return synth.Circuit(n_vars, num_inputs, len(rows), *mats)


def _edge(kind):
    """the edge circuits of the setup's tests: a column in every row, unused columns (infinity points), repeated entries,
    an empty C, every kind of coefficient, and one row that holds every column"""
    if kind == 'wire0_everywhere':
        rows = [([(0, 3), (k % 50 + 2, 1)], [(0, 5)], [(0, 7), (k % 50 + 2, k + 1)]) for k in range(254)]
        return _circuit(60, 2, rows)
    if kind == 'unused_columns':
        return _circuit(80, 2, [([(k + 2, 1)], [(k + 2, 1)], [(k + 3, 1)]) for k in range(20)])
    if kind == 'repeated_entries':
        return _circuit(6, 2, [([(2, 1), (2, 4), (3, 1)], [(2, 1), (2, R_MOD - 1), (2, 6)], [(3, 2), (3, 2)]) for _ in range(30)])
    if kind == 'coefficients':
        rng = random.Random(3)
        vals = [1, R_MOD - 1, R_MOD - 2, (R_MOD - 1) // 2, (R_MOD + 1) // 2] + [rng.randrange(R_MOD) for _ in range(5)]
        rows = [([(k % 7 + 1, vals[k % 10])], [(k % 5 + 2, vals[(k + 3) % 10])], [(k % 6 + 1, vals[(k + 7) % 10])]) for k in range(40)]
        return _circuit(9, 2, rows)
    if kind == 'one_full_row':
        full = [(j, j + 1) for j in range(300)]
        return _circuit(300, 3, [(full, [(1, 1)], full)] + [([(k + 3, 1)], [(k + 3, 1)], [(k + 4, 1)]) for k in range(40)])
    return _circuit(12, 3, [([(k % 9 + 1, 2)], [(k % 7 + 2, 3)], []) for k in range(45)])     # an empty C


EDGES = ['wire0_everywhere', 'unused_columns', 'repeated_entries', 'empty_c', 'coefficients', 'one_full_row']


def _small(kind, size):
    if kind == 'chain':
        return synth.chain_circuit(size)
    if kind == 'circomlike':
        return synth.circomlike_circuit(size)[0]
    if kind == 'tiny':
        return _circuit(2, 1, [([(1, 1)], [(1, 1)], [(1, 1)])])
    return _edge(kind)


def _r1cs(name):
    return R1CS.from_file(R1CSFile.new(open(os.path.join(GOLDEN, name), 'rb').read())).to_circuit()


# ------------------------------------------------------------------------------------------------------------------ CPU
MODEL_CASES = [('tiny', 0), ('chain', 4), ('chain', 7), ('chain', 64), ('circomlike', 3), ('circomlike', 6)] + [(k, 0) for k in EDGES[1:]]


@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('kind,size', MODEL_CASES)
def test_scalar_side_equals_the_weighted_trapdoor(kind, size, flavour):
    """sum_k s_k tau^k = sum_j rho^j (the key's scalar j) for E1-E5, with delta from two contributions"""
    circ = _small(kind, size)
    rng = random.Random(size * 7 + len(kind))
    tau, alpha, beta, delta, rho, sigma = (rng.randrange(1, R_MOD) for _ in range(6))
    for name, key, cer in M.equations(circ, tau, alpha, beta, delta, rho, sigma, flavour):
        assert key == cer, name


@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_scalar_side_with_tau_in_the_domain(flavour):
    circ = synth.chain_circuit(16)
    n = circ.domain_size
    for tau in (1, pow(synth.root_of_unity(n), 5, R_MOD), synth.root_of_unity(2 * n)):
        for name, key, cer in M.equations(circ, tau, 3, 5, 7, 11, 13, flavour):
            assert key == cer, (tau, name)


@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_a_forged_scalar_breaks_the_identity(flavour):
    circ = synth.circomlike_circuit(4)[0]
    names = {'sA': 'a_query', 'sB': 'b_g1_query', 'sC': 'gamma_abc_g1 / l_query', 'h': 'h_query'}
    for vec, first in names.items():
        for i in (0, 5):
            eqs = M.equations(circ, 123, 3, 5, 7, 11, 13, flavour, forged=(vec, i))
            broken = [name for name, key, cer in eqs if key != cer]
            assert broken and broken[0] == first, (vec, i, broken)


def _complex_circuit():
    """the circuit of the reference's complex-circuit-10000-10000 key: synth.chain_circuit restates its .r1cs (a squaring
    chain of 10 000 constraints over 10 002 wires) coefficient for coefficient"""
    return synth.chain_circuit(10002)


def test_matrices_of_the_reference_keys_match_their_circuits():
    for circ, zkey in ((_r1cs('mycircuit.r1cs'), 'test.zkey'), (_complex_circuit(), 'complex-circuit-10000-10000.zkey')):
        _, mats = read_zkey(os.path.join(GOLDEN, zkey))
        assert matrices_reason(circ.matrices(), mats) is None, zkey


def test_matrices_of_another_circuit_are_refused():
    _, mats = read_zkey(os.path.join(GOLDEN, 'test.zkey'))
    assert matrices_reason(_r1cs('circuit2.r1cs').matrices(), mats) == "the matrices' num_constraints 1 differs from the circuit's 131"


def _changed(mats, which, what):
    rowptr, col, val = (np.array(a, copy=True) for a in getattr(mats, which))
    if what == 'value':
        val[-1, 0] ^= 1
    elif what == 'column':
        col[-1] = (col[-1] + 1) % mats.n_vars
    else:                                                   # the last nonzero moved to row 0
        rowptr[1:] += 1
        rowptr[-1] -= 1
        order = np.r_[len(col) - 1, np.arange(len(col) - 1)]
        col, val = col[order], val[order]
    out = type(mats)(**{k: getattr(mats, k) for k in ('num_instance_variables', 'num_witness_variables', 'num_constraints',
                                                        'a_num_non_zero', 'b_num_non_zero', 'c_num_non_zero', 'a', 'b')})
    setattr(out, which, (rowptr, col, val))
    return out


@pytest.mark.parametrize('which', ['a', 'b'])
@pytest.mark.parametrize('what', ['value', 'column', 'row'])
def test_one_changed_coefficient_is_refused(which, what):
    circ = _complex_circuit().matrices()
    _, mats = read_zkey(os.path.join(GOLDEN, 'complex-circuit-10000-10000.zkey'))
    got = matrices_reason(circ, _changed(mats, which, what))
    last_row = int(np.searchsorted(getattr(mats, which)[0], len(getattr(mats, which)[1]) - 1, side='right')) - 1
    assert got == f"matrix {which.upper()} differs from the circuit at row {0 if what == 'row' else last_row}"


def test_canonical_rows_sum_duplicates_and_drop_zeros():
    a = _circuit(5, 1, [([(3, 1), (2, 4), (3, R_MOD - 1)], [(1, 1)], [])])
    b = _circuit(5, 1, [([(2, 4)], [(1, 1)], [])])
    assert matrices_reason(a.matrices(), b.matrices()) is None
    c = _circuit(5, 1, [([(2, 2), (2, 2)], [(1, 1)], [])])
    assert matrices_reason(a.matrices(), c.matrices()) is None


def test_python_entry_refuses_bad_shapes_before_the_library():
    from circom_compat_b200 import LibsnarkReduction
    circ = synth.chain_circuit(16)
    pk = _fake_key(circ, 16)
    short = dict(pk.__dict__); short['h_query'] = pk.h_query[:15]
    from circom_compat_b200 import ProvingKey
    fields = {k: v for k, v in short.items() if k != '_device'}
    r = Groth16.verify_proving_key(circ, None, ProvingKey(**fields))
    assert not r and r.reason == "h_query holds 15 points; a CircomReduction domain of 16 needs 16"
    r = Groth16.verify_proving_key(circ, None, pk, reduction=LibsnarkReduction)
    assert r.reason == "h_query holds 16 points; a LibsnarkReduction domain of 16 needs 15"
    fields['h_query'] = pk.h_query; fields['l_query'] = pk.l_query[1:]
    assert Groth16.verify_proving_key(circ, None, ProvingKey(**fields)).reason == "l_query holds 13 points; the circuit needs 14"
    _, mats = read_zkey(os.path.join(GOLDEN, 'test.zkey'))
    assert Groth16.verify_proving_key(circ, None, pk, mats).reason.startswith("the matrices' ")


def _fake_key(circ, nh):
    from circom_compat_b200 import ProvingKey
    z = lambda k, w: np.zeros((k, w), dtype=np.uint64)
    nv, ni = circ.n_vars, circ.num_inputs
    return ProvingKey(nv, ni - 1, nh, z(1, 8), z(1, 8), z(1, 16), z(1, 16), z(1, 8), z(1, 16), z(ni, 8), z(nv, 8), z(nv, 8),
                      z(nv, 16), z(nv - ni, 8), z(nh, 8))


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope='module')
def gpu():
    from circom_compat_b200 import Context, release_all
    c = Context(0)
    yield c
    release_all()
    c.close()


def _limbs(vals):
    return synth._ints_to_limbs([v % R_MOD for v in vals])


class Ceremony:
    """the points of a ceremony of size 2^power for (tau, alpha, beta) on g1 = k1 G1, g2 = k2 G2, by fixed-base products"""

    def __init__(self, ctx, power, tau, alpha, beta, k1=1, k2=1):
        self.power = self.ceremony_power = power
        n = 1 << power
        t = [1] * (2 * n - 1)
        for i in range(1, 2 * n - 1):
            t[i] = t[i - 1] * tau % R_MOD
        self.tau_g1 = ctx.fixed_base_g1(_limbs([k1 * v for v in t]))
        self.tau_g2 = ctx.fixed_base_g2(_limbs([k2 * v for v in t[:n]]))
        self.alpha_tau_g1 = ctx.fixed_base_g1(_limbs([k1 * alpha * v for v in t[:n]]))
        self.beta_tau_g1 = ctx.fixed_base_g1(_limbs([k1 * beta * v for v in t[:n]]))
        self.beta_g2 = ctx.fixed_base_g2(_limbs([k2 * beta]))


_CEREMONIES = {}


def _ceremony(ctx, power, seed=7, k1=1, k2=1, tau=None):
    key = (power, seed, k1, k2, tau)
    if key not in _CEREMONIES:
        rng = random.Random(seed)
        t, a, b = (rng.randrange(1, R_MOD) for _ in range(3))
        _CEREMONIES[key] = Ceremony(ctx, power, tau if tau is not None else t, a, b, k1, k2)
    return _CEREMONIES[key]


def _reduction(flavour):
    from circom_compat_b200 import CircomReduction, LibsnarkReduction
    return LibsnarkReduction if flavour == 'libsnark' else CircomReduction


def _key(ctx, circ, cer, flavour, contributions=1, seed=1):
    pk = Groth16.generate_parameters_from_powers_of_tau(circ, cer, ctx, _reduction(flavour))
    rng = random.Random(seed)
    for _ in range(contributions):
        pk = Groth16.contribute(pk, rng, ctx)
    return pk


def _recipe(ctx, circ, cer, pk, flavour):
    """the rebuild recipe: the key from the ceremony, the fields a contribution leaves alone compared, then the delta check"""
    from circom_compat_b200 import B2gError
    try:
        rebuilt = Groth16.generate_parameters_from_powers_of_tau(circ, cer, ctx, _reduction(flavour))
    except B2gError:
        return False
    for name in ('alpha_g1', 'beta_g1', 'beta_g2', 'gamma_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query', 'b_g2_query'):
        a, b = np.ascontiguousarray(getattr(rebuilt, name)), np.ascontiguousarray(getattr(pk, name))
        if a.shape != b.shape or a.tobytes() != b.tobytes():
            return False
    return Groth16.verify_contribution(rebuilt, pk, ctx)


def _check(ctx, circ, cer, pk, flavour, **kw):
    return Groth16.verify_proving_key(circ, cer, pk, reduction=_reduction(flavour), ctx=ctx, **kw)


def _with(pk, **fields):
    from circom_compat_b200 import ProvingKey
    arrs = {k: np.array(getattr(pk, k), copy=True) for k in FIELDS}
    arrs.update(fields)
    return ProvingKey(pk.n_vars, pk.n_public, pk.domain_size, *(arrs[k] for k in FIELDS))


SIZES = [('tiny', 0), ('chain', 4), ('chain', 7), ('chain', 256), ('chain', 511), ('circomlike', 2), ('circomlike', 6),
         ('circomlike', 12)] + [(k, 0) for k in EDGES]


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('kind,size', SIZES)
def test_honest_keys_pass(gpu, kind, size, flavour):
    """domains 2 to 2^12 from one 2^12 ceremony, after 0, 1 and 2 contributions; the rebuild recipe agrees"""
    circ, cer = _small(kind, size), _ceremony(gpu, 12)
    for k in (0, 1, 2):
        pk = _key(gpu, circ, cer, flavour, k)
        r = _check(gpu, circ, cer, pk, flavour)
        assert r and r.reason is None, (k, r.reason)
    assert _recipe(gpu, circ, cer, pk, flavour)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('name', ['mycircuit.r1cs', 'circuit2.r1cs'])
def test_honest_keys_of_the_reference_circuits_pass(gpu, name, flavour):
    circ, cer = _r1cs(name), _ceremony(gpu, 12)
    assert _check(gpu, circ, cer, _key(gpu, circ, cer, flavour, 1), flavour)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_honest_keys_at_2_16_and_2_18(gpu, flavour):
    circ, cer = synth.circomlike_circuit(16)[0], _ceremony(gpu, 16)
    pk = _key(gpu, circ, cer, flavour, 1)
    assert _check(gpu, circ, cer, pk, flavour)
    assert _recipe(gpu, circ, cer, pk, flavour)
    if flavour == 'circom':
        circ, cer = synth.chain_circuit(1 << 18), _ceremony(gpu, 18)
        assert _check(gpu, circ, cer, _key(gpu, circ, cer, flavour, 2), flavour)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_other_generators_and_tau_in_the_domain(gpu, flavour):
    circ = synth.circomlike_circuit(8)[0]
    cer = _ceremony(gpu, 8, seed=8, k1=7, k2=5)
    assert _check(gpu, circ, cer, _key(gpu, circ, cer, flavour, 1), flavour)
    circ = synth.chain_circuit(64)
    for tau in (pow(synth.root_of_unity(64), 5, R_MOD), synth.root_of_unity(128)):
        cer = _ceremony(gpu, 7, tau=tau)
        pk = _key(gpu, circ, cer, flavour, 1)
        assert _check(gpu, circ, cer, pk, flavour), tau
        assert _recipe(gpu, circ, cer, pk, flavour)


@pytest.mark.gpu
def test_a_zkey_and_a_memory_mapped_ptau(gpu, tmp_path):
    """synth.write_zkey -> read_zkey with its matrices, against a memory-mapped .ptau of 2^10 for a 2^8 circuit"""
    circ, cer = synth.circomlike_circuit(8)[0], _ceremony(gpu, 10)
    path = tmp_path / 'pot10.ptau'
    path.write_bytes(write_ptau(10, cer.tau_g1, cer.tau_g2, cer.alpha_tau_g1, cer.beta_tau_g1, cer.beta_g2))
    pw = read_ptau(str(path))
    pk = _key(gpu, circ, cer, 'circom', 2)
    synth.write_zkey(str(tmp_path / 'c.zkey'), pk, circ)
    zk, mats = read_zkey(str(tmp_path / 'c.zkey'))
    r = Groth16.verify_proving_key(circ, pw, zk, mats, ctx=gpu)
    assert r, r.reason
    other = synth.circomlike_circuit(8, seed=5)[0]
    assert Groth16.verify_proving_key(other, pw, zk, mats, ctx=gpu).reason.startswith("matrix A differs from the circuit at row")


def _g2_outside_subgroup():
    from batch_model import twist_point_outside_g2
    (x0, x1), (y0, y1) = twist_point_outside_g2(random.Random(5))
    return synth._ints_to_limbs([v * (1 << 256) % Q_MOD for v in (x0, x1, y0, y1)]).reshape(16)


def _neg_g2(p):
    q = np.array(p, copy=True)
    ys = synth._ints_to_limbs([(Q_MOD - int.from_bytes(q[8 + 4 * k:12 + 4 * k].tobytes(), 'little')) % Q_MOD for k in range(2)])
    q[8:] = ys.reshape(8)
    return q


def _used(points, count=1):
    """the first `count` indices of points that are not at infinity (an unused column's points are)"""
    return [int(i) for i in np.flatnonzero(np.asarray(points).any(axis=1))[:count]]


def _forgeries(ctx, circ, cer, pk, flavour):
    """(name, key, ceremony, reason) for an honest key pk of circ on cer (one contribution)"""
    out = []
    a = np.array(pk.a_query, copy=True)
    i, j = _used(a, 2)
    a[[i, j]] = a[[j, i]]
    out.append(('a_query swapped', _with(pk, a_query=a), cer, 'a_query does not match the circuit and ceremony'))
    b = np.array(pk.b_g1_query, copy=True)
    i, = _used(b)
    b[i] = ctx.test_op(10, b[i])[0]
    out.append(('b_g1_query doubled', _with(pk, b_g1_query=b), cer, 'b_g1_query does not match the circuit and ceremony'))
    b2 = np.array(pk.b_g2_query, copy=True)
    i, = _used(b2)
    b2[i] = _neg_g2(b2[i])
    out.append(('b_g2_query negated', _with(pk, b_g2_query=b2), cer, 'b_g2_query does not match the circuit and ceremony'))
    ic = np.array(pk.gamma_abc_g1, copy=True); ic[1] = pk.a_query[5]
    e4 = 'gamma_abc_g1 / l_query do not match the circuit and ceremony'
    out.append(('IC changed', _with(pk, gamma_abc_g1=ic), cer, e4))
    x = Groth16.contribute(pk, x=12345, ctx=ctx)
    y = Groth16.contribute(pk, x=54321, ctx=ctx)
    out.append(('delta multiplied, L kept', _with(x, l_query=pk.l_query), cer, e4))
    out.append(('H of another x', _with(x, h_query=y.h_query), cer, 'h_query does not match the circuit and ceremony'))
    out.append(('delta_g1 of another x', _with(x, delta_g1=y.delta_g1), cer, 'delta_g1 and delta_g2 disagree'))
    other = _ceremony(ctx, cer.power, seed=99)
    out.append(('another ceremony', _key(ctx, circ, other, flavour, 1), cer, "alpha_g1 is not the ceremony's"))
    rnd = Groth16.generate_random_parameters_with_reduction(circ, random.Random(4), ctx, _reduction(flavour))
    out.append(('random parameters', rnd, cer, "alpha_g1 is not the ceremony's"))
    changed = synth.Circuit(circ.n_vars, circ.num_inputs, circ.num_constraints,
                            (circ.A[0], circ.A[1], [(v + 1) % R_MOD if k == 2 else v for k, v in enumerate(circ.A[2])]), circ.B, circ.C)
    out.append(('one coefficient changed', _key(ctx, changed, cer, flavour, 1), cer, 'a_query does not match the circuit and ceremony'))
    for name, src in (('alpha_g1', 'beta_g1'), ('beta_g1', 'alpha_g1'), ('beta_g2', 'gamma_g2'), ('gamma_g2', 'beta_g2')):
        out.append((f'{name} replaced', _with(pk, **{name: np.array(getattr(pk, src), copy=True)}), cer, f"{name} is not the ceremony's"))
    l = np.array(pk.l_query, copy=True); l[17, 4] ^= 1
    out.append(('l_query off the curve', _with(pk, l_query=l), cer, 'l_query[17]: off the curve'))
    a = np.array(pk.a_query, copy=True); a[3, 3] = (1 << 64) - 1
    out.append(('a_query coordinate >= p', _with(pk, a_query=a), cer, 'a_query[3]: a coordinate >= p'))
    b2 = np.array(pk.b_g2_query, copy=True); b2[2] = _g2_outside_subgroup()
    out.append(('b_g2_query outside G2', _with(pk, b_g2_query=b2), cer, 'b_g2_query[2]: not in G2'))
    u = np.array(cer.tau_g2, copy=True); u[3] = _g2_outside_subgroup()
    bad = Ceremony.__new__(Ceremony); bad.__dict__.update(cer.__dict__); bad.tau_g2 = u
    out.append(('tau_g2 outside G2', pk, bad, 'tau_g2[3]: not in G2'))
    t = np.array(cer.tau_g1, copy=True); t[40, 4] ^= 1
    bad = Ceremony.__new__(Ceremony); bad.__dict__.update(cer.__dict__); bad.tau_g1 = t
    out.append(('tau_g1 off the curve', pk, bad, 'tau_g1[40]: off the curve'))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_forgeries_fail_with_their_reason_and_the_recipes_verdict(gpu, flavour):
    circ, cer = synth.circomlike_circuit(6)[0], _ceremony(gpu, 6)
    pk = _key(gpu, circ, cer, flavour, 1)
    for name, key, c, reason in _forgeries(gpu, circ, cer, pk, flavour):
        r = _check(gpu, circ, c, key, flavour)
        assert not r and r.reason == reason, (name, r.reason)
        assert not _recipe(gpu, circ, c, key, flavour), name


@pytest.mark.gpu
def test_a_forgery_for_known_challenges(gpu):
    """a_query[0] += rho X, a_query[1] -= X keeps sum rho^j a_j: it passes with rho and fails with fresh challenges"""
    circ, cer = synth.chain_circuit(64), _ceremony(gpu, 7)
    pk = _key(gpu, circ, cer, 'circom', 1)
    rho, sigma, x = 1234567, 7654321, 99
    d = gpu.fixed_base_g1(_limbs([rho * x, R_MOD - x]))
    a = np.array(pk.a_query, copy=True)
    a[0] = gpu.test_op(8, a[0], d[0])[0]
    a[1] = gpu.test_op(8, a[1], d[1])[0]
    forged = _with(pk, a_query=a)
    assert _check(gpu, circ, cer, forged, 'circom', challenges=[rho, sigma])
    assert _check(gpu, circ, cer, forged, 'circom').reason == 'a_query does not match the circuit and ceremony'
    assert not _recipe(gpu, circ, cer, forged, 'circom')


@pytest.mark.gpu
def test_the_streamed_msm_over_infinity_bases(gpu):
    """all-zero bases, and bases with runs of infinity, as an unused column's key points are"""
    for g2 in (False, True):
        w = 16 if g2 else 8
        assert not gpu.powers_msm(np.zeros((1000, w), dtype=np.uint64), 12345, g2=g2).any()
        fb = gpu.fixed_base_g2 if g2 else gpu.fixed_base_g1
        pts = fb(_limbs(range(1, 301)))
        pts[100:250] = 0
        k = [pow(777, i, R_MOD) if not 100 <= i < 250 else 0 for i in range(300)]
        want = (gpu.msm_g2 if g2 else gpu.msm_g1)(pts, _limbs(k))
        assert gpu.powers_msm(pts, 777, g2=g2).tobytes() == want.tobytes()


def _raw(ctx, circ, cer, pk, ch, null=None, log_size=None):
    from circom_compat_b200 import _native as N
    from circom_compat_b200.groth16 import _circuit_desc, _powers_desc
    from circom_compat_b200.keycheck import KEY_FIELDS
    d, keep, nv, ni, size, nh = _circuit_desc(circ, _reduction('circom'))
    pd, arrays = _powers_desc(cer, size)
    if log_size is not None:
        pd.log_size = log_size
    arrs = {k: np.ascontiguousarray(getattr(pk, k)) for k in KEY_FIELDS}
    kd = N.KeyDesc()
    kd.n_vars, kd.n_ic, kd.n_l, kd.n_h = nv, ni, nv - ni, nh
    for k, a in arrs.items():
        setattr(kd, k, None if k == null else a.ctypes.data)
    cb = np.frombuffer(b''.join(int(v).to_bytes(32, 'little') for v in ch), dtype=np.uint8).copy()
    rep = N.SetupReport()
    return N.lib().b2g_setup_check(ctx._h, C.byref(d), C.byref(pd), C.byref(kd), cb.ctypes.data, C.byref(rep)), rep


@pytest.mark.gpu
def test_errors_leave_the_context_usable(gpu):
    from circom_compat_b200 import _native as N
    circ, cer = synth.chain_circuit(64), _ceremony(gpu, 7)
    pk = _key(gpu, circ, cer, 'circom', 1)

    def still_usable():
        rc, rep = _raw(gpu, circ, cer, pk, [5, 6])
        assert rc == N.B2G_OK and rep.ok == 1 and rep.rule == 0

    still_usable()
    cases = [('rho 0', dict(ch=[0, 6]), N.B2G_E_INPUT), ('sigma r', dict(ch=[5, R_MOD]), N.B2G_E_INPUT),
             ('rho 2^256 - 1', dict(ch=[(1 << 256) - 1, 6]), N.B2G_E_INPUT),
             ('null l_query', dict(ch=[5, 6], null='l_query'), N.B2G_E_SHAPE),
             ('a ceremony too small', dict(ch=[5, 6], log_size=5), N.B2G_E_DOMAIN),
             ('log_size 29', dict(ch=[5, 6], log_size=29), N.B2G_E_DOMAIN)]
    for name, kw, code in cases:
        rc, _ = _raw(gpu, circ, cer, pk, **kw)
        assert rc == code, (name, rc, N.lib().b2g_last_error())
        still_usable()
    assert N.lib().b2g_setup_check(gpu._h, None, None, None, None, None) == N.B2G_E_SHAPE
    assert N.lib().b2g_setup_check(None, None, None, None, None, None) == N.B2G_E_SHAPE
    with pytest.raises(N.PolynomialDegreeTooLarge):
        Groth16.verify_proving_key(synth.chain_circuit(512), cer, _key(gpu, synth.chain_circuit(512), _ceremony(gpu, 9), 'circom', 0),
                                   ctx=gpu)
    with pytest.raises(ValueError, match='two challenges'):
        Groth16.verify_proving_key(circ, cer, pk, ctx=gpu, challenges=[1])
    still_usable()


@pytest.mark.gpu
def test_a_pending_proof_is_refused(gpu):
    from circom_compat_b200 import fr_to_mont, _native as N
    circ, cer = synth.chain_circuit(64), _ceremony(gpu, 7)
    pk = _key(gpu, circ, cer, 'circom', 1)
    w = synth.chain_witness(64)
    pending = Groth16.submit(pk, 5, 7, circ.matrices(), fr_to_mont(w), gpu)
    with pytest.raises(N.B2gError, match='pending'):
        Groth16.verify_proving_key(circ, cer, pk, ctx=gpu)
    assert Groth16.verify(pk, w[1:circ.num_inputs], pending.wait())
    assert Groth16.verify_proving_key(circ, cer, pk, ctx=gpu)


@pytest.mark.gpu
def test_cpp_zkey_verify_mode_matches_python(gpu, tmp_path):
    """B2G_ZKEY_VERIFY=<file.ptau> groth16_bench circuit.r1cs circuit.zkey: the verdict and the reason Python gives"""
    import subprocess
    r1cs = os.path.join(GOLDEN, 'circuit2.r1cs')
    circ, cer = _r1cs('circuit2.r1cs'), _ceremony(gpu, 9)
    ptau = tmp_path / 'pot9.ptau'
    ptau.write_bytes(write_ptau(9, cer.tau_g1, cer.tau_g2, cer.alpha_tau_g1, cer.beta_tau_g1, cer.beta_g2))
    pk = _key(gpu, circ, cer, 'circom', 1)
    b2 = np.array(pk.b_g2_query, copy=True)
    i, = _used(b2)
    b2[i] = _neg_g2(b2[i])
    l = np.array(pk.l_query, copy=True); l[17, 4] ^= 1
    exe = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench')
    for name, key in (('honest', pk), ('b_g2 negated', _with(pk, b_g2_query=b2)), ('l off the curve', _with(pk, l_query=l))):
        path = tmp_path / f'{name}.zkey'
        synth.write_zkey(str(path), key, circ)
        zk, mats = read_zkey(str(path))
        want = Groth16.verify_proving_key(circ, read_ptau(str(ptau)), zk, mats, ctx=gpu)
        out = subprocess.check_output([exe, r1cs, str(path)], text=True, env=dict(os.environ, B2G_ZKEY_VERIFY=str(ptau)))
        line = [x for x in out.splitlines() if x.startswith('key=')][0]
        assert line == ('key=1' if want else f'key=0 {want.reason}'), (name, out)
        assert float(dict(x.split('=', 1) for x in out.splitlines() if x.startswith('ms='))['ms']) > 0
