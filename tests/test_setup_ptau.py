"""Setup from a powers-of-tau ceremony and delta contributions (b2g_setup_from_powers, b2g_delta_update,
b2g_delta_update_check, b2g_points_intt; ptau.read_ptau; Groth16.generate_parameters_from_powers_of_tau, contribute,
verify_contribution).  CPU: the .ptau reader against the test writer and the folded H query against synth.h_query_scalars.
GPU: ceremonies synthesised from seeded (tau, alpha, beta) with fixed-base products; every key byte for byte against
b2g_setup(alpha, beta, 1, delta, tau) on the ceremony's generators."""
import ctypes as C
import os
import random

import numpy as np
import pytest

from circom_compat_b200 import read_ptau, synth
from circom_compat_b200.zkey import Q_MOD, R_MOD
import ptau_model as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
KEY_FIELDS = ('alpha_g1', 'beta_g1', 'beta_g2', 'gamma_g2', 'delta_g1', 'delta_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query',
              'b_g2_query', 'l_query', 'h_query')


def _rows(power, seed=1):
    """pseudo-random point rows of the right shapes (the reader does not look inside points)"""
    rng = np.random.default_rng(seed)
    n = 1 << power
    return [rng.integers(0, 1 << 63, size=s, dtype=np.uint64) for s in ((2 * n - 1, 8), (n, 16), (n, 8), (n, 8), (1, 16))]


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize('power', [1, 3, 6])
def test_read_ptau_round_trip(tmp_path, power):
    rows = _rows(power, power)
    data = P.write_ptau(power, *rows, ceremony_power=power + 2)
    path = tmp_path / 'pot.ptau'
    path.write_bytes(data)
    for src in (data, str(path), path):
        pw = read_ptau(src)
        assert (pw.power, pw.ceremony_power) == (power, power + 2)
        for got, want in zip((pw.tau_g1, pw.tau_g2, pw.alpha_tau_g1, pw.beta_tau_g1, pw.beta_g2), rows):
            assert got.shape == want.shape and got.tobytes() == want.tobytes()


def test_read_ptau_skips_other_sections_and_is_zero_copy(tmp_path):
    """sections in another order with extra ones (the Lagrange sections 12-15 are not read); the views share the file's map"""
    rows = _rows(2, 9)
    secs = [P.section(12, b'\x01' * 40), P.header(2)] + [P.section(2 + k, r.tobytes()) for k, r in enumerate(rows)][::-1]
    pw = read_ptau(P.container(secs + [P.section(7, b'')]))
    assert pw.tau_g1.tobytes() == rows[0].tobytes() and pw.beta_g2.tobytes() == rows[4].tobytes()
    path = tmp_path / 'pot.ptau'
    path.write_bytes(P.write_ptau(2, *rows))
    pw = read_ptau(str(path))
    assert isinstance(pw.tau_g1.base, np.ndarray) or pw.tau_g1.base is not None
    assert not pw.tau_g1.flags.writeable and not pw.tau_g1.flags.owndata


def _refusals():
    rows = _rows(2, 3)
    good = [P.header(2)] + [P.section(2 + k, r.tobytes()) for k, r in enumerate(rows)]
    full = P.container(good)
    return [
        ('magic', P.container(good, magic=b'zkey'), 'magic'),
        ('version', P.container(good, version=2), 'version'),
        ('empty', b'', 'magic'),
        ('field', P.container([P.header(2, q=R_MOD)] + good[1:]), 'field'),
        ('n8', P.container([P.header(2, n8=48, q=Q_MOD)] + good[1:]), 'field element size'),
        ('missing', P.container(good[:3] + good[4:]), 'section 4 is missing'),
        ('missing header', P.container(good[1:]), 'section 1 is missing'),
        ('truncated', full[:-10], 'truncated'),
        ('truncated header', full[:14], 'truncated'),
        ('size vs power', P.container([P.header(3)] + good[1:]), 'power 3 needs'),
        ('short section', P.container(good[:2] + [P.section(3, rows[1][:-1].tobytes())] + good[3:]), 'section 3 holds'),
        ('power 0', P.container([P.header(0)] + good[1:]), 'out of range'),
        ('section 1 size', P.container([P.section(1, P.header(2)[12:] + b'\0\0\0\0')] + good[1:]), 'section 1 holds 48 bytes'),
    ]


@pytest.mark.parametrize('name,data,msg', _refusals(), ids=[r[0] for r in _refusals()])
def test_read_ptau_refusals(name, data, msg):
    with pytest.raises(ValueError, match=msg):
        read_ptau(data)


def test_a_file_of_power_p_serves_every_smaller_domain(tmp_path):
    """the prefix for a domain of 2^k <= 2^p points equals the arrays of a ceremony of power k made from the same powers,
    as views of the file or as copies in host memory; a larger domain or a short array is refused"""
    p = 6
    rows = _rows(p, 4)
    path = tmp_path / 'pot6.ptau'
    path.write_bytes(P.write_ptau(p, *rows))
    pw = read_ptau(str(path))
    for k in range(1, p + 1):
        n = 1 << k
        small = read_ptau(P.write_ptau(k, rows[0][:2 * n - 1], rows[1][:n], rows[2][:n], rows[3][:n], rows[4]))
        for copy in (False, True):
            got = pw.prefix(k, copy=copy)
            for name in ('tau_g1', 'tau_g2', 'alpha_tau_g1', 'beta_tau_g1', 'beta_g2'):
                a, b = getattr(got, name), getattr(small, name)
                assert a.shape == b.shape and a.tobytes() == b.tobytes(), (k, name)
                assert np.shares_memory(a, pw.tau_g1) == (not copy and name == 'tau_g1'), (k, name)
    assert pw.prefix(0).tau_g1.shape == (1, 8)
    with pytest.raises(ValueError, match='exceeds'):
        pw.prefix(p + 1)
    short = pw.prefix(3)
    short.power = 4                       # arrays shorter than the power claims
    with pytest.raises(ValueError, match='tau_g1 holds 15 rows'):
        short.prefix(4)


@pytest.mark.parametrize('n', [1, 2, 4, 8, 16, 64])
def test_folded_circom_h_matches_synth(n):
    tau = random.Random(n).randrange(1, R_MOD)
    assert P.folded_circom_h(n, tau) == synth.h_query_scalars(n, tau, 1)


@pytest.mark.parametrize('n', [2, 8])
def test_folded_circom_h_with_tau_in_the_domain(n):
    """tau a 2n-th root of unity (synth's closed form divides by zero there): the odd entries of the 2n-point transform"""
    w = synth.root_of_unity(2 * n)
    for k in (0, 1, 3, n):
        tau = pow(w, k, R_MOD)
        full = P.intt([pow(tau, i, R_MOD) for i in range(2 * n - 1)] + [0])
        assert P.folded_circom_h(n, tau) == full[1::2]


def test_model_intt_inverts_the_lagrange_basis():
    n, tau = 16, 12345
    assert P.intt([pow(tau, i, R_MOD) for i in range(n)]) == synth.lagrange_at(n, tau)


def test_groth16_bench_still_compiles():
    import subprocess
    src = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench.cpp')
    subprocess.check_call(['/usr/bin/g++', '-std=c++17', '-Wall', '-Werror', '-fsyntax-only', src])


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
    """the points of a ceremony of size 2^power for (tau, alpha, beta) on g1 = k1 G1, g2 = k2 G2, made by fixed-base products"""

    def __init__(self, ctx, power, tau, alpha, beta, k1=1, k2=1):
        self.power, self.tau, self.alpha, self.beta, self.k1, self.k2 = power, tau, alpha, beta, k1, k2
        n = 1 << power
        t = [1] * (2 * n - 1)
        for i in range(1, 2 * n - 1):
            t[i] = t[i - 1] * tau % R_MOD
        self.tau_g1 = ctx.fixed_base_g1(_limbs([k1 * v for v in t]))
        self.tau_g2 = ctx.fixed_base_g2(_limbs([k2 * v for v in t[:n]]))
        self.alpha_tau_g1 = ctx.fixed_base_g1(_limbs([k1 * alpha * v for v in t[:n]]))
        self.beta_tau_g1 = ctx.fixed_base_g1(_limbs([k1 * beta * v for v in t[:n]]))
        self.beta_g2 = ctx.fixed_base_g2(_limbs([k2 * beta]))

    def generators(self):
        return (None, None) if self.k1 == self.k2 == 1 else (self.tau_g1[0], self.tau_g2[0])


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


def _assert_same_key(pk, ref):
    for name in KEY_FIELDS:
        a, b = np.ascontiguousarray(getattr(pk, name)), np.ascontiguousarray(getattr(ref, name))
        assert a.shape == b.shape and a.tobytes() == b.tobytes(), name
    assert (pk.n_vars, pk.n_public, pk.domain_size) == (ref.n_vars, ref.n_public, ref.domain_size)


def _reference_key(ctx, circ, cer, flavour, delta=1):
    from circom_compat_b200 import Groth16
    g1, g2 = cer.generators()
    return Groth16.generate_parameters_with_qap(circ, cer.alpha, cer.beta, 1, delta, g1, g2, tau=cer.tau, ctx=ctx,
                                                reduction=_reduction(flavour))


def _check(ctx, circ, cer, flavour):
    from circom_compat_b200 import Groth16
    pk = Groth16.generate_parameters_from_powers_of_tau(circ, cer, ctx, _reduction(flavour))
    _assert_same_key(pk, _reference_key(ctx, circ, cer, flavour))
    return pk


@pytest.mark.gpu
@pytest.mark.parametrize('g2', [False, True])
def test_points_intt_matches_fixed_base_of_the_scalar_intt(gpu, g2):
    rng = random.Random(11 + g2)
    fb = gpu.fixed_base_g2 if g2 else gpu.fixed_base_g1
    for log_n in range(1, 13):
        n = 1 << log_n
        cases = [[rng.randrange(R_MOD) for _ in range(n)], [rng.randrange(R_MOD)] * n]
        a, b = rng.randrange(R_MOD), rng.randrange(R_MOD)
        cases.append([a if i % 2 else b for i in range(n)])
        cases.append([a if i < n // 2 else R_MOD - a for i in range(n)])
        if log_n > 4 and g2:
            cases = cases[1:]                       # the random G2 vectors above 2^4 points add time, not coverage
        for v in cases:
            got = gpu.points_intt(fb(_limbs(v)), g2=g2)
            assert got.tobytes() == fb(_limbs(P.intt(v))).tobytes(), (log_n, v[:2])


SIZES = [('tiny', 0)] + [('chain', 1 << k) for k in (2, 3, 5, 8, 12)] + [('chain', (1 << k) - 1) for k in (3, 9, 12)] + \
        [('circomlike', k) for k in (2, 3, 6, 10, 12)]


def _circuit_of(kind, size):
    if kind == 'chain':
        return synth.chain_circuit(size)
    if kind == 'circomlike':
        return synth.circomlike_circuit(size)[0]
    return _circuit(2, 1, [([(1, 1)], [(1, 1)], [(1, 1)])])


def _circuit(n_vars, num_inputs, rows):
    mats = []
    for x in range(3):
        r = [k for k, row in enumerate(rows) for _ in row[x]]
        c = [col for row in rows for col, _ in row[x]]
        v = [val % R_MOD for row in rows for _, val in row[x]]
        mats.append((np.array(r, dtype=np.int64), np.array(c, dtype=np.int64), v))
    return synth.Circuit(n_vars, num_inputs, len(rows), *mats)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('kind,size', SIZES)
def test_setup_from_powers_matches_b2g_setup(gpu, kind, size, flavour):
    """domains 2 to 2^12 from one 2^12 ceremony: larger than most of these circuits need"""
    _check(gpu, _circuit_of(kind, size), _ceremony(gpu, 12), flavour)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_setup_from_powers_at_2_16_and_2_18(gpu, flavour):
    _check(gpu, synth.circomlike_circuit(16)[0], _ceremony(gpu, 16), flavour)
    if flavour == 'circom':
        _check(gpu, synth.chain_circuit(1 << 18), _ceremony(gpu, 18), flavour)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('name', ['mycircuit.r1cs', 'circuit2.r1cs'])
def test_setup_from_powers_on_reference_circuits(gpu, name, flavour):
    from circom_compat_b200 import R1CS, R1CSFile
    circ = R1CS.from_file(R1CSFile.new(open(os.path.join(GOLDEN, name), 'rb').read())).to_circuit()
    _check(gpu, circ, _ceremony(gpu, 12), flavour)


def _edge(kind):
    if kind == 'wire0_everywhere':
        m = (1 << 12) - 2
        rows = [([(0, 3), (k % 50 + 2, 1)], [(0, 5)], [(0, 7), (k % 50 + 2, k + 1)]) for k in range(m)]
        return _circuit(60, 2, rows)
    if kind == 'unused_columns':
        rows = [([(k + 2, 1)], [(k + 2, 1)], [(k + 3, 1)]) for k in range(20)]
        return _circuit(80, 2, rows)
    if kind == 'repeated_entries':
        rows = [([(2, 1), (2, 4), (3, 1)], [(2, 1), (2, R_MOD - 1), (2, 6)], [(3, 2), (3, 2)]) for _ in range(30)]
        return _circuit(6, 2, rows)
    if kind == 'coefficients':                        # 1, r - 1, r - 2, (r - 1) / 2, (r + 1) / 2 and full-size values
        rng = random.Random(3)
        vals = [1, R_MOD - 1, R_MOD - 2, (R_MOD - 1) // 2, (R_MOD + 1) // 2] + [rng.randrange(R_MOD) for _ in range(5)]
        rows = [([(k % 7 + 1, vals[k % 10])], [(k % 5 + 2, vals[(k + 3) % 10])], [(k % 6 + 1, vals[(k + 7) % 10])]) for k in range(40)]
        return _circuit(9, 2, rows)
    rows = [([(k % 9 + 1, 2)], [(k % 7 + 2, 3)], []) for k in range(45)]      # an empty C
    return _circuit(12, 3, rows)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('kind', ['wire0_everywhere', 'unused_columns', 'repeated_entries', 'empty_c', 'coefficients'])
def test_setup_from_powers_edge_circuits(gpu, kind, flavour):
    _check(gpu, _edge(kind), _ceremony(gpu, 12), flavour)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_setup_from_powers_with_tau_in_the_domain(gpu, flavour):
    """tau = omega_64^5 (in the circuit's domain of 64 points) and tau = omega_128 (in the 2n domain of the H query):
    the transforms meet repeated and cancelling points"""
    circ = synth.chain_circuit(64)
    for tau in (pow(synth.root_of_unity(64), 5, R_MOD), synth.root_of_unity(128)):
        _check(gpu, circ, _ceremony(gpu, 7, tau=tau), flavour)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_setup_from_powers_on_other_generators(gpu, flavour):
    cer = _ceremony(gpu, 8, seed=8, k1=7, k2=5)
    _check(gpu, synth.circomlike_circuit(8)[0], cer, flavour)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('log_n', [13, 14, 15])
def test_setup_from_powers_at_2_13_to_2_15(gpu, log_n, flavour):
    """from the 2^16 ceremony of the test above"""
    _check(gpu, synth.circomlike_circuit(log_n)[0], _ceremony(gpu, 16), flavour)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_one_ptau_file_serves_every_smaller_domain(gpu, tmp_path, flavour):
    """one 2^8 file, read through its memory map, for the domains 2, 4, ..., 256"""
    from circom_compat_b200 import Groth16
    cer = _ceremony(gpu, 8)
    path = tmp_path / 'pot8.ptau'
    path.write_bytes(P.write_ptau(8, cer.tau_g1, cer.tau_g2, cer.alpha_tau_g1, cer.beta_tau_g1, cer.beta_g2))
    pw = read_ptau(str(path))
    for circ in [_circuit_of('tiny', 0)] + [synth.chain_circuit(1 << k) for k in range(2, 9)]:
        pk = Groth16.generate_parameters_from_powers_of_tau(circ, pw, gpu, _reduction(flavour))
        _assert_same_key(pk, _reference_key(gpu, circ, cer, flavour))


@pytest.mark.gpu
def test_short_powers_are_refused_before_the_device_reads_them(gpu):
    """a hand-made Powers whose arrays are shorter than its power claims: ValueError, nothing read past them"""
    from circom_compat_b200 import Groth16, Powers
    cer = _ceremony(gpu, 8)
    short = Powers(8, 8, cer.tau_g1[:100], cer.tau_g2, cer.alpha_tau_g1, cer.beta_tau_g1, cer.beta_g2)
    with pytest.raises(ValueError, match='tau_g1 holds 100 rows'):
        Groth16.generate_parameters_from_powers_of_tau(synth.chain_circuit(64), short, gpu)
    circ = synth.chain_circuit(32)                                         # 2 x 32 - 1 = 63 rows suffice there
    _assert_same_key(Groth16.generate_parameters_from_powers_of_tau(circ, short, gpu), _reference_key(gpu, circ, cer, 'circom'))


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_contributions_equal_setup_with_delta(gpu, flavour):
    from circom_compat_b200 import Groth16
    cer = _ceremony(gpu, 12)
    circ = synth.circomlike_circuit(9)[0]
    pk0 = Groth16.generate_parameters_from_powers_of_tau(circ, cer, gpu, _reduction(flavour))
    x, y = 0x1234 + R_MOD // 3, R_MOD - 2
    pk1 = Groth16.contribute(pk0, ctx=gpu, x=x)
    _assert_same_key(pk1, _reference_key(gpu, circ, cer, flavour, delta=x))
    pk2 = Groth16.contribute(pk1, ctx=gpu, x=y)
    _assert_same_key(pk2, _reference_key(gpu, circ, cer, flavour, delta=x * y % R_MOD))
    pk3 = Groth16.contribute(pk2, random.Random(5), ctx=gpu)
    assert Groth16.verify_contribution(pk0, pk1, gpu) and Groth16.verify_contribution(pk1, pk2, gpu)
    assert Groth16.verify_contribution(pk0, pk3, gpu)                       # a chain of three
    assert Groth16.verify_contribution(pk0, pk0, gpu)                       # x = 1 is a contribution too


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_proofs_under_a_contributed_key_verify(gpu, flavour):
    from circom_compat_b200 import Groth16, fr_to_mont
    circ, w = synth.circomlike_circuit(10)
    pk = Groth16.contribute(Groth16.generate_parameters_from_powers_of_tau(circ, _ceremony(gpu, 12), gpu, _reduction(flavour)),
                            ctx=gpu)
    cm = circ.matrices(with_c=flavour == 'libsnark')
    p = Groth16.create_proof_with_reduction_and_matrices(pk, 0x77 + R_MOD // 5, 0x99 + R_MOD // 11, cm, circ.num_inputs,
                                                         circ.num_constraints, fr_to_mont(w), gpu, _reduction(flavour))
    inputs = w[1:circ.num_inputs]
    bad = [(inputs[0] + 1) % R_MOD] + inputs[1:]
    assert Groth16.verify_many(pk, [inputs, bad], [p, p], gpu) == [True, False]


def _g2_outside_subgroup():
    from batch_model import twist_point_outside_g2
    (x0, x1), (y0, y1) = twist_point_outside_g2(random.Random(5))
    return synth._ints_to_limbs([v * (1 << 256) % Q_MOD for v in (x0, x1, y0, y1)]).reshape(1, 16)


def _copy_key(pk, **fields):
    from circom_compat_b200 import ProvingKey
    arrs = {k: np.array(getattr(pk, k), copy=True) for k in KEY_FIELDS}
    arrs.update(fields)
    return ProvingKey(pk.n_vars, pk.n_public, pk.domain_size, *(arrs[k] for k in KEY_FIELDS))


@pytest.mark.gpu
def test_update_check_rejects_each_forgery(gpu):
    from circom_compat_b200 import Groth16
    circ = synth.circomlike_circuit(8)[0]
    pk0 = Groth16.generate_parameters_from_powers_of_tau(circ, _ceremony(gpu, 12), gpu)
    x = 0xC0FFEE + R_MOD // 7
    pk1 = Groth16.contribute(pk0, ctx=gpu, x=x)
    assert Groth16.verify_contribution(pk0, pk1, gpu)
    l_bad = np.array(pk1.l_query, copy=True); l_bad[3] = pk1.l_query[4]
    h_bad = np.array(pk1.h_query, copy=True); h_bad[-1] = pk1.h_query[0]
    d1_bad = gpu.fixed_base_g1(_limbs([x + 1]))                             # delta_1 scaled by another factor
    off = np.array(pk1.h_query, copy=True); off[5, 4] ^= 1                  # a point off the curve
    forgeries = {
        'l point': _copy_key(pk1, l_query=l_bad),
        'h point': _copy_key(pk1, h_query=h_bad),
        'delta_1 factor': _copy_key(pk1, delta_g1=d1_bad),
        'delta_2 outside G2': _copy_key(pk1, delta_g2=_g2_outside_subgroup()),
        'off curve': _copy_key(pk1, h_query=off),
        'a_query (host)': _copy_key(pk1, a_query=np.array(pk1.a_query[::-1], copy=True)),
        'gamma_abc (host)': _copy_key(pk1, gamma_abc_g1=np.array(pk0.l_query[:len(pk0.gamma_abc_g1)], copy=True)),
    }
    for name, bad in forgeries.items():
        assert not Groth16.verify_contribution(pk0, bad, gpu), name
    assert Groth16.verify_contribution(pk0, pk1, gpu)


def _raw_powers(ctx, circ, cer, flavour='circom', mutate=None, log_size=None, out_null=False, null_powers=False):
    """b2g_setup_from_powers through ctypes, for the error paths: the return code"""
    from circom_compat_b200 import _native as N
    from circom_compat_b200.groth16 import _mat_desc
    d, keep = _mat_desc(circ.matrices(with_c=True), circ.n_vars, N.REDUCTION_LIBSNARK if flavour == 'libsnark' else N.REDUCTION_CIRCOM,
                        with_c=True)
    arrays = {k: np.array(getattr(cer, k), copy=True) for k in ('tau_g1', 'tau_g2', 'alpha_tau_g1', 'beta_tau_g1', 'beta_g2')}
    if mutate:
        mutate(arrays)
    pd = N.PowersDesc()
    pd.log_size = cer.power if log_size is None else log_size
    for k, a in arrays.items():
        setattr(pd, k, a.ctypes.data)
    if null_powers:
        pd.tau_g2 = None
    n, nv, ni = 1, circ.n_vars, circ.num_inputs
    while n < circ.num_constraints + ni:
        n <<= 1
    arrs = {k: np.zeros(v, dtype=np.uint64) for k, v in {'alpha_g1': 8, 'beta_g1': 8, 'delta_g1': 8, 'beta_g2': 16, 'gamma_g2': 16,
            'delta_g2': 16, 'gamma_abc_g1': ni * 8, 'a_query': nv * 8, 'b_g1_query': nv * 8, 'b_g2_query': nv * 16,
            'l_query': (nv - ni) * 8, 'h_query': n * 8}.items()}
    out = N.SetupOut()
    for k, a in arrs.items():
        setattr(out, k, a.ctypes.data if a.size else None)
    if out_null:
        out.a_query = None
    return N.lib().b2g_setup_from_powers(ctx._h, C.byref(d), C.byref(pd), C.byref(out))


@pytest.mark.gpu
def test_errors_leave_the_context_usable(gpu):
    from circom_compat_b200 import Groth16, _native as N
    from circom_compat_b200.groth16 import _delta_key
    circ = synth.chain_circuit(64)
    cer = _ceremony(gpu, 7)
    ref = Groth16.generate_parameters_from_powers_of_tau(circ, cer, gpu)

    def still_usable():
        _assert_same_key(Groth16.generate_parameters_from_powers_of_tau(circ, cer, gpu), ref)

    def setv(name, i, word, value):
        def f(arrays):
            arrays[name][i, word] = value
        return f

    def no_c(d):
        d.c_rowptr = None

    def g2_bad(arrays):
        arrays['tau_g2'][17] = _g2_outside_subgroup()[0]

    def zero(name):
        def f(arrays):
            arrays[name][0] = 0
        return f

    messages = {}
    cases = [
        ('ceremony too small', dict(log_size=5), N.B2G_E_DOMAIN, None),
        ('log_size 29', dict(log_size=29), N.B2G_E_DOMAIN, None),
        ('tau_g1 off curve', dict(mutate=setv('tau_g1', 100, 4, 1)), N.B2G_E_INPUT, b'tau_g1[100]: off the curve or a coordinate >= p'),
        ('beta_tau_g1 coordinate >= p', dict(mutate=setv('beta_tau_g1', 3, 3, (1 << 64) - 1)), N.B2G_E_INPUT, b'beta_tau_g1[3]: off the curve'),
        ('tau_g2 outside G2', dict(mutate=g2_bad), N.B2G_E_INPUT, b'tau_g2[17]: not in G2'),
        ('beta_g2 off twist', dict(mutate=setv('beta_g2', 0, 9, 5)), N.B2G_E_INPUT, b'beta_g2[0]: off the twist'),
        ('tau_g1[0] infinity', dict(mutate=zero('tau_g1')), N.B2G_E_INPUT, b'tau_g1[0]: at infinity'),
        ('tau_g2[0] infinity', dict(mutate=zero('tau_g2')), N.B2G_E_INPUT, b'tau_g2[0]: at infinity'),
        ('null powers', dict(null_powers=True), N.B2G_E_SHAPE, None),
        ('null output', dict(out_null=True), N.B2G_E_SHAPE, None),
    ]
    for name, kw, code, msg in cases:
        rc = _raw_powers(gpu, circ, cer, **kw)
        assert rc == code, (name, rc, N.lib().b2g_last_error())
        if msg:
            assert N.lib().b2g_last_error().startswith(msg), name
        still_usable()
    # an off-curve point beyond the prefix the circuit reads is not looked at
    assert _raw_powers(gpu, circ, cer, mutate=setv('tau_g1', 200, 4, 1)) == N.B2G_OK
    # the matrix checks keep b2g_setup's codes and messages
    from circom_compat_b200.groth16 import _mat_desc
    d, keep = _mat_desc(circ.matrices(with_c=True), circ.n_vars, N.REDUCTION_CIRCOM, with_c=True)
    d.c_rowptr = None
    assert N.lib().b2g_setup_from_powers(gpu._h, C.byref(d), C.byref(N.PowersDesc()), C.byref(N.SetupOut())) == N.B2G_E_SHAPE
    assert N.lib().b2g_setup_from_powers(gpu._h, None, None, None) == N.B2G_E_SHAPE
    still_usable()
    big = synth.circomlike_circuit(13)[0]                                  # a 2^13 domain from a 2^7 ceremony
    with pytest.raises(N.PolynomialDegreeTooLarge):
        Groth16.generate_parameters_from_powers_of_tau(big, cer, gpu)

    # b2g_points_intt
    pts = gpu.fixed_base_g1(_limbs([1, 2]))
    for log_n in (0, 28):
        assert N.lib().b2g_points_intt(gpu._h, 0, log_n, pts.ctypes.data) == N.B2G_E_DOMAIN
    assert N.lib().b2g_points_intt(gpu._h, 0, 1, None) == N.B2G_E_SHAPE
    assert N.lib().b2g_points_intt(None, 0, 1, pts.ctypes.data) == N.B2G_E_SHAPE

    # b2g_delta_update
    before, keep0 = _delta_key(ref)
    after_arrs = {k: np.zeros_like(v) for k, v in keep0.items()}
    from circom_compat_b200.groth16 import _delta_desc
    after = _delta_desc(after_arrs)

    def update(x, b=before):
        xb = np.frombuffer(int(x).to_bytes(32, 'little'), dtype=np.uint8).copy()
        return N.lib().b2g_delta_update(gpu._h, C.byref(b), xb.ctypes.data, C.byref(after))
    for name, x, code in (('x = 0', 0, N.B2G_E_INPUT), ('x = r', R_MOD, N.B2G_E_INPUT), ('x = 2^256 - 1', (1 << 256) - 1, N.B2G_E_INPUT)):
        assert update(x) == code, name
        still_usable()
    for field, word in (('l_query', 4), ('h_query', 12), ('delta_g1', 1)):
        bad_arrs = {k: v.copy() for k, v in keep0.items()}
        bad_arrs[field].reshape(-1)[word] ^= 1
        assert update(5, _delta_desc(bad_arrs)) == N.B2G_E_INPUT, field
        assert N.lib().b2g_last_error().startswith(field.encode()), field
    bad_arrs = {k: v.copy() for k, v in keep0.items()}
    bad_arrs['delta_g2'] = _g2_outside_subgroup()
    assert update(5, _delta_desc(bad_arrs)) == N.B2G_E_INPUT and N.lib().b2g_last_error() == b'delta_g2[0]: not in G2'
    assert N.lib().b2g_delta_update(gpu._h, C.byref(before), None, C.byref(after)) == N.B2G_E_SHAPE
    assert update(5) == N.B2G_OK
    still_usable()

    # b2g_delta_update_check
    count = before.n_l + before.n_h
    w = np.ones(count * 2, dtype=np.uint64)
    verdict = np.zeros(1, dtype=np.uint8)
    assert N.lib().b2g_delta_update_check(gpu._h, C.byref(before), C.byref(after), w.ctypes.data, verdict.ctypes.data) == N.B2G_OK
    assert verdict[0] == 1
    w[2 * (count - 1):] = 0
    assert N.lib().b2g_delta_update_check(gpu._h, C.byref(before), C.byref(after), w.ctypes.data, verdict.ctypes.data) == N.B2G_E_INPUT
    assert N.lib().b2g_delta_update_check(gpu._h, C.byref(before), None, w.ctypes.data, verdict.ctypes.data) == N.B2G_E_SHAPE
    with pytest.raises(N.B2gError):
        Groth16.verify_contribution(ref, ref, gpu, weights=[0] * count)
    still_usable()


@pytest.mark.gpu
def test_new_entries_refuse_a_pending_proof(gpu):
    from circom_compat_b200 import Groth16, fr_to_mont, _native as N
    circ = synth.chain_circuit(64)
    cer = _ceremony(gpu, 7)
    pk = Groth16.generate_parameters_from_powers_of_tau(circ, cer, gpu)
    w = synth.chain_witness(64)
    pending = Groth16.submit(pk, 5, 7, circ.matrices(), fr_to_mont(w), gpu)
    assert _raw_powers(gpu, circ, cer) == N.B2G_E_SHAPE and b'pending' in N.lib().b2g_last_error()
    with pytest.raises(N.B2gError, match='pending'):
        Groth16.contribute(pk, ctx=gpu, x=3)
    with pytest.raises(N.B2gError, match='pending'):
        Groth16.verify_contribution(pk, pk, gpu)
    with pytest.raises(N.B2gError, match='pending'):
        gpu.points_intt(cer.tau_g1[:4])
    assert Groth16.verify(pk, w[1:circ.num_inputs], pending.wait())
    assert Groth16.verify_contribution(pk, Groth16.contribute(pk, ctx=gpu), gpu)


@pytest.mark.gpu
def test_update_check_rules_on_their_own(gpu):
    """keys whose pairing equations hold (after = before, so both sides are equal) but which break one point rule each:
    only that rule can reject them"""
    from circom_compat_b200 import Groth16
    pk = Groth16.generate_parameters_from_powers_of_tau(synth.circomlike_circuit(6)[0], _ceremony(gpu, 12), gpu)
    assert Groth16.verify_contribution(pk, pk, gpu)
    t = _g2_outside_subgroup()
    off_l = np.array(pk.l_query, copy=True); off_l[2, 4] ^= 1
    off_h = np.array(pk.h_query, copy=True); off_h[0, 1] ^= 1
    big = np.array(pk.h_query, copy=True); big[1, 3] = (1 << 64) - 1   # a coordinate >= p
    off_d1 = np.array(pk.delta_g1, copy=True).reshape(1, 8); off_d1[0, 4] ^= 1
    cases = {
        'delta_2 outside G2': dict(delta_g2=t),
        'l point off its curve': dict(l_query=off_l),
        'h point off its curve': dict(h_query=off_h),
        'h coordinate >= p': dict(h_query=big),
        'delta_1 off its curve': dict(delta_g1=off_d1),
        'delta_1 at infinity': dict(delta_g1=np.zeros((1, 8), dtype=np.uint64)),
        'delta_2 at infinity': dict(delta_g2=np.zeros((1, 16), dtype=np.uint64)),
    }
    for name, fields in cases.items():
        bad = _copy_key(pk, **fields)
        assert not Groth16.verify_contribution(bad, bad, gpu), name


@pytest.mark.gpu
def test_cpp_setup_ptau_mode_matches_python(gpu, tmp_path):
    """B2G_SETUP_PTAU=<file> groth16_bench circuit2.r1cs circuit2_witness.wtns: .r1cs + .ptau -> key -> one contribution ->
    check -> prove -> verify in C++; its key equals Python's for the same file and x"""
    import subprocess
    from circom_compat_b200 import Groth16, R1CS, R1CSFile, serialize_proving_key
    cer = _ceremony(gpu, 8, seed=21)
    path = tmp_path / 'pot8.ptau'
    path.write_bytes(P.write_ptau(8, cer.tau_g1, cer.tau_g2, cer.alpha_tau_g1, cer.beta_tau_g1, cer.beta_g2))
    exe = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench')
    out = subprocess.check_output([exe, os.path.join(GOLDEN, 'circuit2.r1cs'), os.path.join(GOLDEN, 'circuit2_witness.wtns'), '0x77'],
                                  text=True, env=dict(os.environ, B2G_SETUP_PTAU=str(path)))
    kv = dict(line.split('=', 1) for line in out.splitlines() if '=' in line)
    circ = R1CS.from_file(R1CSFile.new(open(os.path.join(GOLDEN, 'circuit2.r1cs'), 'rb').read())).to_circuit()
    pk0 = Groth16.generate_parameters_from_powers_of_tau(circ, read_ptau(str(path)), gpu)
    pk = Groth16.contribute(pk0, ctx=gpu, x=int(kv['x'], 16))
    assert bytes.fromhex(kv['key']) == serialize_proving_key(pk, True, gpu)
    assert kv['contribution'] == '1' and kv['verified'] == '1'
