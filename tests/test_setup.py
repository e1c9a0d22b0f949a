"""Groth16 setup on the GPU (b2g_setup, Groth16.generate_parameters_with_qap / generate_random_parameters_with_reduction, the
C++ mirror's B2G_SETUP mode).  CPU: the big-int model of the device algorithm (setup_model.py) against the closed forms of
synth.setup_scalars and oracle.pyref.trapdoor_setup_scalars.  GPU: keys byte for byte against synth.setup (host scalars,
device fixed-base products), proofs under the keys, every error code, and the C++ mirror."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from circom_compat_b200 import synth
from circom_compat_b200.zkey import R_MOD
from oracle import pyref as o
import setup_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
KEY_FIELDS = ('alpha_g1', 'beta_g1', 'beta_g2', 'gamma_g2', 'delta_g1', 'delta_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query',
              'b_g2_query', 'l_query', 'h_query')


def _secrets(seed):
    rng = random.Random(seed)
    return [rng.randrange(1, R_MOD) for _ in range(5)]           # alpha, beta, gamma, delta, tau


def _circuit(n_vars, num_inputs, rows):
    """a synth.Circuit from rows of (A, B, C) lists of (col, value)"""
    mats = []
    for x in range(3):
        r = [k for k, row in enumerate(rows) for _ in row[x]]
        c = [col for row in rows for col, _ in row[x]]
        v = [val % R_MOD for row in rows for _, val in row[x]]
        mats.append((np.array(r, dtype=np.int64), np.array(c, dtype=np.int64), v))
    return synth.Circuit(n_vars, num_inputs, len(rows), *mats)


def _tiny_full():
    """m + num_inputs = 2: the domain of two points, exactly full"""
    return _circuit(2, 1, [([(1, 1)], [(1, 1)], [(1, 1)])])


def _r1cs(name):
    from circom_compat_b200 import R1CS, R1CSFile
    return R1CS.from_file(R1CSFile.new(open(os.path.join(GOLDEN, name), 'rb').read())).to_circuit()


# ------------------------------------------------------------------------------------------------------------------ CPU
CPU_CIRCUITS = [('chain', 4), ('chain', 7), ('chain', 64), ('chain', 131), ('circomlike', 2), ('circomlike', 6), ('tiny', 0)]


def _cpu_circuit(kind, size):
    if kind == 'chain':
        return synth.chain_circuit(size)
    if kind == 'circomlike':
        return synth.circomlike_circuit(size)[0]
    return _tiny_full()


@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('kind,size', CPU_CIRCUITS)
def test_model_matches_synth_setup_scalars(kind, size, flavour):
    circ = _cpu_circuit(kind, size)
    alpha, beta, gamma, delta, tau = _secrets(size * 7 + len(kind))
    got = M.setup_scalars(circ, tau, alpha, beta, gamma, delta, flavour)
    ref = synth.setup_scalars(circ, trapdoor=(tau, alpha, beta, gamma, delta), flavour=flavour)
    assert got['lagrange'] == ref.lagrange
    assert got['a'] == ref.a_t and got['b'] == ref.b_t
    assert got['ic'] == ref.ic_t and got['l'] == ref.l_t
    assert got['h'] == ref.h_t
    assert len(got['h']) == got['n'] - (flavour == 'libsnark')


@pytest.mark.parametrize('kind,size', CPU_CIRCUITS)
def test_model_matches_pyref_trapdoor_scalars(kind, size):
    """gamma = 1 and the snarkjs H query, as the oracle's closed form takes them"""
    circ = _cpu_circuit(kind, size)
    alpha, beta, _, delta, tau = _secrets(size + 3)
    rows = [[[], [], []] for _ in range(circ.num_constraints)]
    for x, (rs, cs, vs) in enumerate((circ.A, circ.B, circ.C)):
        for r, c, v in zip(np.asarray(rs).tolist(), np.asarray(cs).tolist(), vs):
            rows[r][x].append((v, c))
    ref = o.trapdoor_setup_scalars([r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows], circ.n_vars,
                                   circ.num_inputs, tau, alpha, beta, delta)
    got = M.setup_scalars(circ, tau, alpha, beta, 1, delta, 'circom')
    assert got['n'] == ref['n']
    assert got['a'] == ref['a'] and got['b'] == ref['b']
    assert got['ic'] == ref['ic'] and got['l'] == ref['l'] and got['h'] == ref['h']


@pytest.mark.parametrize('n', [2, 8, 64])
def test_model_lagrange_inside_the_domain_is_the_indicator(n):
    """tau = omega^k: the inverse NTT of the powers gives ark-poly's indicator vector, with no special case"""
    w = synth.root_of_unity(n)
    for k in range(n):
        assert M.lagrange(n, pow(w, k, R_MOD)) == [int(i == k) for i in range(n)]


def test_model_column_sums_of_a_hot_column():
    """the constant wire in every row, repeated entries and an empty column: the sorted runs sum exactly"""
    L = list(range(1, 9))
    rows = [0, 1, 2, 3, 3, 4, 5, 6, 7, 7]
    cols = [0, 0, 0, 0, 0, 2, 0, 0, 0, 2]
    vals = [5, 5, 5, 5, 1, 9, 5, 5, 5, R_MOD - 1]
    got = M.column_sums(rows, cols, vals, L, 3)
    assert got == [(5 * sum(L[:4]) + L[3] + 5 * sum(L[5:])) % R_MOD, 0, (9 * L[4] - L[7]) % R_MOD]


def test_groth16_bench_compiles():
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


def _reduction(flavour):
    from circom_compat_b200 import CircomReduction, LibsnarkReduction
    return LibsnarkReduction if flavour == 'libsnark' else CircomReduction


def _assert_same_key(pk, ref):
    for name in KEY_FIELDS:
        a, b = np.ascontiguousarray(getattr(pk, name)), np.ascontiguousarray(getattr(ref, name))
        assert a.shape == b.shape and a.tobytes() == b.tobytes(), name
    assert (pk.n_vars, pk.n_public, pk.domain_size) == (ref.n_vars, ref.n_public, ref.domain_size)


def _check_against_synth(gpu, circ, flavour, seed):
    from circom_compat_b200 import Groth16
    alpha, beta, gamma, delta, tau = _secrets(seed)
    pk = Groth16.generate_parameters_with_qap(circ, alpha, beta, gamma, delta, tau=tau, ctx=gpu, reduction=_reduction(flavour))
    ref, _ = synth.setup(gpu, circ, trapdoor=(tau, alpha, beta, gamma, delta), flavour=flavour)
    _assert_same_key(pk, ref)
    return pk


GPU_SIZES = [('tiny', 0)] + [('chain', 1 << k) for k in (2, 3, 5, 8, 12)] + [('chain', (1 << k) - 1) for k in (3, 9, 12)] + \
            [('circomlike', k) for k in (2, 3, 6, 10, 12)]


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('kind,size', GPU_SIZES)
def test_setup_matches_synth_setup(gpu, kind, size, flavour):
    """domains from 2 to 2^12: exactly full (chain 2^k, circomlike, tiny) and with free rows (chain 2^k - 1)"""
    _check_against_synth(gpu, _cpu_circuit(kind, size), flavour, size + 11)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_setup_matches_synth_setup_at_2_18(gpu, flavour):
    circ, _ = synth.circomlike_circuit(18)
    _check_against_synth(gpu, circ, flavour, 18)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('name', ['mycircuit.r1cs', 'circuit2.r1cs'])
def test_setup_matches_synth_setup_on_reference_circuits(gpu, name, flavour):
    _check_against_synth(gpu, _r1cs(name), flavour, len(name))


def _edge(kind):
    if kind == 'wire0_everywhere':                    # the constant wire in every row of A, B and C, at 2^16
        m = (1 << 16) - 2
        rows = [([(0, 3), (k % 50 + 2, 1)], [(0, 5)], [(0, 7), (k % 50 + 2, k + 1)]) for k in range(m)]
        return _circuit(60, 2, rows)
    if kind == 'unused_columns':                      # wires 40.. occur in no row: infinity in every query
        rows = [([(k + 2, 1)], [(k + 2, 1)], [(k + 3, 1)]) for k in range(20)]
        return _circuit(80, 2, rows)
    if kind == 'repeated_entries':                    # the same (row, col) several times in one matrix
        rows = [([(2, 1), (2, 4), (3, 1)], [(2, 1), (2, R_MOD - 1), (2, 6)], [(3, 2), (3, 2)]) for _ in range(30)]
        return _circuit(6, 2, rows)
    rows = [([(k % 9 + 1, 2)], [(k % 7 + 2, 3)], []) for k in range(45)]      # an empty C
    return _circuit(12, 3, rows)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('kind', ['wire0_everywhere', 'unused_columns', 'repeated_entries', 'empty_c'])
def test_setup_edge_circuits(gpu, kind, flavour):
    circ = _edge(kind)
    pk = _check_against_synth(gpu, circ, flavour, 5)
    if kind == 'unused_columns':
        for name in ('a_query', 'b_g1_query', 'b_g2_query'):
            assert not np.asarray(getattr(pk, name))[40:].any(), name
        assert not np.asarray(pk.l_query)[38:].any()


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_setup_on_given_generators(gpu, flavour):
    """g1 = k1 G, g2 = k2 G: every point is the fixed-base product of k1 (k2) times synth.setup_scalars' scalar"""
    from circom_compat_b200 import Groth16
    circ, _ = synth.circomlike_circuit(7)
    alpha, beta, gamma, delta, tau = _secrets(77)
    k1, k2 = 0x1234567 + R_MOD // 3, 0xABCDEF + R_MOD // 5
    g1, g2 = gpu.fixed_base_g1(synth._ints_to_limbs([k1])), gpu.fixed_base_g2(synth._ints_to_limbs([k2]))
    pk = Groth16.generate_parameters_with_qap(circ, alpha, beta, gamma, delta, g1[0], g2[0], tau=tau, ctx=gpu,
                                              reduction=_reduction(flavour))
    td = synth.setup_scalars(circ, trapdoor=(tau, alpha, beta, gamma, delta), flavour=flavour)

    def on1(xs):
        return gpu.fixed_base_g1(synth._ints_to_limbs([k1 * x % R_MOD for x in xs]))

    def on2(xs):
        return gpu.fixed_base_g2(synth._ints_to_limbs([k2 * x % R_MOD for x in xs]))
    expect = {'alpha_g1': on1([alpha]), 'beta_g1': on1([beta]), 'delta_g1': on1([delta]), 'beta_g2': on2([beta]),
              'gamma_g2': on2([gamma]), 'delta_g2': on2([delta]), 'gamma_abc_g1': on1(td.ic_t), 'a_query': on1(td.a_t),
              'b_g1_query': on1(td.b_t), 'b_g2_query': on2(td.b_t), 'l_query': on1(td.l_t), 'h_query': on1(td.h_t)}
    for name, arr in expect.items():
        assert np.ascontiguousarray(getattr(pk, name)).tobytes() == arr.tobytes(), name


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_random_parameters_replay_the_draws(gpu, flavour):
    from circom_compat_b200 import Groth16
    circ, _ = synth.circomlike_circuit(9)
    pk = Groth16.generate_random_parameters_with_reduction(circ, random.Random(4242), gpu, _reduction(flavour))
    alpha, beta, gamma, delta, tau = _secrets(4242)
    ref, _ = synth.setup(gpu, circ, trapdoor=(tau, alpha, beta, gamma, delta), flavour=flavour)
    _assert_same_key(pk, ref)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_setup_keys_prove_and_verify(gpu, flavour):
    from circom_compat_b200 import Groth16, fr_to_mont
    from oracle import cref as c
    circ, w = synth.circomlike_circuit(10)
    alpha, beta, gamma, delta, tau = _secrets(1010)
    red = _reduction(flavour)
    pk = Groth16.generate_parameters_with_qap(circ, alpha, beta, gamma, delta, tau=tau, ctx=gpu, reduction=red)
    cm = circ.matrices(with_c=flavour == 'libsnark')
    r, s = 0x1111 + R_MOD // 7, 0x2222 + R_MOD // 9
    p = Groth16.create_proof_with_reduction_and_matrices(pk, r, s, cm, circ.num_inputs, circ.num_constraints, fr_to_mont(w), gpu, red)
    inputs = w[1:circ.num_inputs]
    bad = [(inputs[0] + 1) % R_MOD] + inputs[1:]
    assert Groth16.verify_many(pk, [inputs, bad], [p, p], gpu) == [True, False]
    assert Groth16.verify(pk, inputs, p) and not Groth16.verify(pk, bad, p)
    if flavour == 'circom':
        td = synth.setup_scalars(circ, trapdoor=(tau, alpha, beta, gamma, delta))
        da, db, dc = synth.expected_proof_dlogs_independent(td, circ, w, r, s)
        ea = c.limbs_to_ints(c.fq_from_mont(c.fixed_base_g1(c.ints_to_limbs([da, dc]))))
        eb = c.limbs_to_ints(c.fq_from_mont(c.fixed_base_g2(c.ints_to_limbs([db]))))
        assert p.a == (ea[0], ea[1]) and p.c == (ea[2], ea[3]) and p.b == ((eb[0], eb[1]), (eb[2], eb[3]))


def _raw_setup(ctx, circ, flavour, secrets, g1=None, g2=None, mutate=None, out_fields=None, null_tau=False):
    """b2g_setup through ctypes, for the error paths: (return code, arrays)"""
    from circom_compat_b200 import _native as N
    from circom_compat_b200.groth16 import _mat_desc
    m = circ.matrices(with_c=True)
    red = N.REDUCTION_LIBSNARK if flavour == 'libsnark' else N.REDUCTION_CIRCOM
    d, keep = _mat_desc(m, circ.n_vars, red, with_c=True)
    if mutate:
        keep = keep + mutate(d)
    sb = np.frombuffer(b''.join(int(v).to_bytes(32, 'little') for v in secrets), dtype=np.uint8).copy()
    sec = N.SetupSecrets()
    for i, name in enumerate(('alpha', 'beta', 'gamma', 'delta', 'tau')):
        setattr(sec, name, sb.ctypes.data + 32 * i)
    if null_tau:
        sec.tau = None
    if g1 is not None:
        sec.g1 = g1.ctypes.data
    if g2 is not None:
        sec.g2 = g2.ctypes.data
    n = M.domain_size(circ.num_constraints, circ.num_inputs)
    nv, ni = circ.n_vars, circ.num_inputs
    shapes = {'alpha_g1': 8, 'beta_g1': 8, 'delta_g1': 8, 'beta_g2': 16, 'gamma_g2': 16, 'delta_g2': 16, 'gamma_abc_g1': ni * 8,
              'a_query': nv * 8, 'b_g1_query': nv * 8, 'b_g2_query': nv * 16, 'l_query': (nv - ni) * 8, 'h_query': n * 8}
    arrs = {k: np.zeros(v, dtype=np.uint64) for k, v in shapes.items()}
    out = N.SetupOut()
    for k, a in arrs.items():
        setattr(out, k, a.ctypes.data if a.size else None)
    if out_fields:
        out_fields(out)
    rc = N.lib().b2g_setup(ctx._h, C.byref(d), C.byref(sec), C.byref(out))
    return rc, arrs


@pytest.mark.gpu
def test_setup_errors_leave_the_context_usable(gpu):
    from circom_compat_b200 import _native as N
    circ = synth.chain_circuit(64)
    good = _secrets(9)
    rc, ref = _raw_setup(gpu, circ, 'libsnark', good)
    assert rc == N.B2G_OK

    def no_c(d):
        d.c_rowptr = None
        return []

    def inputs(v):
        def f(d):
            d.num_inputs = v
            return []
        return f

    def rowptr(bad):
        def f(d):
            rp = np.ctypeslib.as_array(C.cast(d.a_rowptr, C.POINTER(C.c_uint32)), shape=(circ.num_constraints + 1,)).copy()
            if bad == 'start':
                rp[0] = 1
            else:
                rp[5] = rp[6] + 1
            d.a_rowptr = rp.ctypes.data
            return [rp]
        return f

    def column(d):
        col = np.ctypeslib.as_array(C.cast(d.b_col, C.POINTER(C.c_uint32)), shape=(circ.num_constraints,)).copy()
        col[3] = circ.n_vars
        d.b_col = col.ctypes.data
        return [col]

    def reduction(d):
        d.reduction = 7
        return []

    def null_out(o_):
        o_.b_g2_query = None

    def big_domain(d):
        d.num_constraints, d.num_inputs, d.n_vars = (1 << 26), 2, 64
        rp = np.zeros((1 << 26) + 1, dtype=np.uint32)
        d.a_rowptr = d.b_rowptr = d.c_rowptr = rp.ctypes.data
        return [rp]

    def libsnark_domain(d):                   # 2^27 rows and 2 inputs need 2^28 points; checked before any row pointer is read
        d.num_constraints, d.num_inputs, d.n_vars = (1 << 27), 2, 64
        return []

    def too_big(d):                           # three column-sum vectors of 2^32 - 1 elements: 384 GiB of device memory
        d.n_vars = 0xFFFFFFFF
        return []

    g1_gen = gpu.fixed_base_g1(synth._ints_to_limbs([1]))[0]
    g2_gen = gpu.fixed_base_g2(synth._ints_to_limbs([1]))[0]
    off_curve = g1_gen.copy(); off_curve[4] ^= 1
    twist_off = g2_gen.copy(); twist_off[8] ^= 1
    coord_big = g1_gen.copy(); coord_big[3] = 0xFFFFFFFFFFFFFFFF
    cases = [
        ('null C', 'libsnark', good, dict(mutate=no_c), N.B2G_E_SHAPE),
        ('null C circom', 'circom', good, dict(mutate=no_c), N.B2G_E_SHAPE),
        ('num_inputs 0', 'circom', good, dict(mutate=inputs(0)), N.B2G_E_SHAPE),
        ('num_inputs > n_vars', 'circom', good, dict(mutate=inputs(65)), N.B2G_E_SHAPE),
        ('rowptr start', 'circom', good, dict(mutate=rowptr('start')), N.B2G_E_SHAPE),
        ('rowptr decreasing', 'libsnark', good, dict(mutate=rowptr('decrease')), N.B2G_E_SHAPE),
        ('column >= n_vars', 'circom', good, dict(mutate=column), N.B2G_E_SHAPE),
        ('unknown reduction', 'circom', good, dict(mutate=reduction), N.B2G_E_SHAPE),
        ('null output', 'circom', good, dict(out_fields=null_out), N.B2G_E_SHAPE),
        ('circom domain 2^27', 'circom', good, dict(mutate=big_domain), N.B2G_E_DOMAIN),
        ('libsnark domain 2^28', 'libsnark', good, dict(mutate=libsnark_domain), N.B2G_E_DOMAIN),
        ('null secret', 'circom', good, dict(null_tau=True), N.B2G_E_SHAPE),
        ('buffers do not fit', 'libsnark', good, dict(mutate=too_big), N.B2G_E_DEVICE),
        ('alpha = r', 'circom', [R_MOD] + good[1:], {}, N.B2G_E_INPUT),
        ('tau = 2^256 - 1', 'libsnark', good[:4] + [(1 << 256) - 1], {}, N.B2G_E_INPUT),
        ('gamma = 0', 'circom', good[:2] + [0] + good[3:], {}, N.B2G_E_INPUT),
        ('delta = 0', 'libsnark', good[:3] + [0] + good[4:], {}, N.B2G_E_INPUT),
        ('g1 at infinity', 'circom', good, dict(g1=np.zeros(8, dtype=np.uint64)), N.B2G_E_INPUT),
        ('g1 off curve', 'circom', good, dict(g1=off_curve), N.B2G_E_INPUT),
        ('g1 coordinate >= p', 'circom', good, dict(g1=coord_big), N.B2G_E_INPUT),
        ('g2 at infinity', 'libsnark', good, dict(g2=np.zeros(16, dtype=np.uint64)), N.B2G_E_INPUT),
        ('g2 off twist', 'libsnark', good, dict(g2=twist_off), N.B2G_E_INPUT),
        ('g2 outside G2', 'libsnark', good, dict(g2=_g2_outside_subgroup()), N.B2G_E_INPUT),
    ]
    for name, flavour, secrets, kw, code in cases:
        rc, _ = _raw_setup(gpu, circ, flavour, secrets, **kw)
        assert rc == code, (name, rc, N.lib().b2g_last_error())
        rc, arrs = _raw_setup(gpu, circ, 'libsnark', good)
        assert rc == N.B2G_OK, name
        assert all(arrs[k].tobytes() == ref[k].tobytes() for k in ref), name
    # the matrix checks keep b2g_matrices_load's messages
    _raw_setup(gpu, circ, 'circom', good, mutate=column)
    assert N.lib().b2g_last_error() == b"matrix B column index out of range"


def _g2_outside_subgroup():
    """a point of the twist outside G2, affine Montgomery"""
    from batch_model import twist_point_outside_g2
    (x0, x1), (y0, y1) = twist_point_outside_g2(random.Random(5))
    return synth._ints_to_limbs([v * (1 << 256) % o.Q_MOD for v in (x0, x1, y0, y1)]).reshape(-1)


@pytest.mark.gpu
def test_setup_refuses_a_pending_proof(gpu):
    """b2g_prove_submit, then b2g_setup on the same context: B2G_E_SHAPE; the proof then completes and verifies, and the
    next setup succeeds"""
    from circom_compat_b200 import Groth16, fr_to_mont
    from circom_compat_b200 import _native as N
    circ = synth.chain_circuit(64)
    s = _secrets(64)
    pk = Groth16.generate_parameters_with_qap(circ, *s[:4], tau=s[4], ctx=gpu)
    w = synth.chain_witness(64)
    pending = Groth16.submit(pk, 5, 7, circ.matrices(), fr_to_mont(w), gpu)
    rc, _ = _raw_setup(gpu, circ, 'circom', s)
    assert rc == N.B2G_E_SHAPE and b'pending' in N.lib().b2g_last_error()
    p = pending.wait()
    assert Groth16.verify(pk, w[1:circ.num_inputs], p)
    rc, _ = _raw_setup(gpu, circ, 'circom', s)
    assert rc == N.B2G_OK


@pytest.mark.gpu
def test_setup_is_deterministic_across_calls_and_contexts(gpu):
    from circom_compat_b200 import Context, Groth16, LibsnarkReduction
    circ, _ = synth.circomlike_circuit(11)
    s = _secrets(31)
    k1 = Groth16.generate_parameters_with_qap(circ, *s[:4], tau=s[4], ctx=gpu, reduction=LibsnarkReduction)
    k2 = Groth16.generate_parameters_with_qap(circ, *s[:4], tau=s[4], ctx=gpu, reduction=LibsnarkReduction)
    other = Context(0)
    try:
        k3 = Groth16.generate_parameters_with_qap(circ, *s[:4], tau=s[4], ctx=other, reduction=LibsnarkReduction)
    finally:
        other.close()
    _assert_same_key(k1, k2)
    _assert_same_key(k1, k3)


@pytest.mark.gpu
def test_cpp_setup_mode_matches_python(gpu):
    """B2G_SETUP=<seed> groth16_bench circuit2.r1cs circuit2_witness.wtns: tests/groth16.rs:75-105 in C++; its key is Python's
    serialize_proving_key(generate_parameters_with_qap(...)) for the printed secrets, and its proof verifies"""
    from circom_compat_b200 import Groth16, LibsnarkReduction, serialize_proving_key
    exe = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench')
    out = subprocess.check_output([exe, os.path.join(GOLDEN, 'circuit2.r1cs'), os.path.join(GOLDEN, 'circuit2_witness.wtns')],
                                  text=True, env=dict(os.environ, B2G_SETUP='0x5E7'))
    kv = dict(line.split('=', 1) for line in out.splitlines() if '=' in line)
    alpha, beta, gamma, delta, tau = (int(kv[k], 16) for k in ('alpha', 'beta', 'gamma', 'delta', 'tau'))
    pk = Groth16.generate_parameters_with_qap(_r1cs('circuit2.r1cs'), alpha, beta, gamma, delta, tau=tau, ctx=gpu,
                                              reduction=LibsnarkReduction)
    assert bytes.fromhex(kv['key']) == serialize_proving_key(pk, True, gpu)
    assert kv['verified'] == '1'
