"""b2g_verify_many / Groth16.verify_many: Groth16 verification of many proofs in one device pass, on the device pairing of
csrc/pairing.cuh.  The tower and pairing test ops are compared bit for bit with the host verifier's big-int arithmetic
(circom_compat_b200/verifier.py); batch verdicts are compared proof by proof with verify_with_processed_vk."""
import ctypes as C
import random

import numpy as np
import pytest

from circom_compat_b200 import verifier as V
from oracle import pairing_model as M
from oracle import pyref as o

pytestmark = pytest.mark.gpu

P, R = V.P, o.R_MOD
_RM = 1 << 256


# ---------------------------------------------------------------------------------------------- encodings
def _mont_words(vals):
    return np.frombuffer(b''.join((v * _RM % P).to_bytes(32, 'little') for v in vals), dtype='<u8').copy()


def _f12_vals(f):
    return [c for f6 in f for f2 in f6 for c in f2]


def _f12_words(fs):
    return np.concatenate([_mont_words(_f12_vals(f)) for f in fs]).reshape(len(fs), 48)


def _f12_from_row(row):
    raw = np.ascontiguousarray(row, dtype='<u8').tobytes()
    v = [int.from_bytes(raw[i:i + 32], 'little') * pow(_RM, -1, P) % P for i in range(0, 384, 32)]
    return tuple(tuple((v[6 * a + 2 * b], v[6 * a + 2 * b + 1]) for b in range(3)) for a in range(2))


def _rand_f12(rng):
    return tuple(tuple((rng.randrange(P), rng.randrange(P)) for _ in range(3)) for _ in range(2))


def _g1_words(pts):
    return np.concatenate([_mont_words([0, 0] if p is None else list(p)) for p in pts]).reshape(len(pts), 8)


def _g2_words(pts):
    return np.concatenate([_mont_words([0] * 4 if q is None else [q[0][0], q[0][1], q[1][0], q[1][1]]) for q in pts]).reshape(len(pts), 16)


def _proof(a, b, c):
    from circom_compat_b200 import Proof
    vals = ([0, 0] if a is None else list(a)) + ([0] * 4 if b is None else [b[0][0], b[0][1], b[1][0], b[1][1]]) + \
           ([0, 0] if c is None else list(c))
    return Proof(b''.join(int(v).to_bytes(32, 'little') for v in vals))


def _g1(k):
    return o.G1.mul(o.G1_GEN, k)


def _g2(k):
    return o.G2.mul(o.G2_GEN, k)


def _twist_point_outside_g2(rng):
    while True:
        x = (rng.randrange(P), rng.randrange(P))
        y = o._fq2_sqrt(V.f2_add(V.f2_mul(V.f2_sqr(x), x), V.TWIST_B))
        if y is not None:
            return (x, y)


# ---------------------------------------------------------------------------------------------- test ops
def test_fq12_ops_match_big_int(ctx):
    from circom_compat_b200 import verifier as V
    rng = random.Random(30)
    xs, ys = [_rand_f12(rng) for _ in range(6)], [_rand_f12(rng) for _ in range(6)]
    # cyclotomic elements for op 32: the easy part of a random element
    cyc = [V.f12_mul(M.frobenius(g, 2), g) for g in (V.f12_mul(V.f12_conj(x), V.f12_inv(x)) for x in xs)]
    a, b = _f12_words(xs), _f12_words(ys)
    got = lambda op, aa, bb=None: [_f12_from_row(r) for r in ctx.test_op(op, aa, bb)]
    assert got(30, a, b) == [V.f12_mul(x, y) for x, y in zip(xs, ys)]
    assert got(31, a) == [V.f12_mul(x, x) for x in xs]
    assert got(32, _f12_words(cyc)) == [V.f12_mul(g, g) for g in cyc]
    for k, op in ((1, 33), (2, 34), (3, 35)):
        assert got(op, a) == [V.f12_pow(x, P ** k) for x in xs[:2]] + [M.frobenius(x, k) for x in xs[2:]]
    assert got(38, a) == [V.f12_inv(x) for x in xs]
    lines = [tuple((rng.randrange(P), rng.randrange(P)) for _ in range(3)) for _ in xs]
    lw = np.concatenate([_mont_words([v for c in l for v in c]) for l in lines]).reshape(len(xs), 24)
    assert got(39, a, lw) == [V.f12_mul(x, ((l[0], V.F2_ZERO, V.F2_ZERO), (l[1], l[2], V.F2_ZERO))) for x, l in zip(xs, lines)]


def test_final_exponentiation_matches_host(ctx):
    rng = random.Random(36)
    xs = [_rand_f12(rng) for _ in range(3)] + [V.miller_loop([(_g1(5), _g2(7))])]
    got = [_f12_from_row(r) for r in ctx.test_op(36, _f12_words(xs))]
    assert got == [V.final_exponentiation(x) for x in xs]


def test_line_steps_and_miller_loop_match_the_model(ctx):
    """the projective steps and the Miller loop, whose values (unlike the pairing's) are the model's, not the host's"""
    rng = random.Random(40)
    ts = [(_g2(k)[0], _g2(k)[1], (1, 0)) for k in (3, 5)]
    z = (rng.randrange(P), rng.randrange(P))
    ts.append((V.f2_mul(_g2(7)[0], z), V.f2_mul(_g2(7)[1], z), z))                 # Z != 1
    tw = np.concatenate([_mont_words([v for c in t for v in c]) for t in ts]).reshape(len(ts), 24)
    qs = [_g2(11), _g2(13), _g2(17)]

    def split(row):
        f = _f12_from_row(row)
        return (f[0][0], f[0][1], f[0][2]), (f[1][0], f[1][1], f[1][2])
    assert [split(r) for r in ctx.test_op(41, tw)] == [M.dbl_step(t) for t in ts]
    assert [split(r) for r in ctx.test_op(42, tw, _g2_words(qs))] == [M.add_step(t, q) for t, q in zip(ts, qs)]
    ps = [_g1(2), _g1(rng.randrange(1, R))]
    got = [_f12_from_row(r) for r in ctx.test_op(40, _g1_words(ps), _g2_words(qs[:2]))]
    assert got == [M.miller_loop([(p, q)]) for p, q in zip(ps, qs)]


def test_pairing_matches_host(ctx):
    rng = random.Random(37)
    ks = [(1, 1), (2, 1), (1, 3)] + [(rng.randrange(1, R), rng.randrange(1, R)) for _ in range(2)]
    ps, qs = [_g1(a) for a, _ in ks] + [None, _g1(3)], [_g2(b) for _, b in ks] + [_g2(2), None]
    got = [_f12_from_row(r) for r in ctx.test_op(37, _g1_words(ps), _g2_words(qs))]
    assert got[0] == V.pairing(o.G1_GEN, o.G2_GEN)
    assert got[-2:] == [V.F12_ONE, V.F12_ONE]
    assert got[:-2] == [V.pairing(p, q) for p, q in zip(ps[:-2], qs[:-2])]
    assert got[1] == V.f12_mul(got[0], got[0]) and got[2] == V.f12_pow(got[0], 3)     # bilinearity


# ---------------------------------------------------------------------------------------------- keys and proofs
def _synthetic(n_public, seed, count):
    """a verifying key with known discrete logs and `count` valid proofs: A = a G1, B = b G2 and C solved from
    a b = alpha beta + (ic_0 + sum x_i ic_i) gamma + c delta"""
    rng = random.Random(seed)
    al, be, ga, de = (rng.randrange(1, R) for _ in range(4))
    ic = [rng.randrange(1, R) for _ in range(n_public + 1)]
    vk = V.VerifyingKey(_g1(al), _g2(be), _g2(ga), _g2(de), [_g1(k) for k in ic])
    inputs, proofs = [], []
    for j in range(count):
        xs = [[0, R - 1, 1][j % 3] if i == 0 else rng.randrange(R) for i in range(n_public)]
        a, b = rng.randrange(1, R), rng.randrange(1, R)
        prep = (ic[0] + sum(x * k for x, k in zip(xs, ic[1:]))) % R
        c = (a * b - al * be - prep * ga) * pow(de, -1, R) % R
        inputs.append(xs)
        proofs.append(_proof(_g1(a), _g2(b), _g1(c)))
    return vk, inputs, proofs


@pytest.fixture(scope='module')
def complex_batch(complex_zkey_bytes, golden):
    """the reference's bench key (2^14) and 1 000 proofs of chain witnesses a, a + 1, ... (create_proofs in chunks)"""
    from circom_compat_b200 import Context, Groth16, fr_to_mont, read_zkey, release
    pk, cm = read_zkey(complex_zkey_bytes)
    cx = Context(0)
    a0 = int(golden['complex_zkey']['a'])
    rng = random.Random(1000)
    inputs, proofs = [], []
    for base in range(0, 1000, 250):
        ws = [o.chain_witness(pk.n_vars, a0 + base + k) for k in range(250)]
        rs = [(rng.randrange(R), rng.randrange(R)) for _ in ws]
        proofs += Groth16.create_proofs(pk, rs, cm, [fr_to_mont(w) for w in ws], cx)
        inputs += [list(w[1:pk.n_public + 1]) for w in ws]
    release(cm)
    yield pk, inputs, proofs
    release(pk)
    cx.close()


def test_golden_test_zkey_proofs(ctx, golden, test_zkey_bytes):
    from circom_compat_b200 import Groth16, Proof, read_zkey, release
    pk, _ = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    xs = [int(x) for x in g['witness'][1:pk.n_public + 1]]
    proofs = [Proof(bytes.fromhex(c['proof_hex'])) for c in g['proofs']]
    pvk = Groth16.process_vk(pk)
    assert all(Groth16.verify_with_processed_vk(pvk, xs, p) for p in proofs)
    assert Groth16.verify_many(pk, [xs] * len(proofs), proofs, ctx) == [True] * len(proofs)
    assert Groth16.verify_many(pvk, [xs] * len(proofs), proofs, ctx) == [True] * len(proofs)
    # the device's e(alpha, beta) (op 37 on the key's points) equals the host's prepared value
    assert _f12_from_row(ctx.test_op(37, _g1_words([pvk.vk.alpha_g1]), _g2_words([pvk.vk.beta_g2]))[0]) == pvk.alpha_g1_beta_g2
    release(pk)


@pytest.mark.parametrize('count', [1, 31, 33, 1000])
def test_reference_bench_key_batches(ctx, complex_batch, count):
    from circom_compat_b200 import Groth16
    pk, inputs, proofs = complex_batch
    assert Groth16.verify_many(pk, inputs[:count], proofs[:count], ctx) == [True] * count


def test_libsnark_reduction_proofs(ctx):
    from circom_compat_b200 import Groth16, LibsnarkReduction, fr_to_mont, synth, release
    circ, w = synth.circomlike_circuit(12)
    pk, _ = synth.setup(ctx, circ, flavour='libsnark')
    cm = circ.matrices(with_c=True)
    rng = random.Random(12)
    rs = [(rng.randrange(R), rng.randrange(R)) for _ in range(5)]
    proofs = Groth16.create_proofs(pk, rs, cm, [fr_to_mont(w)] * 5, ctx, LibsnarkReduction)
    xs = list(w[1:circ.num_inputs])
    assert Groth16.verify_many(pk, [xs] * 5, proofs, ctx) == [True] * 5
    release(pk); release(cm)


@pytest.mark.parametrize('n_public', [0, 1, 100])
def test_synthetic_keys(ctx, n_public):
    """0 and 100 public inputs; inputs 0, r - 1 and 1 in first position"""
    from circom_compat_b200 import Groth16, release
    vk, inputs, proofs = _synthetic(n_public, 100 + n_public, 6)
    assert Groth16.verify_many(vk, inputs, proofs, ctx) == [True] * 6
    pvk = V.prepare_verifying_key(vk)
    assert V.verify_with_processed_vk(pvk, inputs[0], proofs[0])
    if n_public:
        bad = [[(xs[0] + 1) % R] + xs[1:] for xs in inputs]
        assert Groth16.verify_many(vk, bad, proofs, ctx) == [False] * 6
    release(vk)


def test_mixed_batch_matches_host(ctx, complex_batch):
    """valid and tampered proofs at random positions; verdicts equal verify_with_processed_vk proof by proof, except a
    coordinate >= p, which is invalid on the device (the host verifier reduces it)"""
    from circom_compat_b200 import Groth16
    pk, inputs, proofs = complex_batch
    pvk = Groth16.process_vk(pk)
    rng = random.Random(7)
    g1 = o.G1_GEN
    cases = []                                                        # (inputs, proof, expected or None = ask the host)
    for j in range(40):
        cases.append((inputs[j], proofs[j], None))
    outside = _twist_point_outside_g2(rng)
    assert V.g2_on_curve(outside) and o.G2.mul(outside, R - 1) != o.G2.neg(outside)    # on the twist, not in G2
    for j in range(40, 100):
        xs, p = list(inputs[j]), proofs[j]
        a, b, c = p.a, p.b, p.c
        kind = j % 12
        expect = None
        if kind == 0: a = (a[0], (P - a[1]) % P)                         # A negated
        elif kind == 1: b = proofs[j - 1].b                              # B of another proof
        elif kind == 2: c = o.G1.add(c, g1)                              # C + G
        elif kind == 3: xs[0] = (xs[0] + 1) % R                          # wrong public input
        elif kind == 4: xs = xs[::-1] if len(set(xs)) > 1 else [(x + 2) % R for x in xs]   # permuted inputs
        elif kind == 5: a = None
        elif kind == 6: b = None
        elif kind == 7: c = None
        elif kind == 8: a = (a[0], (a[1] + 1) % P)                       # off the curve
        elif kind == 9: b = (b[0], (b[1][0], (b[1][1] + 1) % P))         # off the twist
        elif kind == 10: a = (a[0] + P, a[1]); expect = False            # a coordinate >= p
        else: b = outside                                                # on the twist, outside G2
        cases.append((xs, _proof(a, b, c), expect))
    rng.shuffle(cases)
    got = Groth16.verify_many(pk, [c[0] for c in cases], [c[1] for c in cases], ctx)
    want = [Groth16.verify_with_processed_vk(pvk, xs, p) if e is None else e for xs, p, e in cases]
    assert got == want
    assert sum(want) >= 40 and not all(want)


def test_off_curve_vk_is_refused(ctx):
    from circom_compat_b200 import B2gError
    vk, _, _ = _synthetic(2, 5, 1)
    bad_g1 = V.VerifyingKey(vk.alpha_g1, vk.beta_g2, vk.gamma_g2, vk.delta_g2, vk.gamma_abc_g1[:2] + [(1, 3)])
    bad_g2 = V.VerifyingKey(vk.alpha_g1, vk.beta_g2, (vk.gamma_g2[0], (vk.gamma_g2[1][0], (vk.gamma_g2[1][1] + 1) % P)), vk.delta_g2,
                            vk.gamma_abc_g1)
    for bad in (bad_g1, bad_g2):
        with pytest.raises(B2gError) as e:
            ctx.vk_handle(bad)
        assert e.value.code == -4


def test_errors_leave_the_context_usable(ctx):
    from circom_compat_b200 import B2gError, Groth16, release
    from circom_compat_b200 import _native as N
    vk, inputs, proofs = _synthetic(2, 9, 5)
    assert Groth16.verify_many(vk, [], [], ctx) == []
    with pytest.raises(V.MalformedVerifyingKey):
        Groth16.verify_many(vk, [inputs[0] + [1]], proofs[:1], ctx)
    for bad in (R, -1, 1 << 256):
        with pytest.raises(B2gError) as e:
            Groth16.verify_many(vk, [[bad, 1]] + inputs[1:], proofs, ctx)
        assert e.value.code == -4
    L, h = N.lib(), ctx.vk_handle(vk)
    pub_r = (C.c_uint8 * 64).from_buffer_copy(R.to_bytes(32, 'little') + (1).to_bytes(32, 'little'))
    buf1 = (C.c_uint8 * 256).from_buffer_copy(proofs[0].data)
    assert L.b2g_verify_many(ctx._h, h, 1, pub_r, buf1, (C.c_uint8 * 1)()) == -4      # >= r refused by the library itself
    assert L.b2g_last_error() == b'public input 0 of proof 0 is not below the scalar field modulus r'
    buf = (C.c_uint8 * 256)()
    out = (C.c_uint8 * 8)()
    pub = (C.c_uint8 * 64)()
    assert L.b2g_verify_many(ctx._h, h, 0, pub, buf, out) == -2
    assert L.b2g_last_error() == b'b2g_verify_many: count must be at least 1'
    for args in ((h, 0, pub, None, out), (h, 1, None, buf, out), (h, 1, pub, None, out), (None, 1, pub, buf, out), (h, 1, pub, buf, None)):
        assert L.b2g_verify_many(ctx._h, *args) == -2
        assert L.b2g_last_error() == b'null pointer'
    tampered = [_proof(p.a, p.b, o.G1.add(p.c, o.G1_GEN)) for p in proofs]
    for k in (5, 1, 5):
        assert Groth16.verify_many(vk, inputs[:k], proofs[:k], ctx) == [True] * k
        assert Groth16.verify_many(vk, inputs[:k], tampered[:k], ctx) == [False] * k
    release(vk)


# ---------------------------------------------------------------------------------------------- every loop shape, accepted
def _shape_key(seed, n_public, gamma_inf=False, delta_inf=False):
    rng = random.Random(seed)
    logs = {k: rng.randrange(1, R) for k in ('al', 'be', 'ga', 'de')}
    ic = [rng.randrange(1, R) for _ in range(n_public + 1)]
    vk = V.VerifyingKey(_g1(logs['al']), _g2(logs['be']), None if gamma_inf else _g2(logs['ga']),
                        None if delta_inf else _g2(logs['de']), [_g1(k) for k in ic])
    return vk, logs, ic, rng


def _prep(ic, xs):
    return (ic[0] + sum(x * k for x, k in zip(xs, ic[1:]))) % R


def _shape_cases():
    """(vk, inputs, proof, Miller-loop shape) with a valid proof for every shape the batch can take: the stepped pair (A, B)
    present or not, and 0 / 1 / 2 prepared pairs (the prepared inputs, C, gamma or delta at infinity drop a pair).
    Exponents: a b = al be + prep ga + c de, a term dropping out with its infinite point."""
    out = []
    vk, L, ic, rng = _shape_key(1, 1)
    xs = [rng.randrange(R)]
    p = _prep(ic, xs)
    b = rng.randrange(1, R)
    a = (L['al'] * L['be'] + p * L['ga']) * pow(b, -1, R) % R                      # C at infinity
    out.append((vk, xs, _proof(_g1(a), _g2(b), None), 'v+1 (C = 0)'))
    x0 = (-ic[0]) * pow(ic[1], -1, R) % R                                           # prepared inputs at infinity
    a, b = rng.randrange(1, R), rng.randrange(1, R)
    c = (a * b - L['al'] * L['be']) * pow(L['de'], -1, R) % R
    out.append((vk, [x0], _proof(_g1(a), _g2(b), _g1(c)), 'v+1 (prepared = 0)'))
    c = -(L['al'] * L['be'] + p * L['ga']) * pow(L['de'], -1, R) % R               # A = B = infinity
    out.append((vk, xs, _proof(None, None, _g1(c)), '0+2'))
    x1 = ((-L['al'] * L['be'] * pow(L['ga'], -1, R)) - ic[0]) * pow(ic[1], -1, R) % R    # A = B = C = infinity
    out.append((vk, [x1], _proof(None, None, None), '0+1'))
    vk, L, ic, rng = _shape_key(2, 1, gamma_inf=True)                              # gamma at infinity
    xs = [rng.randrange(R)]
    a, b = rng.randrange(1, R), rng.randrange(1, R)
    c = (a * b - L['al'] * L['be']) * pow(L['de'], -1, R) % R
    out.append((vk, xs, _proof(_g1(a), _g2(b), _g1(c)), 'v+1 (gamma = 0)'))
    b = rng.randrange(1, R)
    a = L['al'] * L['be'] * pow(b, -1, R) % R                                       # gamma and C at infinity
    out.append((vk, xs, _proof(_g1(a), _g2(b), None), 'v+0'))
    vk, L, ic, rng = _shape_key(3, 2, delta_inf=True)                              # delta at infinity: C is free
    xs = [rng.randrange(R), rng.randrange(R)]
    b = rng.randrange(1, R)
    a = (L['al'] * L['be'] + _prep(ic, xs) * L['ga']) * pow(b, -1, R) % R
    out.append((vk, xs, _proof(_g1(a), _g2(b), _g1(rng.randrange(1, R))), 'v+1 (delta = 0)'))
    return out


def test_every_miller_loop_shape_accepts_a_valid_proof(ctx):
    from circom_compat_b200 import Groth16, release
    for vk, xs, proof, shape in _shape_cases():
        pvk = V.prepare_verifying_key(vk)
        assert V.verify_with_processed_vk(pvk, xs, proof), shape
        bad = _proof(proof.a if proof.a != (0, 0) else None, proof.b if proof.b != ((0, 0), (0, 0)) else None,
                     o.G1.add(None if proof.c == (0, 0) else proof.c, o.G1_GEN))
        assert Groth16.verify_many(vk, [xs, xs], [proof, bad], ctx) == [True, V.verify_with_processed_vk(pvk, xs, bad)], shape
        release(vk)


def test_off_curve_points_are_refused_where_the_product_would_hold(ctx):
    """B (A) at infinity removes e(A, B) from the product, and C is solved so that the rest equals e(alpha, beta): only the
    on-curve check of A (B) makes these proofs invalid"""
    from circom_compat_b200 import Groth16, release
    vk, L, ic, rng = _shape_key(4, 1)
    xs = [rng.randrange(R)]
    c = -(L['al'] * L['be'] + _prep(ic, xs) * L['ga']) * pow(L['de'], -1, R) % R
    g2 = o.G2_GEN
    off_b = (g2[0], (g2[1][0], (g2[1][1] + 1) % P))
    cases = [_proof(None, None, _g1(c)), _proof((1, 3), None, _g1(c)), _proof(None, off_b, _g1(c))]
    pvk = V.prepare_verifying_key(vk)
    assert [V.verify_with_processed_vk(pvk, xs, p) for p in cases] == [True, False, False]
    assert Groth16.verify_many(vk, [xs] * 3, cases, ctx) == [True, False, False]
    release(vk)


def test_loaded_key_holds_the_host_alpha_beta(ctx, test_zkey_bytes):
    from circom_compat_b200 import Groth16, read_zkey, release
    from circom_compat_b200 import _native as N
    pk, _ = read_zkey(test_zkey_bytes)
    for key in (pk, _shape_key(5, 3)[0]):
        out = np.zeros(48, dtype=np.uint64)
        N.check(N.lib().b2g_vk_alpha_beta(ctx.vk_handle(key), out.ctypes.data))
        assert _f12_from_row(out) == Groth16.process_vk(key).alpha_g1_beta_g2
        release(key)


def test_cpp_mirror_verify_many(complex_zkey_bytes, golden):
    """Groth16::verify_many through groth16_bench (B2G_VERIFY_MANY=9: nine proofs, A negated in every other one) agrees with
    the C++ host verify_with_processed_vk proof by proof"""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, 'circom_compat_b200', 'host', 'groth16_bench')
    out = subprocess.check_output([exe, os.path.join(root, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'),
                                   'chain:%d' % int(golden['complex_zkey']['a']), '0'], text=True, env=dict(os.environ, B2G_VERIFY_MANY='9'))
    line = [l for l in out.splitlines() if l.startswith('verify_many')][0]
    assert 'verify_many 9 proofs (5 valid): agree=1' in line, line
