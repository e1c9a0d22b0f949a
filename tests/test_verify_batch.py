"""b2g_verify_batch / Groth16.verify_batch: one random-linear-combination pairing check for a whole batch of proofs.  The
batch verdict is compared with verify_many (every proof valid) plus the G2 membership of every B, and with the big-int model
of the weighted equation (tests/batch_model.py); the new test ops are compared bit for bit with big-int
arithmetic."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from batch_model import g2_in_subgroup, outside_b_proof, twist_point_outside_g2, verify_batch_rlc
from circom_compat_b200 import verifier as V
from oracle import pairing_model as M
from oracle import pyref as o

pytestmark = pytest.mark.gpu

P, R = V.P, o.R_MOD
_RM = 1 << 256


# ---------------------------------------------------------------------------------------------- encodings and keys
def _mont_words(vals):
    return np.frombuffer(b''.join((v * _RM % P).to_bytes(32, 'little') for v in vals), dtype='<u8').copy()


def _f12_words(fs):
    return np.concatenate([_mont_words([c for f6 in f for f2 in f6 for c in f2]) for f in fs]).reshape(len(fs), 48)


def _f12_from_row(row):
    raw = np.ascontiguousarray(row, dtype='<u8').tobytes()
    v = [int.from_bytes(raw[i:i + 32], 'little') * pow(_RM, -1, P) % P for i in range(0, 384, 32)]
    return tuple(tuple((v[6 * a + 2 * b], v[6 * a + 2 * b + 1]) for b in range(3)) for a in range(2))


def _g1_words(pts):
    return np.concatenate([_mont_words([0, 0] if p is None else list(p)) for p in pts]).reshape(len(pts), 8)


def _g2_words(pts):
    return np.concatenate([_mont_words([0] * 4 if q is None else [q[0][0], q[0][1], q[1][0], q[1][1]]) for q in pts]).reshape(len(pts), 16)


def _g1_from_row(row):
    raw = np.ascontiguousarray(row, dtype='<u8').tobytes()
    x, y = (int.from_bytes(raw[i:i + 32], 'little') * pow(_RM, -1, P) % P for i in (0, 32))
    return None if (x, y) == (0, 0) else (x, y)


def _proof(a, b, c):
    from circom_compat_b200 import Proof
    vals = ([0, 0] if a is None else list(a)) + ([0] * 4 if b is None else [b[0][0], b[0][1], b[1][0], b[1][1]]) + \
           ([0, 0] if c is None else list(c))
    return Proof(b''.join(int(v).to_bytes(32, 'little') for v in vals))


def _pts(p):
    a, b, c = V._proof_points(p)
    return a, b, c


def _g1(k):
    return o.G1.mul(o.G1_GEN, k)


def _g2(k):
    return o.G2.mul(o.G2_GEN, k)


def _weights(rng, n):
    return [rng.getrandbits(128) | (1 << 127) for _ in range(n)]


def _synthetic(n_public, seed, count):
    """a verifying key with known discrete logs and `count` valid proofs"""
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
    """the reference's bench key (2^14) and 1 000 proofs of chain witnesses a, a + 1, ..."""
    from circom_compat_b200 import Context, Groth16, fr_to_mont, read_zkey, release
    pk, cm = read_zkey(complex_zkey_bytes)
    cx = Context(0)
    a0 = int(golden['complex_zkey']['a'])
    rng = random.Random(1001)
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


# ---------------------------------------------------------------------------------------------- test ops
def test_batch_test_ops_match_big_int(ctx):
    rng = random.Random(45)
    qs = [_g2(rng.randrange(1, R)) for _ in range(3)] + [o.G2_GEN, None] + [twist_point_outside_g2(rng) for _ in range(3)]
    got = ctx.test_op(43, _g2_words(qs))[:, 0]
    assert [bool(v) for v in got] == [g2_in_subgroup(q) for q in qs] == [True] * 5 + [False] * 3
    ps = [_g1(rng.randrange(1, R)) for _ in range(4)] + [None, o.G1_GEN]
    ks = [rng.getrandbits(128) | (1 << 127), (1 << 128) - 1, 1, rng.getrandbits(64), rng.getrandbits(128), 2]
    kw = np.frombuffer(b''.join(k.to_bytes(16, 'little') for k in ks), dtype='<u8').copy()
    got = [_g1_from_row(r) for r in ctx.test_op(44, _g1_words(ps), kw)]
    assert got == [o.G1.mul(p, k) if p is not None else None for p, k in zip(ps, ks)]
    xs = [tuple(tuple((rng.randrange(P), rng.randrange(P)) for _ in range(3)) for _ in range(2)) for _ in range(4)]
    cyc = [V.f12_mul(M.frobenius(g, 2), g) for g in (V.f12_mul(V.f12_conj(x), V.f12_inv(x)) for x in xs)]
    es = [rng.randrange(R), R - 1, 0, 1]
    ew = np.frombuffer(b''.join(e.to_bytes(32, 'little') for e in es), dtype='<u8').copy()
    got = [_f12_from_row(r) for r in ctx.test_op(45, _f12_words(cyc), ew)]
    assert got == [V.f12_pow(g, e) for g, e in zip(cyc, es)]


# ---------------------------------------------------------------------------------------------- valid batches
def test_golden_test_zkey_proofs(ctx, golden, test_zkey_bytes):
    from circom_compat_b200 import Groth16, Proof, read_zkey, release
    pk, _ = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    xs = [int(x) for x in g['witness'][1:pk.n_public + 1]]
    proofs = [Proof(bytes.fromhex(c['proof_hex'])) for c in g['proofs']]
    assert Groth16.verify_batch(pk, [xs] * len(proofs), proofs, ctx)
    assert Groth16.verify_batch(Groth16.process_vk(pk), [xs] * len(proofs), proofs, ctx)
    release(pk)


@pytest.mark.parametrize('count', [1, 31, 33, 64, 65, 1000])
def test_reference_bench_key_batches(ctx, complex_batch, count):
    from circom_compat_b200 import Groth16
    pk, inputs, proofs = complex_batch
    assert Groth16.verify_batch(pk, inputs[:count], proofs[:count], ctx)


@pytest.mark.parametrize('n_public', [0, 1, 100])
def test_synthetic_keys(ctx, n_public):
    from circom_compat_b200 import Groth16, release
    vk, inputs, proofs = _synthetic(n_public, 200 + n_public, 6)
    assert Groth16.verify_batch(vk, inputs, proofs, ctx)
    if n_public:
        bad = [list(xs) for xs in inputs]
        bad[3][0] = (bad[3][0] + 1) % R
        assert not Groth16.verify_batch(vk, bad, proofs, ctx)
    release(vk)


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
    """a valid proof for every shape of test_verify_many's every-shape test: (A, B) present or not, the prepared inputs, C,
    gamma or delta at infinity"""
    out = []
    vk, L, ic, rng = _shape_key(1, 1)
    xs = [rng.randrange(R)]
    p = _prep(ic, xs)
    b = rng.randrange(1, R)
    a = (L['al'] * L['be'] + p * L['ga']) * pow(b, -1, R) % R
    out.append((vk, xs, _proof(_g1(a), _g2(b), None), 'C = 0'))
    x0 = (-ic[0]) * pow(ic[1], -1, R) % R
    a, b = rng.randrange(1, R), rng.randrange(1, R)
    c = (a * b - L['al'] * L['be']) * pow(L['de'], -1, R) % R
    out.append((vk, [x0], _proof(_g1(a), _g2(b), _g1(c)), 'prepared = 0'))
    c = -(L['al'] * L['be'] + p * L['ga']) * pow(L['de'], -1, R) % R
    out.append((vk, xs, _proof(None, None, _g1(c)), 'A = B = 0'))
    x1 = ((-L['al'] * L['be'] * pow(L['ga'], -1, R)) - ic[0]) * pow(ic[1], -1, R) % R
    out.append((vk, [x1], _proof(None, None, None), 'A = B = C = 0'))
    vk, L, ic, rng = _shape_key(2, 1, gamma_inf=True)
    xs = [rng.randrange(R)]
    a, b = rng.randrange(1, R), rng.randrange(1, R)
    c = (a * b - L['al'] * L['be']) * pow(L['de'], -1, R) % R
    out.append((vk, xs, _proof(_g1(a), _g2(b), _g1(c)), 'gamma = 0'))
    b = rng.randrange(1, R)
    a = L['al'] * L['be'] * pow(b, -1, R) % R
    out.append((vk, xs, _proof(_g1(a), _g2(b), None), 'gamma = C = 0'))
    vk, L, ic, rng = _shape_key(3, 2, delta_inf=True)
    xs = [rng.randrange(R), rng.randrange(R)]
    b = rng.randrange(1, R)
    a = (L['al'] * L['be'] + _prep(ic, xs) * L['ga']) * pow(b, -1, R) % R
    out.append((vk, xs, _proof(_g1(a), _g2(b), _g1(rng.randrange(1, R))), 'delta = 0'))
    return out


def test_every_loop_shape_accepts_a_valid_batch(ctx):
    from circom_compat_b200 import Groth16, release
    rng = random.Random(46)
    for vk, xs, proof, shape in _shape_cases():
        pvk = V.prepare_verifying_key(vk)
        assert V.verify_with_processed_vk(pvk, xs, proof), shape
        assert Groth16.verify_batch(vk, [xs], [proof], ctx), shape
        assert Groth16.verify_batch(vk, [xs, xs], [proof, proof], ctx, weights=_weights(rng, 2)), shape
        a, b, c = _pts(proof)
        bad = _proof(a, b, o.G1.add(c, o.G1_GEN))
        want = V.verify_with_processed_vk(pvk, xs, bad)
        assert Groth16.verify_batch(vk, [xs, xs], [proof, bad], ctx) == want, shape
        release(vk)


def test_more_than_a_chunk_and_tree_level(ctx, complex_batch):
    """4 200 proofs: three chunks of the input-scalar sums, three levels of the Miller-value product, two of the r C sum; a
    wrong input in the last chunk or a tampered last proof fails the batch"""
    from circom_compat_b200 import Groth16
    pk, inputs, proofs = complex_batch
    n = 4200
    xs, ps = [inputs[k % 1000] for k in range(n)], [proofs[k % 1000] for k in range(n)]
    assert Groth16.verify_batch(pk, xs, ps, ctx)
    bad_xs = list(xs)
    bad_xs[4100] = [(bad_xs[4100][0] + 1) % R] + bad_xs[4100][1:]
    assert not Groth16.verify_batch(pk, bad_xs, ps, ctx)
    a, b, c = _pts(ps[-1])
    assert not Groth16.verify_batch(pk, xs, ps[:-1] + [_proof(a, b, o.G1.add(c, o.G1_GEN))], ctx)


def test_more_than_128_public_inputs(ctx):
    """131 prepared points: two levels of their tree sum"""
    from circom_compat_b200 import Groth16, release
    vk, inputs, proofs = _synthetic(130, 230, 3)
    assert Groth16.verify_batch(vk, inputs, proofs, ctx)
    bad = [list(x) for x in inputs]
    bad[1][129] = (bad[1][129] + 1) % R
    assert not Groth16.verify_batch(vk, bad, proofs, ctx)
    release(vk)


# ---------------------------------------------------------------------------------------------- invalid batches
def _tampered(kind, xs, p, prev, outside):
    xs, (a, b, c) = list(xs), _pts(p)
    if kind == 0: a = (a[0], (P - a[1]) % P)
    elif kind == 1: b = _pts(prev)[1]
    elif kind == 2: c = o.G1.add(c, o.G1_GEN)
    elif kind == 3: xs[0] = (xs[0] + 1) % R
    elif kind == 4: xs = xs[::-1] if len(set(xs)) > 1 else [(x + 2) % R for x in xs]
    elif kind == 5: a = None
    elif kind == 6: b = None
    elif kind == 7: c = None
    elif kind == 8: a = (a[0], (a[1] + 1) % P)
    elif kind == 9: b = (b[0], (b[1][0], (b[1][1] + 1) % P))
    elif kind == 10: a = (a[0] + P, a[1])
    else: b = outside
    return xs, _proof(a, b, c)


def test_one_tampered_proof_fails_the_batch(ctx, complex_batch):
    """every tampering kind of test_verify_many's mixed batch, first, in the middle or last among 200 valid proofs: the
    verdict equals all(verify_many) and every B in G2"""
    from circom_compat_b200 import Groth16
    pk, inputs, proofs = complex_batch
    outside = twist_point_outside_g2(random.Random(47))
    ins, prs = inputs[:200], proofs[:200]
    for kind in range(12):
        for pos in (0, 100, 199):
            xs, bad = _tampered(kind, ins[pos], prs[pos], prs[pos - 1], outside)
            bi, bp = ins[:pos] + [xs] + ins[pos + 1:], prs[:pos] + [bad] + prs[pos + 1:]
            want = all(Groth16.verify_many(pk, bi, bp, ctx)) and g2_in_subgroup(_pts(bad)[1])
            assert Groth16.verify_batch(pk, bi, bp, ctx) == want, (kind, pos)
            assert not want, (kind, pos)                           # every kind here breaks its proof


def test_b_outside_g2_is_refused_where_verify_many_accepts(ctx):
    """A at infinity removes e(A, B) and C solves the rest of the equation, so verify_many (no subgroup check) accepts the
    proof whatever B on the twist it carries.  With B outside G2, only the membership test can refuse it: the batch is
    False alone and at every position among valid proofs, and True with B in G2 instead"""
    from circom_compat_b200 import Groth16, release
    vk, xs, (a, b, c) = outside_b_proof(81)
    bad = _proof(a, b, c)
    good = [_proof(a, _g2(k), c) for k in (3, 5, 7)]
    assert not g2_in_subgroup(b)
    assert Groth16.verify_many(vk, [xs] * 4, good + [bad], ctx) == [True] * 4
    assert Groth16.verify_batch(vk, [xs] * 3, good, ctx)
    assert not Groth16.verify_batch(vk, [xs], [bad], ctx)
    for pos in (0, 1, 3):
        assert not Groth16.verify_batch(vk, [xs] * 4, good[:pos] + [bad] + good[pos:], ctx), pos
    release(vk)


def test_weights_scale_their_own_proof(ctx):
    """C_3 + w_7 D and C_7 - w_3 D cancel in sum w_i C_i for exactly these weights (with high bits set): any changed or swapped
    weight makes the batch fail, so weight i scales proof i over all 128 bits"""
    from circom_compat_b200 import Groth16, release
    vk, inputs, proofs = _synthetic(2, 48, 10)
    rng = random.Random(48)
    w = _weights(rng, 10)
    d = _g1(rng.randrange(1, R))
    i, j = 3, 7
    bad = list(proofs)
    ai, bi, ci = _pts(proofs[i])
    aj, bj, cj = _pts(proofs[j])
    bad[i] = _proof(ai, bi, o.G1.add(ci, o.G1.mul(d, w[j])))
    bad[j] = _proof(aj, bj, o.G1.add(cj, o.G1.neg(o.G1.mul(d, w[i]))))
    assert Groth16.verify_batch(vk, inputs, bad, ctx, weights=w)
    assert not Groth16.verify_batch(vk, inputs, bad, ctx)                      # fresh random weights
    swapped = list(w)
    swapped[i], swapped[j] = w[j], w[i]
    assert not Groth16.verify_batch(vk, inputs, bad, ctx, weights=swapped)
    for k, bit in ((i, 127), (i, 3), (j, 0), (j, 64)):
        changed = list(w)
        changed[k] ^= 1 << bit
        assert not Groth16.verify_batch(vk, inputs, bad, ctx, weights=changed), (k, bit)
    release(vk)


def test_device_verdict_equals_the_model(ctx):
    """random mixed batches of a small key against verify_batch_rlc with the same weights, and the cancelling pair with all
    weights 1 (accepted by both, although both proofs are invalid)"""
    from circom_compat_b200 import Groth16, release
    vk, inputs, proofs = _synthetic(2, 49, 24)
    pvk = V.prepare_verifying_key(vk)
    rng = random.Random(49)
    outside = twist_point_outside_g2(rng)
    verdicts = []
    for t in range(4):
        idx = rng.sample(range(24), 5)
        ins, prs = [inputs[k] for k in idx], [proofs[k] for k in idx]
        if t:
            pos = rng.randrange(5)
            ins[pos], prs[pos] = _tampered(rng.choice([0, 2, 3, 6, 9, 10, 11]), ins[pos], prs[pos], prs[pos - 1], outside)
        w = _weights(rng, 5)
        want = verify_batch_rlc(pvk, ins, prs, w)
        verdicts.append(want)
        assert Groth16.verify_batch(vk, ins, prs, ctx, weights=w) == want, t
    assert verdicts[0] and not all(verdicts)
    d = _g1(777)
    (a1, b1, c1), (a2, b2, c2) = _pts(proofs[0]), _pts(proofs[1])
    pair = [_proof(a1, b1, o.G1.add(c1, d)), _proof(a2, b2, o.G1.add(c2, o.G1.neg(d)))]
    assert verify_batch_rlc(pvk, inputs[:2], pair, [1, 1])
    assert Groth16.verify_batch(vk, inputs[:2], pair, ctx, weights=[1, 1])
    assert not Groth16.verify_batch(vk, inputs[:2], pair, ctx)
    release(vk)


# ---------------------------------------------------------------------------------------------- errors
def test_errors_leave_the_context_usable(ctx, golden, test_zkey_bytes):
    from circom_compat_b200 import B2gError, Groth16, fr_to_mont, read_zkey, release
    from circom_compat_b200 import _native as N
    vk, inputs, proofs = _synthetic(2, 50, 5)
    assert Groth16.verify_batch(vk, [], [], ctx) is True
    with pytest.raises(V.MalformedVerifyingKey):
        Groth16.verify_batch(vk, [inputs[0] + [1]], proofs[:1], ctx)
    with pytest.raises(ValueError):
        Groth16.verify_batch(vk, inputs, proofs, ctx, weights=[1, 2])
    for bad in (R, -1):
        with pytest.raises(B2gError) as e:
            Groth16.verify_batch(vk, [[bad, 1]] + inputs[1:], proofs, ctx)
        assert e.value.code == -4
    for bad in (0, 1 << 128):
        with pytest.raises(B2gError) as e:
            Groth16.verify_batch(vk, inputs, proofs, ctx, weights=[1, 2, bad, 4, 5])
        assert e.value.code == -4
    L, h = N.lib(), ctx.vk_handle(vk)
    buf = (C.c_uint8 * 512).from_buffer_copy(proofs[0].data + proofs[1].data)
    pub = (C.c_uint8 * 128).from_buffer_copy(b''.join(int(x).to_bytes(32, 'little') for x in inputs[0] + inputs[1]))
    w = (C.c_uint8 * 32).from_buffer_copy((5).to_bytes(16, 'little') + (7).to_bytes(16, 'little'))
    w0 = (C.c_uint8 * 32).from_buffer_copy((5).to_bytes(16, 'little') + bytes(16))
    pub_r = (C.c_uint8 * 128).from_buffer_copy(R.to_bytes(32, 'little') + bytes(96))
    out = (C.c_uint8 * 1)()
    assert L.b2g_verify_batch(ctx._h, h, 2, pub, buf, w0, out) == -4                  # a zero weight
    assert L.b2g_last_error() == b'weight 1 is zero'
    assert L.b2g_verify_batch(ctx._h, h, 2, pub_r, buf, w, out) == -4                 # an input >= r
    assert L.b2g_last_error() == b'public input 0 of proof 0 is not below the scalar field modulus r'
    assert L.b2g_verify_batch(ctx._h, h, 0, pub, buf, w, out) == -2
    assert L.b2g_last_error() == b'b2g_verify_batch: count must be at least 1'
    for args in ((h, 0, pub, None, w, out), (h, 2, None, buf, w, out), (h, 2, pub, None, w, out), (h, 2, pub, buf, None, out),
                 (h, 2, pub, buf, w, None), (None, 2, pub, buf, w, out)):
        assert L.b2g_verify_batch(ctx._h, *args) == -2
        assert L.b2g_last_error() == b'null pointer'
    assert L.b2g_verify_batch(ctx._h, h, 2, pub, buf, w, out) == 0 and out[0] == 1
    # a proof pending on the context
    pk, cm = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    case = g['proofs'][0]
    pending = Groth16.submit(pk, int(case['r']), int(case['s']), cm, fr_to_mont([int(x) for x in g['witness']]), ctx)
    with pytest.raises(B2gError) as e:
        Groth16.verify_batch(vk, inputs, proofs, ctx)
    assert e.value.code == -2
    assert e.value.msg == 'a submitted proof is still pending on this context: call b2g_prove_wait first'
    assert pending.wait().data.hex() == case['proof_hex']
    tampered = [_proof(*_pts(p)[:2], o.G1.add(_pts(p)[2], o.G1_GEN)) for p in proofs]
    for k in (5, 1, 5):
        assert Groth16.verify_batch(vk, inputs[:k], proofs[:k], ctx)
        assert not Groth16.verify_batch(vk, inputs[:k], tampered[:k], ctx)
        assert Groth16.verify_many(vk, inputs[:k], proofs[:k], ctx) == [True] * k
    release(vk); release(pk); release(cm)


def test_cpp_mirror_verify_batch(complex_zkey_bytes, golden):
    """Groth16::verify_batch through groth16_bench (B2G_VERIFY_BATCH=9): true on nine valid proofs, false with the last A
    negated, as the C++ host verifier over every proof"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, 'circom_compat_b200', 'host', 'groth16_bench')
    out = subprocess.check_output([exe, os.path.join(root, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'),
                                   'chain:%d' % int(golden['complex_zkey']['a']), '0'], text=True, env=dict(os.environ, B2G_VERIFY_BATCH='9'))
    line = [l for l in out.splitlines() if l.startswith('verify_batch')][0]
    assert 'verify_batch 9 proofs: valid=1 tampered=0 host=1/0 agree=1' in line, line
