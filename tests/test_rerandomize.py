"""Groth16.rerandomize_proof / rerandomize_proofs (b2g_rerandomize_many): ark-groth16 0.5.0's Groth16::rerandomize_proof on
the device, compared bit for bit with the big-int model of tests/rerandomize_model.py.  The CPU tests check the model and the
factor draw; the GPU tests check the device rows against the model, the verifiers and the C++ mirror."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from circom_compat_b200 import verifier as V
from oracle import pyref as o
from rerandomize_model import proof_bytes, proof_points, rerandomize_proof

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P, R = o.Q_MOD, o.R_MOD
FACTORS = [(1, 2), (2, 1), (R - 1, R - 2), (R - 2, R - 1), ((R - 1) // 2, (R - 1) // 2), (1, 1), (R - 1, R - 1),
           (123456789, 123456789), (2, R - 1)]


def _golden_key_and_proofs(golden, test_zkey_bytes):
    from circom_compat_b200 import Proof, read_zkey
    pk, _ = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    xs = [int(x) for x in g['witness'][1:pk.n_public + 1]]
    return pk, xs, [Proof(bytes.fromhex(c['proof_hex'])) for c in g['proofs']]


def _rand_factors(rng, n):
    return [(rng.randrange(1, R), rng.randrange(1, R)) for _ in range(n)]


def _model_rows(delta, proofs, factors):
    return [proof_bytes(rerandomize_proof(delta, proof_points(p.data), r1, r2)) for p, (r1, r2) in zip(proofs, factors)]


# ---------------------------------------------------------------------------------------------- CPU: the model and the draw
def test_model_rerandomized_golden_proofs_verify(golden, test_zkey_bytes):
    """the model's rerandomized golden proofs pass oracle.pyref.verify and the product's host verifier"""
    from circom_compat_b200 import Proof
    pk, xs, proofs = _golden_key_and_proofs(golden, test_zkey_bytes)
    vk = V.VerifyingKey.from_proving_key(pk)
    pvk = V.prepare_verifying_key(vk)
    z = o.read_zkey(test_zkey_bytes, decode_points=False)
    rng = random.Random(11)
    for p, (r1, r2) in zip(proofs[:2], _rand_factors(rng, 2)):
        q = rerandomize_proof(vk.delta_g2, proof_points(p.data), r1, r2)
        assert proof_bytes(q) != p.data
        assert o.verify(z, xs, q)
        assert V.verify_with_processed_vk(pvk, xs, Proof(proof_bytes(q)))


def test_model_with_r1_one(golden, test_zkey_bytes):
    """r1 = 1: A' = A, B' = B + r2 delta_2, C' = C + r2 A"""
    pk, _, proofs = _golden_key_and_proofs(golden, test_zkey_bytes)
    delta = V.VerifyingKey.from_proving_key(pk).delta_g2
    a, b, c = proof_points(proofs[0].data)
    for r2 in (1, 2, R - 1, 987654321):
        a2, b2, c2 = rerandomize_proof(delta, (a, b, c), 1, r2)
        assert a2 == a
        assert b2 == o.G2.add(b, o.G2.mul(delta, r2))
        assert c2 == o.G1.add(c, o.G1.mul(a, r2))


def test_model_keeps_an_invalid_proof_invalid(golden, test_zkey_bytes):
    """A negated: the proof is invalid, and so is every rerandomization of it"""
    from circom_compat_b200 import Proof
    pk, xs, proofs = _golden_key_and_proofs(golden, test_zkey_bytes)
    vk = V.VerifyingKey.from_proving_key(pk)
    pvk = V.prepare_verifying_key(vk)
    a, b, c = proof_points(proofs[0].data)
    bad = (o.G1.neg(a), b, c)
    assert not V.verify_with_processed_vk(pvk, xs, Proof(proof_bytes(bad)))
    q = rerandomize_proof(vk.delta_g2, bad, 5, 7)
    assert not V.verify_with_processed_vk(pvk, xs, Proof(proof_bytes(q)))


class _Words:
    """an rng of fixed 64-bit words (next_u64), then random ones"""

    def __init__(self, words, seed=0):
        self.words, self.rest = list(words), random.Random(seed)

    def next_u64(self):
        return self.words.pop(0) if self.words else self.rest.getrandbits(64)


def test_factor_draw_redraws_both_when_one_is_zero():
    from circom_compat_b200.groth16 import _rerandomize_factors, fr_rand
    # r1's four limbs are zero (r1 = 0): r2 is drawn, then both again
    rng = _Words([0, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12])
    want_r2 = fr_rand(_Words([1, 2, 3, 4]))
    r1, r2 = _rerandomize_factors(rng)
    assert (r1, r2) == (fr_rand(_Words([5, 6, 7, 8])), fr_rand(_Words([9, 10, 11, 12])))
    assert want_r2 != r2
    # r2 = 0: both again
    rng = _Words([1, 2, 3, 4, 0, 0, 0, 0, 13, 14, 15, 16, 17, 18, 19, 20])
    assert _rerandomize_factors(rng) == (fr_rand(_Words([13, 14, 15, 16])), fr_rand(_Words([17, 18, 19, 20])))
    # a limb set >= r is rejected by fr_rand itself, inside the draw of r1
    rng = _Words([2 ** 64 - 1] * 4 + [21, 22, 23, 24, 25, 26, 27, 28])
    assert _rerandomize_factors(rng) == (fr_rand(_Words([21, 22, 23, 24])), fr_rand(_Words([25, 26, 27, 28])))


def test_factor_draw_matches_fr_rand_on_a_seeded_random():
    from circom_compat_b200.groth16 import _rerandomize_factors, fr_rand
    for seed in (0, 1, 2024):
        a, b = random.Random(seed), random.Random(seed)
        for _ in range(5):
            assert _rerandomize_factors(a) == (fr_rand(b), fr_rand(b))


def test_factors_out_of_range_are_refused_before_the_device():
    from circom_compat_b200 import B2gError, Groth16, Proof
    vk = V.VerifyingKey(o.G1_GEN, o.G2_GEN, o.G2_GEN, o.G2_GEN, [o.G1_GEN])
    for bad in ((0, 1), (1, 0), (R, 1), (1, R), (-1, 1)):
        with pytest.raises(B2gError) as e:
            Groth16.rerandomize_proofs(vk, [Proof(bytes(256))], factors=[bad])
        assert e.value.code == -4
    with pytest.raises(ValueError):
        Groth16.rerandomize_proofs(vk, [Proof(bytes(256))], factors=[(1, 1), (1, 1)])
    assert Groth16.rerandomize_proofs(vk, [], factors=[]) == []


class _MT19937_64:
    """std::mt19937_64 (the C++ mirror's rng in groth16_bench), with next_u64 for fr_rand"""
    M64 = (1 << 64) - 1

    def __init__(self, seed):
        self.mt = [seed & self.M64]
        for i in range(1, 312):
            self.mt.append((6364136223846793005 * (self.mt[-1] ^ (self.mt[-1] >> 62)) + i) & self.M64)
        self.i = 312

    def next_u64(self):
        if self.i == 312:
            for k in range(312):
                x = (self.mt[k] & 0xFFFFFFFF80000000) | (self.mt[(k + 1) % 312] & 0x7FFFFFFF)
                self.mt[k] = self.mt[(k + 156) % 312] ^ (x >> 1) ^ (0xB5026F5AA96619E9 if x & 1 else 0)
            self.i = 0
        y = self.mt[self.i]
        self.i += 1
        y ^= (y >> 29) & 0x5555555555555555
        y ^= (y << 17) & 0x71D67FFFEDA60000
        y ^= (y << 37) & 0xFFF7EEE000000000
        y ^= y >> 43
        return y & self.M64


def test_mt19937_64_model():
    """the C++ standard's check value: the 10 000th output of a default-constructed std::mt19937_64"""
    g = _MT19937_64(5489)
    for _ in range(9999):
        g.next_u64()
    assert g.next_u64() == 9981545732273789042


# ---------------------------------------------------------------------------------------------- GPU: bit-exact rows
def _synthetic_key(n_public, seed, count):
    """a verifying key with known discrete logs and `count` valid proofs (C solved from the verifying equation)"""
    from circom_compat_b200 import Proof
    rng = random.Random(seed)
    al, be, ga, de = (rng.randrange(1, R) for _ in range(4))
    ic = [rng.randrange(1, R) for _ in range(n_public + 1)]
    vk = V.VerifyingKey(o.G1.mul(o.G1_GEN, al), o.G2.mul(o.G2_GEN, be), o.G2.mul(o.G2_GEN, ga), o.G2.mul(o.G2_GEN, de),
                        [o.G1.mul(o.G1_GEN, k) for k in ic])
    inputs, proofs = [], []
    for _ in range(count):
        xs = [rng.randrange(R) for _ in range(n_public)]
        a, b = rng.randrange(1, R), rng.randrange(1, R)
        prep = (ic[0] + sum(x * k for x, k in zip(xs, ic[1:]))) % R
        c = (a * b - al * be - prep * ga) * pow(de, -1, R) % R
        inputs.append(xs)
        proofs.append(Proof(proof_bytes((o.G1.mul(o.G1_GEN, a), o.G2.mul(o.G2_GEN, b), o.G1.mul(o.G1_GEN, c)))))
    return vk, inputs, proofs


@pytest.mark.gpu
def test_golden_proofs_bit_exact(ctx, golden, test_zkey_bytes):
    from circom_compat_b200 import Groth16, release
    pk, xs, proofs = _golden_key_and_proofs(golden, test_zkey_bytes)
    delta = V.VerifyingKey.from_proving_key(pk).delta_g2
    rows = [p for p in proofs for _ in FACTORS]
    factors = FACTORS * len(proofs)
    got = Groth16.rerandomize_proofs(pk, rows, ctx=ctx, factors=factors)
    assert [q.data for q in got] == _model_rows(delta, rows, factors)
    assert Groth16.verify_many(pk, [xs] * len(got), got, ctx) == [True] * len(got)
    release(pk)


@pytest.mark.gpu
def test_reference_bench_key_bit_exact(ctx, golden, complex_zkey_bytes):
    from circom_compat_b200 import Groth16, fr_to_mont, read_zkey, release
    pk, cm = read_zkey(complex_zkey_bytes)
    a0 = int(golden['complex_zkey']['a'])
    rng = random.Random(14)
    ws = [o.chain_witness(pk.n_vars, a0 + k) for k in range(3)]
    proofs = Groth16.create_proofs(pk, [(rng.randrange(R), rng.randrange(R)) for _ in ws], cm, [fr_to_mont(w) for w in ws], ctx)
    inputs = [list(w[1:pk.n_public + 1]) for w in ws]
    rows, ins = [p for p in proofs for _ in FACTORS], [x for x in inputs for _ in FACTORS]
    factors = FACTORS * len(proofs)
    got = Groth16.rerandomize_proofs(pk, rows, ctx=ctx, factors=factors)
    assert [q.data for q in got] == _model_rows(V.VerifyingKey.from_proving_key(pk).delta_g2, rows, factors)
    assert Groth16.verify_many(pk, ins, got, ctx) == [True] * len(got)
    release(pk); release(cm)


@pytest.mark.gpu
def test_synthetic_100_input_key_bit_exact(ctx):
    from circom_compat_b200 import Groth16, release
    vk, inputs, proofs = _synthetic_key(100, 100, 3)
    rng = random.Random(100)
    factors = FACTORS + _rand_factors(rng, 3)
    rows, ins = [proofs[i % 3] for i in range(len(factors))], [inputs[i % 3] for i in range(len(factors))]
    got = Groth16.rerandomize_proofs(vk, rows, ctx=ctx, factors=factors)
    assert [q.data for q in got] == _model_rows(vk.delta_g2, rows, factors)
    assert Groth16.verify_many(vk, ins, got, ctx) == [True] * len(got)
    assert Groth16.verify_batch(vk, ins, got, ctx)
    release(vk)


@pytest.mark.gpu
def test_infinity_edges(ctx):
    """A, B or C at infinity, C = -r2 A (C' = infinity) and B = -r2 delta_2 (B' = infinity), against the model"""
    from circom_compat_b200 import Groth16, Proof, release
    vk, _, proofs = _synthetic_key(1, 7, 1)
    a, b, c = proof_points(proofs[0].data)
    d = vk.delta_g2
    rng = random.Random(8)
    cases = []                                                          # (points, r1, r2)
    for r1, r2 in FACTORS[:4] + _rand_factors(rng, 2):
        cases += [((None, b, c), r1, r2), ((a, None, c), r1, r2), ((a, b, None), r1, r2), ((None, None, None), r1, r2),
                  ((a, b, o.G1.neg(o.G1.mul(a, r2))), r1, r2), ((a, o.G2.neg(o.G2.mul(d, r2)), c), r1, r2),
                  ((None, b, None), r1, r2)]
    rows = [Proof(proof_bytes(pts)) for pts, _, _ in cases]
    factors = [(r1, r2) for _, r1, r2 in cases]
    got = Groth16.rerandomize_proofs(vk, rows, ctx=ctx, factors=factors)
    want = [rerandomize_proof(d, pts, r1, r2) for pts, r1, r2 in cases]
    assert [q.data for q in got] == [proof_bytes(w) for w in want]
    for (pts, _, _), w in zip(cases, want):
        if pts[0] is None:
            assert w[0] is None and w[2] == pts[2]                      # A' = infinity, C' = C
    assert [w[2] is None for w in want][4::7] == [True] * 6             # C = -r2 A
    assert [w[1] is None for w in want][5::7] == [True] * 6             # B = -r2 delta_2
    release(vk)


@pytest.mark.gpu
def test_outputs_verify_and_differ(ctx, golden, test_zkey_bytes):
    """rerandomized valid proofs pass verify_many, verify_batch and (on a sample) the host verifier, and differ from their
    inputs; rerandomize_proof draws from its rng as rerandomize_proofs does"""
    from circom_compat_b200 import Groth16, release
    pk, xs, proofs = _golden_key_and_proofs(golden, test_zkey_bytes)
    rows = [proofs[i % len(proofs)] for i in range(200)]
    got = Groth16.rerandomize_proofs(pk, rows, random.Random(3), ctx)
    assert all(q.data != p.data for p, q in zip(rows, got))
    assert len({q.data for q in got}) == len(got)
    assert Groth16.verify_many(pk, [xs] * len(got), got, ctx) == [True] * len(got)
    assert Groth16.verify_batch(pk, [xs] * len(got), got, ctx)
    pvk = Groth16.process_vk(pk)
    assert all(Groth16.verify_with_processed_vk(pvk, xs, q) for q in got[:3])
    one = random.Random(3)
    assert [Groth16.rerandomize_proof(pk, p, one, ctx).data for p in rows[:4]] == [q.data for q in got[:4]]
    assert Groth16.rerandomize_proofs(pk, rows[:2], ctx=ctx)[0].data != rows[0].data      # secrets.SystemRandom by default
    release(pk)


@pytest.mark.gpu
def test_malformed_rows(ctx, golden, test_zkey_bytes):
    """a coordinate >= p, or A, B or C off its curve: ok = 0 and the 0xFF row; the rows around it are unaffected"""
    from circom_compat_b200 import Groth16, Proof, release
    pk, xs, proofs = _golden_key_and_proofs(golden, test_zkey_bytes)
    delta = V.VerifyingKey.from_proving_key(pk).delta_g2
    a, b, c = proof_points(proofs[0].data)

    def coord_ge_p(k):
        d = bytearray(proofs[0].data)
        d[32 * k:32 * k + 32] = (int.from_bytes(d[32 * k:32 * k + 32], 'little') + P).to_bytes(32, 'little')
        return Proof(bytes(d))
    bad = [coord_ge_p(k) for k in range(8)] + [Proof(proof_bytes(pts)) for pts in (
        ((a[0], (a[1] + 1) % P), b, c), (a, (b[0], (b[1][0], (b[1][1] + 1) % P)), c), (a, b, (c[0], (c[1] + 1) % P)),
        ((1, 1), None, None))] + [Proof(b'\xff' * 256)]
    rows, want_ok = [], []
    for q in bad:
        rows += [proofs[1], q, proofs[2]]
        want_ok += [True, False, True]
    factors = _rand_factors(random.Random(5), len(rows))
    got = Groth16.rerandomize_proofs(pk, rows, ctx=ctx, factors=factors)
    assert [q is not None for q in got] == want_ok
    good = [(p, f) for p, f, k in zip(rows, factors, want_ok) if k]
    assert [q.data for q in got if q is not None] == _model_rows(delta, [p for p, _ in good], [f for _, f in good])
    # the raw rows: 0xFF where ok = 0, which verify_many reports invalid
    from circom_compat_b200 import _native as N
    h = ctx.vk_handle(pk)
    buf = np.frombuffer(b''.join(p.data for p in rows), dtype=np.uint8).copy()
    r1 = np.frombuffer(b''.join(f.to_bytes(32, 'little') for f, _ in factors), dtype=np.uint8).copy()
    r2 = np.frombuffer(b''.join(f.to_bytes(32, 'little') for _, f in factors), dtype=np.uint8).copy()
    out, ok = np.zeros((len(rows), 256), dtype=np.uint8), np.zeros(len(rows), dtype=np.uint8)
    ptr = lambda x: C.c_void_p(x.ctypes.data)
    assert N.lib().b2g_rerandomize_many(ctx._h, h, len(rows), ptr(buf), ptr(r1), ptr(r2), ptr(out), ptr(ok)) == 0
    assert [bool(k) for k in ok] == want_ok
    assert all(out[i].tobytes() == b'\xff' * 256 for i in range(len(rows)) if not want_ok[i])
    sentinel = Proof(b'\xff' * 256)
    assert Groth16.verify_many(pk, [xs], [sentinel], ctx) == [False]
    with pytest.raises(ValueError):
        Groth16.rerandomize_proof(pk, bad[0], random.Random(1), ctx)
    release(pk)


@pytest.mark.gpu
def test_large_calls_match_single_calls(ctx, golden, test_zkey_bytes):
    """row i of a 4 096-proof call equals a one-proof call on proof i; a 65 536-proof call runs and matches on a sample"""
    from circom_compat_b200 import Groth16, release
    pk, xs, proofs = _golden_key_and_proofs(golden, test_zkey_bytes)
    rng = random.Random(4096)
    base = [proofs[i % len(proofs)] for i in range(4096)]
    rows = Groth16.rerandomize_proofs(pk, base, rng, ctx)               # 4 096 distinct valid proofs
    factors = _rand_factors(rng, 4096)
    got = Groth16.rerandomize_proofs(pk, rows, ctx=ctx, factors=factors)
    for i in range(4096):
        assert Groth16.rerandomize_proofs(pk, [rows[i]], ctx=ctx, factors=[factors[i]])[0].data == got[i].data, i
    delta = V.VerifyingKey.from_proving_key(pk).delta_g2
    sample = rng.sample(range(4096), 8)
    assert [got[i].data for i in sample] == _model_rows(delta, [rows[i] for i in sample], [factors[i] for i in sample])
    big_rows = rows * 16
    big_f = _rand_factors(rng, len(big_rows))
    big = Groth16.rerandomize_proofs(pk, big_rows, ctx=ctx, factors=big_f)
    assert len(big) == 65536 and all(q is not None for q in big)
    sample = rng.sample(range(65536), 12) + [0, 65535]
    assert [big[i].data for i in sample] == _model_rows(delta, [big_rows[i] for i in sample], [big_f[i] for i in sample])
    assert Groth16.verify_batch(pk, [xs] * 65536, big, ctx)
    release(pk)


@pytest.mark.gpu
def test_errors_leave_the_context_usable(ctx, golden, test_zkey_bytes):
    from circom_compat_b200 import B2gError, Groth16, fr_to_mont, read_zkey, release
    from circom_compat_b200 import _native as N
    pk, xs, proofs = _golden_key_and_proofs(golden, test_zkey_bytes)
    L, h = N.lib(), ctx.vk_handle(pk)
    n = 3
    rows = (C.c_uint8 * (256 * n)).from_buffer_copy(b''.join(p.data for p in proofs[:n]))
    one = (C.c_uint8 * (32 * n)).from_buffer_copy(b''.join((k + 1).to_bytes(32, 'little') for k in range(n)))
    out, ok = (C.c_uint8 * (256 * n))(), (C.c_uint8 * n)()
    want = Groth16.rerandomize_proofs(pk, proofs[:n], ctx=ctx, factors=[(k + 1, k + 1) for k in range(n)])

    def good_call():
        assert L.b2g_rerandomize_many(ctx._h, h, n, rows, one, one, out, ok) == 0
        assert list(ok) == [1] * n and bytes(out) == b''.join(q.data for q in want)

    good_call()
    assert L.b2g_rerandomize_many(ctx._h, h, 0, rows, one, one, out, ok) == -2
    assert L.b2g_last_error() == b'b2g_rerandomize_many: count must be at least 1'
    good_call()
    args = [ctx._h, h, n, rows, one, one, out, ok]
    for k in (0, 1, 3, 4, 5, 6, 7):
        bad = list(args)
        bad[k] = None
        assert L.b2g_rerandomize_many(*bad) == -2
        assert L.b2g_last_error() == b'null pointer'
        good_call()
    for which, value, at in ((0, 0, 1), (1, 0, 2), (0, R, 0), (1, R + 5, 1), (1, (1 << 256) - 1, 2)):
        fs = [bytearray((k + 1).to_bytes(32, 'little')) for k in range(n)]
        fs[at] = bytearray(value.to_bytes(32, 'little'))
        bad_f = (C.c_uint8 * (32 * n)).from_buffer_copy(b''.join(fs))
        r1, r2 = (bad_f, one) if which == 0 else (one, bad_f)
        assert L.b2g_rerandomize_many(ctx._h, h, n, rows, r1, r2, out, ok) == -4
        assert L.b2g_last_error() == b'b2g_rerandomize_many: factor r%d of proof %d is not in [1, r)' % (which + 1, at)
        good_call()
    # buffers that cannot fit: refused before the factors are read, and the context's buffers are allocated again
    assert L.b2g_rerandomize_many(ctx._h, h, 0xFFFFFFFF, rows, one, one, out, ok) == -3
    assert b'do not fit in device memory' in L.b2g_last_error()
    good_call()
    # a proof pending on the context
    pk2, cm = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    case = g['proofs'][0]
    pending = Groth16.submit(pk2, int(case['r']), int(case['s']), cm, fr_to_mont([int(x) for x in g['witness']]), ctx)
    with pytest.raises(B2gError) as e:
        Groth16.rerandomize_proofs(pk, proofs[:n], ctx=ctx, factors=[(k + 1, k + 1) for k in range(n)])
    assert e.value.code == -2
    assert pending.wait().data.hex() == case['proof_hex']
    good_call()
    release(pk); release(pk2); release(cm)


@pytest.mark.gpu
def test_cpp_mirror_rerandomize_many(ctx, golden, complex_zkey_bytes):
    """Groth16::rerandomize_many through groth16_bench (B2G_RERANDOMIZE=5, factors from std::mt19937_64 seeded 0x5EED): the
    C++ rows equal Groth16.rerandomize_proofs's on the same inputs with the same rng stream, and pass the host verifier"""
    from circom_compat_b200 import Groth16, Proof, read_zkey, release
    exe = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench')
    out = subprocess.check_output([exe, os.path.join(ROOT, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'),
                                   'chain:%d' % int(golden['complex_zkey']['a']), '0'], text=True,
                                  env=dict(os.environ, B2G_RERANDOMIZE='5'))
    lines = dict(l.split('=', 1) for l in out.splitlines() if l.startswith('rerand'))
    ins = [Proof(bytes.fromhex(lines['rerand_in[%d]' % i])) for i in range(5)]
    pk, _ = read_zkey(complex_zkey_bytes)
    py = Groth16.rerandomize_proofs(pk, ins, _MT19937_64(0x5EED), ctx)
    assert [lines['rerand[%d]' % i] for i in range(5)] == [q.data.hex() for q in py]
    assert 'rerandomize 5 proofs: valid=5 changed=5' in out, out
    release(pk)
