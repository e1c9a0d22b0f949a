"""Compressed proofs on the device: b2g_proofs_decompress / Groth16.decompress_proofs, b2g_verify_many_compressed and
b2g_verify_batch_compressed.  The decoder is compared with the strict big-int model (tests/compressed_model.py), the verdicts
with the uncompressed verifiers on the model-decoded rows, and the new test ops 46-48 with big-int arithmetic."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from batch_model import outside_b_proof, twist_point_outside_g2
from compressed_model import (P, SENTINEL, decoded_row, g1_no_root_x, g2_bytes, g2_decompress, g2_no_root_x, proof_row,
                              twist_point_real_y, Undecodable)
from circom_compat_b200 import verifier as V
from circom_compat_b200 import ethereum as eth
from oracle import pyref as o
from test_verify_batch import _mont_words, _proof, _shape_cases, _synthetic, _weights, complex_batch  # noqa: F401

pytestmark = pytest.mark.gpu

R = o.R_MOD
_RM_INV = pow(1 << 256, -1, P)


def _compress(p) -> bytes:
    return eth.serialize_compressed(eth.Proof.from_proof(p))


def _mont_from(raw: bytes) -> int:
    return int.from_bytes(raw, 'little') * _RM_INV % P


def _rows(out):
    return [np.ascontiguousarray(r, dtype='<u8').tobytes() for r in out]


# ---------------------------------------------------------------------------------------------- test ops
def _fq2_has_root(a):
    y = o._fq2_sqrt(a)
    return y is not None and o.FQ2.sqr(y) == a


def test_fq_sqrt_op(ctx):
    rng = random.Random(46)
    squares = [rng.randrange(P) ** 2 % P for _ in range(6)]
    non = []
    while len(non) < 6:
        v = rng.randrange(1, P)
        if o._fq_sqrt(v) is None:
            non.append(v)
    vals = squares + non + [0, 1, P - 1, 4]
    got = _rows(ctx.test_op(46, _mont_words(vals)))
    for v, row in zip(vals, got):
        flag = int.from_bytes(row[32:40], 'little')
        assert flag == (o._fq_sqrt(v) is not None), v
        assert row[40:64] == bytes(24)
        if flag:
            assert pow(_mont_from(row[:32]), 2, P) == v
    assert [int.from_bytes(r[32:40], 'little') for r in got[-4:]] == [1, 1, 0, 1]


def test_fq2_sqrt_op(ctx):
    rng = random.Random(47)
    vals = [o.FQ2.sqr((rng.randrange(P), rng.randrange(P))) for _ in range(6)]
    while len(vals) < 12:                                           # non-squares: a non-residue norm
        a = (rng.randrange(P), rng.randrange(1, P))
        if not _fq2_has_root(a):
            vals.append(a)
    res = rng.randrange(1, P) ** 2 % P
    non = next(v for v in range(2, 100) if o._fq_sqrt(v) is None)
    vals += [(0, 0), (res, 0), (non, 0), (P - 1, 0), (1, 0), (0, 1), (0, res)]
    got = _rows(ctx.test_op(47, _mont_words([c for a in vals for c in a])))
    for a, row in zip(vals, got):
        flag = int.from_bytes(row[64:72], 'little')
        assert flag == _fq2_has_root(a), a
        if flag:
            assert o.FQ2.sqr((_mont_from(row[:32]), _mont_from(row[32:64]))) == a, a
        else:
            assert row[:64] == bytes(64)
    assert [int.from_bytes(r[64:72], 'little') for r in got[:6]] == [1] * 6
    assert [int.from_bytes(r[64:72], 'little') for r in got[6:12]] == [0] * 6
    assert [int.from_bytes(r[64:72], 'little') for r in got[12:15]] == [1, 1, 1]      # a1 = 0: zero, residue, non-residue


def test_g2_point_decode_op(ctx):
    """op 48 decodes without the G2 check; it is the only way to reach the y.c1 = 0 tie of the sign rule"""
    rng = random.Random(48)
    blobs = []
    for _ in range(3):
        q = o.G2.mul(o.G2_GEN, rng.randrange(1, R))
        blobs += [_compress(_proof(None, q, None))[32:96], _compress(_proof(None, o.G2.neg(q), None))[32:96]]
    outside = twist_point_outside_g2(rng)
    blobs.append(_compress(_proof(None, outside, None))[32:96])
    x, y = twist_point_real_y()
    blobs += [g2_bytes(x), g2_bytes(x, 0x80)]
    blobs += [g2_bytes((5, 7), 0x40), g2_bytes((0, 0), 0x40), g2_bytes((5, 7), 0xC0), g2_bytes((P, 1)), g2_bytes((1, P)),
              g2_bytes((P - 1, P), 0x40), g2_bytes(g2_no_root_x()), g2_bytes(((1 << 256) - 1, 0))]
    a = np.frombuffer(b''.join(blobs), dtype='<u8').copy()
    got = _rows(ctx.test_op(48, a))
    decodes = []
    for blob, row in zip(blobs, got):
        try:
            q = g2_decompress(blob, subgroup=False)
            want = proof_row(None, q, None)[64:192]
        except Undecodable:
            q, want = 'bad', b'\xff' * 128
        decodes.append(q != 'bad')
        assert row[:128] == want, blob.hex()
        assert int.from_bytes(row[128:136], 'little') == (q != 'bad')
    assert decodes == [True] * 7 + [True, True] + [True, True, False, False, False, False, False, False]
    small, big = sorted((y[0], P - y[0]))
    assert int.from_bytes(got[7][64:96], 'little') == small and int.from_bytes(got[8][64:96], 'little') == big
    assert got[7][96:128] == bytes(32) and got[8][96:128] == bytes(32)


# ---------------------------------------------------------------------------------------------- decompress_proofs
def _round_trip(ctx, proofs):
    from circom_compat_b200 import Groth16
    got = Groth16.decompress_proofs([_compress(p) for p in proofs], ctx)
    assert [g.data if g is not None else None for g in got] == [p.data for p in proofs]


def test_round_trip_golden_proofs(ctx, golden):
    from circom_compat_b200 import Proof
    _round_trip(ctx, [Proof(bytes.fromhex(c['proof_hex'])) for c in golden['test_zkey']['proofs']])


def test_round_trip_bench_key_proofs(ctx, complex_batch):
    _round_trip(ctx, complex_batch[2])


def test_round_trip_infinity_and_signs(ctx):
    proofs = [p for _, _, p, _ in _shape_cases()]
    rng = random.Random(49)
    for _ in range(8):
        a, b, c = (o.G1.mul(o.G1_GEN, rng.randrange(1, R)), o.G2.mul(o.G2_GEN, rng.randrange(1, R)), o.G1.mul(o.G1_GEN, rng.randrange(1, R)))
        proofs += [_proof(a, b, c), _proof(o.G1.neg(a), o.G2.neg(b), o.G1.neg(c))]
    proofs.append(_proof(None, None, None))
    _round_trip(ctx, proofs)


def _bad_kinds():
    """(name, function of a valid 128-byte blob -> undecodable blob)"""
    def put(off, v, keep_flags=False):
        def f(b):
            b = bytearray(b)
            flags = b[off + 31] & 0xC0
            b[off:off + 32] = v.to_bytes(32, 'little')
            if keep_flags:
                b[off + 31] |= flags
            return bytes(b)
        return f

    def flags(k):
        return lambda b: bytes(b[:k]) + bytes([b[k] | 0xC0]) + bytes(b[k + 1:])
    outside = _compress(_proof(None, twist_point_outside_g2(random.Random(50)), None))[32:96]
    return [('flags A', flags(31)), ('flags B', flags(95)), ('flags C', flags(127)),
            ('A.x = p', put(0, P)), ('A.x = 2^254 - 1', put(0, (1 << 254) - 1)),
            ('C.x = p', put(96, P)), ('C.x = 2^254 - 1', put(96, (1 << 254) - 1)),
            ('B.x.c0 = p', put(32, P)), ('B.x.c1 = p', put(64, P)), ('B.x.c1 = 2^254 - 1', put(64, (1 << 254) - 1, True)),
            ('A.x without root', put(0, g1_no_root_x())), ('C.x without root', put(96, g1_no_root_x())),
            ('B.x without root', lambda b: bytes(b[:32]) + g2_bytes(g2_no_root_x()) + bytes(b[96:])),
            ('B outside G2', lambda b: bytes(b[:32]) + outside + bytes(b[96:]))]


def test_undecodable_proofs_are_refused(ctx, complex_batch):
    from circom_compat_b200 import Groth16
    _, _, proofs = complex_batch
    good = [_compress(p) for p in proofs[:40]]
    blobs = list(good)
    kinds = _bad_kinds()
    for i, (_, f) in enumerate(kinds):
        blobs[2 * i + 1] = f(good[2 * i + 1])
    inf = bytearray(good[0])                                        # an infinity flag with a nonzero x below p
    inf[31] = (inf[31] & 0x3F) | 0x40
    blobs.append(bytes(inf))
    got = Groth16.decompress_proofs(blobs, ctx)
    for i, (blob, g) in enumerate(zip(blobs, got)):
        want = decoded_row(blob)
        assert (g.data if g is not None else SENTINEL) == want, i
    for i, (name, _) in enumerate(kinds):
        assert got[2 * i + 1] is None, name
        assert got[2 * i].data == proofs[2 * i].data, name
    assert got[-1].data == proof_row(None, proofs[0].b, proofs[0].c)
    # the raw C ABI writes the 0xFF row and ok = 0
    from circom_compat_b200 import _native as N
    data = np.frombuffer(b''.join(blobs), dtype=np.uint8).copy()
    out, ok = np.zeros((len(blobs), 256), dtype=np.uint8), np.zeros(len(blobs), dtype=np.uint8)
    N.check(N.lib().b2g_proofs_decompress(ctx._h, len(blobs), C.c_void_p(data.ctypes.data), C.c_void_p(out.ctypes.data), C.c_void_p(ok.ctypes.data)))
    for i in range(len(kinds)):
        assert ok[2 * i + 1] == 0 and out[2 * i + 1].tobytes() == SENTINEL
        assert ok[2 * i] == 1
    assert ok[-1] == 1


# ---------------------------------------------------------------------------------------------- verify_many_compressed
def test_verify_many_compressed_mixed_batch(ctx, complex_batch):
    """valid proofs, flipped sign bits and every undecodable kind: a decodable proof's verdict is verify_many's on the
    model-decoded row, an undecodable one's is False"""
    from circom_compat_b200 import Groth16, Proof
    pk, inputs, proofs = complex_batch
    n = 60
    blobs = [_compress(p) for p in proofs[:n]]
    for i, (_, f) in enumerate(_bad_kinds()):
        blobs[3 * i + 1] = f(blobs[3 * i + 1])
    for i in range(2, n, 9):                                        # A -> -A, B -> -B, C -> -C by the sign bits
        b = bytearray(blobs[i])
        b[[31, 95, 127][(i // 9) % 3]] ^= 0x80
        blobs[i] = bytes(b)
    got = Groth16.verify_many_compressed(pk, inputs[:n], blobs, ctx)
    rows = [decoded_row(b) for b in blobs]
    want = Groth16.verify_many(pk, inputs[:n], [Proof(r) for r in rows], ctx)
    assert got == want
    assert [got[3 * i + 1] for i in range(len(_bad_kinds()))] == [False] * len(_bad_kinds())
    assert [got[i] for i in range(2, n, 9)] == [False] * len(range(2, n, 9))
    assert sum(got) == n - len(_bad_kinds()) - len(range(2, n, 9))


def test_verify_many_compressed_refuses_b_outside_g2(ctx):
    """the proof verify_many accepts with B outside G2 does not decode, so its compressed verdict is False"""
    from circom_compat_b200 import Groth16, release
    vk, xs, (a, b, c) = outside_b_proof(82)
    bad = _proof(a, b, c)
    good = [_proof(a, o.G2.mul(o.G2_GEN, k), c) for k in (3, 5)]
    assert Groth16.verify_many(vk, [xs] * 3, good + [bad], ctx) == [True] * 3
    assert Groth16.verify_many_compressed(vk, [xs] * 3, [_compress(p) for p in good + [bad]], ctx) == [True, True, False]
    assert not Groth16.verify_batch_compressed(vk, [xs] * 3, [_compress(p) for p in good + [bad]], ctx)
    assert Groth16.verify_batch_compressed(vk, [xs] * 2, [_compress(p) for p in good], ctx)
    release(vk)


# ---------------------------------------------------------------------------------------------- verify_batch_compressed
@pytest.mark.parametrize('count', [1, 33, 1000, 4200])
def test_verify_batch_compressed_valid(ctx, complex_batch, count):
    """4 200 proofs cross a chunk of the input-scalar sums"""
    from circom_compat_b200 import Groth16
    pk, inputs, proofs = complex_batch
    xs, bl = [inputs[k % 1000] for k in range(count)], [_compress(proofs[k % 1000]) for k in range(count)]
    assert Groth16.verify_batch_compressed(pk, xs, bl, ctx)
    assert Groth16.verify_many_compressed(pk, xs, bl, ctx) == [True] * count


@pytest.mark.parametrize('n_public', [0, 1, 100])
def test_verify_batch_compressed_keys(ctx, n_public):
    from circom_compat_b200 import Groth16, release
    vk, inputs, proofs = _synthetic(n_public, 300 + n_public, 6)
    blobs = [_compress(p) for p in proofs]
    assert Groth16.verify_batch_compressed(vk, inputs, blobs, ctx)
    assert Groth16.verify_many_compressed(vk, inputs, blobs, ctx) == [True] * 6
    bad = list(blobs)
    bad[4] = bytes(bad[4][:31]) + bytes([bad[4][31] ^ 0x80]) + bytes(bad[4][32:])
    assert not Groth16.verify_batch_compressed(vk, inputs, bad, ctx)
    release(vk)


def test_verify_batch_compressed_shapes(ctx):
    from circom_compat_b200 import Groth16, release
    for vk, xs, proof, shape in _shape_cases():
        assert Groth16.verify_batch_compressed(vk, [xs, xs], [_compress(proof)] * 2, ctx), shape
        assert Groth16.verify_many_compressed(vk, [xs], [_compress(proof)], ctx) == [True], shape
        release(vk)


def test_one_undecodable_proof_fails_the_batch(ctx, complex_batch):
    """every undecodable kind and a flipped sign bit, first, in the middle or last among 200 valid proofs; with the same
    weights the verdict equals verify_batch on the model-decoded rows"""
    from circom_compat_b200 import Groth16, Proof
    pk, inputs, proofs = complex_batch
    rng = random.Random(51)
    ins, blobs = inputs[:200], [_compress(p) for p in proofs[:200]]
    kinds = _bad_kinds() + [('sign of A', lambda b: bytes(b[:31]) + bytes([b[31] ^ 0x80]) + bytes(b[32:]))]
    for name, f in kinds:
        for pos in (0, 100, 199):
            bl = list(blobs)
            bl[pos] = f(bl[pos])
            w = _weights(rng, 200)
            got = Groth16.verify_batch_compressed(pk, ins, bl, ctx, weights=w)
            want = Groth16.verify_batch(pk, ins, [Proof(decoded_row(b)) for b in bl], ctx, weights=w)
            assert got == want and not got, (name, pos)
    w = _weights(rng, 200)
    assert Groth16.verify_batch_compressed(pk, ins, blobs, ctx, weights=w)
    assert Groth16.verify_batch(pk, ins, proofs[:200], ctx, weights=w)


# ---------------------------------------------------------------------------------------------- errors
def test_errors_leave_the_context_usable(ctx, golden, test_zkey_bytes):
    from circom_compat_b200 import B2gError, Groth16, fr_to_mont, read_zkey, release
    from circom_compat_b200 import _native as N
    vk, inputs, proofs = _synthetic(2, 52, 5)
    blobs = [_compress(p) for p in proofs]
    assert Groth16.decompress_proofs([], ctx) == []
    assert Groth16.verify_many_compressed(vk, [], [], ctx) == []
    assert Groth16.verify_batch_compressed(vk, [], [], ctx) is True
    for bad in (blobs[0][:127], blobs[0] + b'\x00', proofs[0].data, proofs[0]):
        with pytest.raises(ValueError):
            Groth16.decompress_proofs(blobs[:2] + [bad], ctx)
        with pytest.raises(ValueError):
            Groth16.verify_many_compressed(vk, inputs[:3], blobs[:2] + [bad], ctx)
        with pytest.raises(ValueError):
            Groth16.verify_batch_compressed(vk, inputs[:3], blobs[:2] + [bad], ctx)
    with pytest.raises(V.MalformedVerifyingKey):
        Groth16.verify_many_compressed(vk, [inputs[0] + [1]], blobs[:1], ctx)
    with pytest.raises(ValueError):
        Groth16.verify_batch_compressed(vk, inputs, blobs, ctx, weights=[1, 2])
    with pytest.raises(B2gError) as e:
        Groth16.verify_batch_compressed(vk, inputs, blobs, ctx, weights=[1, 2, 0, 4, 5])
    assert e.value.code == -4
    with pytest.raises(B2gError) as e:
        Groth16.verify_many_compressed(vk, [[R, 1]] + inputs[1:], blobs, ctx)
    assert e.value.code == -4
    L, h = N.lib(), ctx.vk_handle(vk)
    buf = (C.c_uint8 * 256).from_buffer_copy(blobs[0] + blobs[1])
    pub = (C.c_uint8 * 128).from_buffer_copy(b''.join(int(x).to_bytes(32, 'little') for x in inputs[0] + inputs[1]))
    pub_r = (C.c_uint8 * 128).from_buffer_copy(R.to_bytes(32, 'little') + bytes(96))
    w = (C.c_uint8 * 32).from_buffer_copy((5).to_bytes(16, 'little') + (7).to_bytes(16, 'little'))
    w0 = (C.c_uint8 * 32).from_buffer_copy((5).to_bytes(16, 'little') + bytes(16))
    rows, ok, out = (C.c_uint8 * 512)(), (C.c_uint8 * 2)(), (C.c_uint8 * 2)()
    pub_r_text = b'public input 0 of proof 0 is not below the scalar field modulus r'
    assert L.b2g_proofs_decompress(ctx._h, 0, buf, rows, ok) == -2
    assert L.b2g_last_error() == b'b2g_proofs_decompress: count must be at least 1'
    for args in ((None, rows, ok), (buf, None, ok), (buf, rows, None)):
        assert L.b2g_proofs_decompress(ctx._h, 2, *args) == -2
        assert L.b2g_last_error() == b'null pointer'
    assert L.b2g_proofs_decompress(None, 2, buf, rows, ok) == -2
    assert L.b2g_last_error() == b'null pointer'
    assert L.b2g_verify_many_compressed(ctx._h, h, 0, pub, buf, out) == -2
    assert L.b2g_last_error() == b'b2g_verify_many_compressed: count must be at least 1'
    assert L.b2g_verify_many_compressed(ctx._h, h, 2, pub_r, buf, out) == -4
    assert L.b2g_last_error() == pub_r_text
    for args in ((h, 0, pub, None, out), (h, 2, None, buf, out), (h, 2, pub, None, out), (h, 2, pub, buf, None), (None, 2, pub, buf, out)):
        assert L.b2g_verify_many_compressed(ctx._h, *args) == -2
        assert L.b2g_last_error() == b'null pointer'
    assert L.b2g_verify_batch_compressed(ctx._h, h, 2, pub, buf, w0, out) == -4
    assert L.b2g_last_error() == b'weight 1 is zero'
    assert L.b2g_verify_batch_compressed(ctx._h, h, 2, pub_r, buf, w, out) == -4
    assert L.b2g_last_error() == pub_r_text
    assert L.b2g_verify_batch_compressed(ctx._h, h, 0, pub, buf, w, out) == -2
    assert L.b2g_last_error() == b'b2g_verify_batch_compressed: count must be at least 1'
    for args in ((h, 0, pub, None, w, out), (h, 2, None, buf, w, out), (h, 2, pub, None, w, out), (h, 2, pub, buf, None, out),
                 (h, 2, pub, buf, w, None)):
        assert L.b2g_verify_batch_compressed(ctx._h, *args) == -2
        assert L.b2g_last_error() == b'null pointer'
    assert L.b2g_proofs_decompress(ctx._h, 2, buf, rows, ok) == 0 and list(ok) == [1, 1]
    assert bytes(rows) == proofs[0].data + proofs[1].data
    assert L.b2g_verify_many_compressed(ctx._h, h, 2, pub, buf, out) == 0 and list(out) == [1, 1]
    assert L.b2g_verify_batch_compressed(ctx._h, h, 2, pub, buf, w, out) == 0 and out[0] == 1
    # a proof pending on the context
    pk, cm = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    case = g['proofs'][0]
    pending = Groth16.submit(pk, int(case['r']), int(case['s']), cm, fr_to_mont([int(x) for x in g['witness']]), ctx)
    for call in (lambda: Groth16.decompress_proofs(blobs, ctx), lambda: Groth16.verify_many_compressed(vk, inputs, blobs, ctx),
                 lambda: Groth16.verify_batch_compressed(vk, inputs, blobs, ctx)):
        with pytest.raises(B2gError) as e:
            call()
        assert e.value.code == -2
        assert e.value.msg == 'a submitted proof is still pending on this context: call b2g_prove_wait first'
    assert pending.wait().data.hex() == case['proof_hex']
    for k in (5, 1, 5):
        assert [p.data for p in Groth16.decompress_proofs(blobs[:k], ctx)] == [p.data for p in proofs[:k]]
        assert Groth16.verify_many_compressed(vk, inputs[:k], blobs[:k], ctx) == [True] * k
        assert Groth16.verify_batch_compressed(vk, inputs[:k], blobs[:k], ctx)
        assert Groth16.verify_many(vk, inputs[:k], proofs[:k], ctx) == [True] * k
    release(vk); release(pk); release(cm)


def test_cpp_mirror_verify_compressed(complex_zkey_bytes, golden):
    """Groth16::verify_many_compressed / verify_batch_compressed / decompress_proofs through groth16_bench
    (B2G_VERIFY_COMPRESSED=9): every other proof's A sign bit flipped"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, 'circom_compat_b200', 'host', 'groth16_bench')
    out = subprocess.check_output([exe, os.path.join(root, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'),
                                   'chain:%d' % int(golden['complex_zkey']['a']), '0'], text=True,
                                  env=dict(os.environ, B2G_VERIFY_COMPRESSED='9'))
    line = [l for l in out.splitlines() if l.startswith('verify_compressed')][0]
    assert line == 'verify_compressed 9 proofs (5 valid): many agree=1, batch valid=1 flipped=0, round trip=1', line
