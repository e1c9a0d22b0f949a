"""b2g_verify_batch_locate / Groth16.verify_batch_locate: the batch check of verify_batch once per group of 64 proofs over the
group's well-formed proofs, with verify_many's verdict for the well-formed proofs of a failing group.  Verdict vectors are
compared with verify_many AND the G2 membership of B, and with a big-int model of the grouping rules built on
batch_model.verify_batch_rlc."""
import ctypes as C
import os
import random
import subprocess

import pytest

from batch_model import g2_in_subgroup, outside_b_proof, twist_point_outside_g2, verify_batch_rlc
from circom_compat_b200 import verifier as V
from oracle import pyref as o
from test_verify_batch import _proof, _pts, _shape_cases, _synthetic, _tampered, _weights, complex_batch  # noqa: F401
from test_verify_compressed import _bad_kinds, _compress

pytestmark = pytest.mark.gpu

P, R = V.P, o.R_MOD
GROUP = 64


# ---------------------------------------------------------------------------------------------- the model
def _well_formed(proof) -> bool:
    a, b, c = V._proof_points(proof)
    coords = [v for pt in (a, c) if pt is not None for v in pt] + ([v for xy in b for v in xy] if b is not None else [])
    return all(v < P for v in coords) and V.g1_on_curve(a) and V.g1_on_curve(c) and V.g2_on_curve(b) and g2_in_subgroup(b)


def locate_model(pvk, inputs, proofs, weights):
    """the verdicts b2g_verify_batch_locate computes for these weights: 0 for a malformed proof, 1 in a group whose well-formed
    proofs pass verify_batch_rlc, else the host verifier's verdict"""
    out = []
    for g in range(0, len(proofs), GROUP):
        idx = range(g, min(g + GROUP, len(proofs)))
        wf = [i for i in idx if _well_formed(proofs[i])]
        holds = not wf or verify_batch_rlc(pvk, [inputs[i] for i in wf], [proofs[i] for i in wf], [weights[i] for i in wf])
        out += [i in wf and (holds or V.verify_with_processed_vk(pvk, inputs[i], proofs[i])) for i in idx]
    return out


def _expected(ctx, vk, inputs, proofs):
    """verify_many's verdict AND the G2 membership of B, per proof"""
    from circom_compat_b200 import Groth16
    return [m and g2_in_subgroup(_pts(p)[1]) for m, p in zip(Groth16.verify_many(vk, inputs, proofs, ctx), proofs)]


def _neg_a(p):
    a, b, c = _pts(p)
    return _proof((a[0], P - a[1]), b, c)


# ---------------------------------------------------------------------------------------------- valid batches
@pytest.mark.parametrize('count', [1, 63, 64, 65, 1000, 4200])
def test_valid_bench_key_batches(ctx, complex_batch, count):
    from circom_compat_b200 import Groth16
    pk, inputs, proofs = complex_batch
    xs, ps = [inputs[k % 1000] for k in range(count)], [proofs[k % 1000] for k in range(count)]
    assert Groth16.verify_batch_locate(pk, xs, ps, ctx) == [True] * count


def test_golden_test_zkey_proofs(ctx, golden, test_zkey_bytes):
    from circom_compat_b200 import Groth16, Proof, read_zkey, release
    pk, _ = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    xs = [int(x) for x in g['witness'][1:pk.n_public + 1]]
    proofs = [Proof(bytes.fromhex(c['proof_hex'])) for c in g['proofs']]
    assert Groth16.verify_batch_locate(pk, [xs] * len(proofs), proofs, ctx) == [True] * len(proofs)
    assert Groth16.verify_batch_locate(Groth16.process_vk(pk), [xs] * len(proofs), proofs, ctx) == [True] * len(proofs)
    release(pk)


@pytest.mark.parametrize('n_public', [0, 1, 100, 130])
def test_synthetic_keys(ctx, n_public):
    """130 inputs: 131 prepared points per group, more than one CTA's worth of the group sum"""
    from circom_compat_b200 import Groth16, release
    vk, inputs, proofs = _synthetic(n_public, 300 + n_public, 70)
    assert Groth16.verify_batch_locate(vk, inputs, proofs, ctx) == [True] * 70
    if n_public:
        bad = [list(xs) for xs in inputs]
        bad[66][n_public - 1] = (bad[66][n_public - 1] + 1) % R
        assert Groth16.verify_batch_locate(vk, bad, proofs, ctx) == [k != 66 for k in range(70)]
    release(vk)


# ---------------------------------------------------------------------------------------------- invalid proofs
def test_every_tampering_kind_at_group_edges(ctx, complex_batch):
    """every tampering kind of test_verify_batch at the first and last proof of the first two groups and at the last of
    1 000: the verdicts equal verify_many AND B in G2, and only the tampered proof is False"""
    from circom_compat_b200 import Groth16
    pk, inputs, proofs = complex_batch
    outside = twist_point_outside_g2(random.Random(60))
    for kind in range(12):
        for pos in (0, 63, 64, 127, 999):
            xs, bad = _tampered(kind, inputs[pos], proofs[pos], proofs[pos - 1], outside)
            bi, bp = inputs[:pos] + [xs] + inputs[pos + 1:], proofs[:pos] + [bad] + proofs[pos + 1:]
            want = [True] * 1000
            want[pos] = Groth16.verify_many(pk, [xs], [bad], ctx)[0] and g2_in_subgroup(_pts(bad)[1])
            got = Groth16.verify_batch_locate(pk, bi, bp, ctx)
            assert got == want, (kind, pos)
            assert not got[pos], (kind, pos)


def test_several_bad_proofs(ctx, complex_batch):
    """in one group, in different groups, a whole group invalid, a whole group malformed"""
    from circom_compat_b200 import Groth16
    pk, inputs, proofs = complex_batch
    n = 300
    xs, ps = inputs[:n], list(proofs[:n])
    cases = {'one group': [3, 17, 40], 'different groups': [5, 70, 200, 299],
             'a whole group': list(range(64, 128)), 'a malformed group': list(range(128, 192))}
    for name, bad in cases.items():
        qs = list(ps)
        for k in bad:
            if name == 'a malformed group':
                a, b, c = _pts(ps[k])
                qs[k] = _proof((a[0], (a[1] + 1) % P), b, c)          # off the curve
            else:
                qs[k] = _neg_a(ps[k])
        want = [k not in bad for k in range(n)]
        assert _expected(ctx, pk, xs, qs) == want, name
        assert Groth16.verify_batch_locate(pk, xs, qs, ctx) == want, name


def test_one_bad_proof_in_every_group(ctx):
    """4 200 proofs of a 100-input key, one invalid proof per group: every group fails and the fallback checks all 4 134
    well-formed proofs, so its per-(proof, input) buffers grow to 4 134 x 100 records"""
    from circom_compat_b200 import Groth16, release
    vk, inputs, proofs = _synthetic(100, 400, 70)
    n = 4200
    xs, ps = [inputs[k % 70] for k in range(n)], [proofs[k % 70] for k in range(n)]
    rng = random.Random(61)
    bad = {g * GROUP + rng.randrange(min(GROUP, n - g * GROUP)) for g in range((n + GROUP - 1) // GROUP)}
    qs = [_neg_a(p) if k in bad else p for k, p in enumerate(ps)]
    assert Groth16.verify_batch_locate(vk, xs, qs, ctx) == [k not in bad for k in range(n)]
    release(vk)


def test_b_outside_g2(ctx):
    """verify_many accepts the proof whose B is outside G2; the new call refuses it and keeps its group's other proofs"""
    from circom_compat_b200 import Groth16, release
    vk, xs, (a, b, c) = outside_b_proof(82)
    bad = _proof(a, b, c)
    good = [_proof(a, _g2k, c) for _g2k in (o.G2.mul(o.G2_GEN, k) for k in range(3, 73))]
    assert Groth16.verify_many(vk, [xs], [bad], ctx) == [True]
    assert Groth16.verify_batch_locate(vk, [xs], [bad], ctx) == [False]
    for pos in (0, 5, 63, 64, 70):
        ps = good[:pos] + [bad] + good[pos:]
        assert Groth16.verify_batch_locate(vk, [xs] * len(ps), ps, ctx) == [k != pos for k in range(len(ps))], pos
    release(vk)


def _cancelling_pair(vk, inputs, proofs, i, j, w, rng):
    """proofs i and j made invalid so that their errors cancel for weights w: C_i + w_j D and C_j - w_i D"""
    d = o.G1.mul(o.G1_GEN, rng.randrange(1, R))
    bad = list(proofs)
    ai, bi, ci = _pts(proofs[i])
    aj, bj, cj = _pts(proofs[j])
    bad[i] = _proof(ai, bi, o.G1.add(ci, o.G1.mul(d, w[j])))
    bad[j] = _proof(aj, bj, o.G1.add(cj, o.G1.neg(o.G1.mul(d, w[i]))))
    return bad


def test_groups_are_independent(ctx):
    """the cancelling pair of test_weights_scale_their_own_proof: inside one group the chosen weights make both proofs pass,
    as the model says; split over two groups, verify_batch over the whole batch passes while the new call flags both"""
    from circom_compat_b200 import Groth16, release
    vk, inputs, proofs = _synthetic(2, 62, 100)
    pvk = V.prepare_verifying_key(vk)
    rng = random.Random(62)
    w = _weights(rng, 100)
    for i, j, together in ((3, 7, True), (3, 70, False)):
        bad = _cancelling_pair(vk, inputs, proofs, i, j, w, rng)
        assert not V.verify_with_processed_vk(pvk, inputs[i], bad[i]) and not V.verify_with_processed_vk(pvk, inputs[j], bad[j])
        assert Groth16.verify_batch(vk, inputs, bad, ctx, weights=w)
        want = [together or k not in (i, j) for k in range(100)]
        assert locate_model(pvk, inputs, bad, w) == want, (i, j)
        assert Groth16.verify_batch_locate(vk, inputs, bad, ctx, weights=w) == want, (i, j)
        assert Groth16.verify_batch_locate(vk, inputs, bad, ctx) == [k not in (i, j) for k in range(100)], (i, j)
    release(vk)


def test_every_loop_shape_next_to_a_bad_proof(ctx):
    """each Miller-loop shape of the group pair loop (gamma or delta at infinity, the prepared inputs or sum r C at
    infinity) as a valid proof in a group with an invalid neighbour, and alone"""
    from circom_compat_b200 import Groth16, release
    for vk, xs, proof, shape in _shape_cases():
        a, b, c = _pts(proof)
        bad = _proof(a, b, o.G1.add(c, o.G1_GEN))
        pvk = V.prepare_verifying_key(vk)
        want_bad = V.verify_with_processed_vk(pvk, xs, bad)
        assert Groth16.verify_batch_locate(vk, [xs], [proof], ctx) == [True], shape
        assert Groth16.verify_batch_locate(vk, [xs] * 3, [proof, bad, proof], ctx) == [True, want_bad, True], shape
        release(vk)


def test_device_verdicts_equal_the_model(ctx):
    """random mixed batches of 150 proofs (three groups) of a two-input key, against locate_model with the same weights"""
    from circom_compat_b200 import Groth16, release
    vk, inputs, proofs = _synthetic(2, 63, 150)
    pvk = V.prepare_verifying_key(vk)
    rng = random.Random(63)
    outside = twist_point_outside_g2(rng)
    for t in range(2):
        ins, prs = list(inputs), list(proofs)
        for pos in rng.sample(range(150), 4 + 3 * t):
            ins[pos], prs[pos] = _tampered(rng.randrange(12), ins[pos], prs[pos], prs[pos - 1], outside)
        w = _weights(rng, 150)
        want = locate_model(pvk, ins, prs, w)
        assert Groth16.verify_batch_locate(vk, ins, prs, ctx, weights=w) == want, t
        assert want == _expected(ctx, vk, ins, prs), t
        assert not all(want)
    release(vk)


# ---------------------------------------------------------------------------------------------- compressed
def test_compressed(ctx, complex_batch):
    """every undecodable kind is False and the rest True; the verdicts equal decompress_proofs followed by
    verify_batch_locate on the decoded rows"""
    from circom_compat_b200 import Groth16, Proof
    pk, inputs, proofs = complex_batch
    n = 200
    blobs = [_compress(p) for p in proofs[:n]]
    kinds = _bad_kinds()
    at = [5 * i + 1 for i in range(len(kinds))] + [150]
    for k, (_, f) in zip(at, kinds + [kinds[0]]):
        blobs[k] = f(blobs[k])
    w = _weights(random.Random(64), n)
    got = Groth16.verify_batch_locate_compressed(pk, inputs[:n], blobs, ctx, weights=w)
    assert got == [k not in at for k in range(n)]
    decoded = Groth16.decompress_proofs(blobs, ctx)
    rows = [d if d is not None else Proof(b'\xff' * 256) for d in decoded]
    assert Groth16.verify_batch_locate(pk, inputs[:n], rows, ctx, weights=w) == got
    flipped = list(blobs)                                           # a decodable invalid proof: the sign of A flipped
    b = bytearray(flipped[70])
    b[31] ^= 0x80
    flipped[70] = bytes(b)
    got = Groth16.verify_batch_locate_compressed(pk, inputs[:n], flipped, ctx)
    assert got == [k not in at and k != 70 for k in range(n)]


# ---------------------------------------------------------------------------------------------- errors
def test_errors_leave_the_context_usable(ctx, golden, test_zkey_bytes):
    from circom_compat_b200 import B2gError, Groth16, fr_to_mont, read_zkey, release
    from circom_compat_b200 import _native as N
    vk, inputs, proofs = _synthetic(2, 65, 5)
    assert Groth16.verify_batch_locate(vk, [], [], ctx) == []
    assert Groth16.verify_batch_locate_compressed(vk, [], [], ctx) == []
    with pytest.raises(V.MalformedVerifyingKey):
        Groth16.verify_batch_locate(vk, [inputs[0] + [1]], proofs[:1], ctx)
    with pytest.raises(ValueError):
        Groth16.verify_batch_locate(vk, inputs, proofs, ctx, weights=[1, 2])
    with pytest.raises(ValueError):
        Groth16.verify_batch_locate_compressed(vk, inputs[:1], [b'\x00' * 127], ctx)
    for bad in (R, -1):
        with pytest.raises(B2gError) as e:
            Groth16.verify_batch_locate(vk, [[bad, 1]] + inputs[1:], proofs, ctx)
        assert e.value.code == -4
    for bad in (0, 1 << 128):
        with pytest.raises(B2gError) as e:
            Groth16.verify_batch_locate(vk, inputs, proofs, ctx, weights=[1, 2, bad, 4, 5])
        assert e.value.code == -4
    L, h = N.lib(), ctx.vk_handle(vk)
    comp = b''.join(_compress(p) for p in proofs[:2])
    for entry, rows in ((L.b2g_verify_batch_locate, proofs[0].data + proofs[1].data), (L.b2g_verify_batch_locate_compressed, comp)):
        buf = (C.c_uint8 * len(rows)).from_buffer_copy(rows)
        pub = (C.c_uint8 * 128).from_buffer_copy(b''.join(int(x).to_bytes(32, 'little') for x in inputs[0] + inputs[1]))
        w = (C.c_uint8 * 32).from_buffer_copy((5).to_bytes(16, 'little') + (7).to_bytes(16, 'little'))
        w0 = (C.c_uint8 * 32).from_buffer_copy((5).to_bytes(16, 'little') + bytes(16))
        pub_r = (C.c_uint8 * 128).from_buffer_copy(R.to_bytes(32, 'little') + bytes(96))
        out = (C.c_uint8 * 2)()
        assert entry(ctx._h, h, 2, pub, buf, w0, out) == -4                      # a zero weight
        assert L.b2g_last_error() == b'weight 1 is zero'
        assert entry(ctx._h, h, 2, pub_r, buf, w, out) == -4                     # an input >= r
        assert L.b2g_last_error() == b'public input 0 of proof 0 is not below the scalar field modulus r'
        assert entry(ctx._h, h, 0, pub, buf, w, out) == -2
        assert L.b2g_last_error() == entry.__name__.encode() + b': count must be at least 1'
        for args in ((ctx._h, h, 0, pub, None, w, out), (ctx._h, h, 2, None, buf, w, out), (ctx._h, h, 2, pub, None, w, out),
                     (ctx._h, h, 2, pub, buf, None, out), (ctx._h, h, 2, pub, buf, w, None), (None, h, 2, pub, buf, w, out),
                     (ctx._h, None, 2, pub, buf, w, out)):
            assert entry(*args) == -2
            assert L.b2g_last_error() == b'null pointer'
        assert entry(ctx._h, h, 2, pub, buf, w, out) == 0 and list(out) == [1, 1]
    # a proof pending on the context
    pk, cm = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    case = g['proofs'][0]
    pending = Groth16.submit(pk, int(case['r']), int(case['s']), cm, fr_to_mont([int(x) for x in g['witness']]), ctx)
    with pytest.raises(B2gError) as e:
        Groth16.verify_batch_locate(vk, inputs, proofs, ctx)
    assert e.value.code == -2
    assert e.value.msg == 'a submitted proof is still pending on this context: call b2g_prove_wait first'
    assert pending.wait().data.hex() == case['proof_hex']
    release(vk); release(pk); release(cm)


def test_interleaved_with_the_other_verifiers(ctx):
    """the new call, verify_many and verify_batch on one context, smaller after larger and larger after smaller, with the
    same answers every time"""
    from circom_compat_b200 import Groth16, release
    vk, inputs, proofs = _synthetic(3, 66, 40)
    n = 300
    xs, ps = [inputs[k % 40] for k in range(n)], [proofs[k % 40] for k in range(n)]
    bad = {2, 150, 299}
    qs = [_neg_a(p) if k in bad else p for k, p in enumerate(ps)]
    want = [k not in bad for k in range(n)]
    for m in (n, 7, 70, n, 1, 130):
        assert Groth16.verify_batch_locate(vk, xs[:m], qs[:m], ctx) == want[:m], m
        assert Groth16.verify_many(vk, xs[:m], qs[:m], ctx) == want[:m], m
        assert Groth16.verify_batch(vk, xs[:m], qs[:m], ctx) == all(want[:m]), m
        assert Groth16.verify_batch(vk, xs[:m], ps[:m], ctx), m
        assert Groth16.verify_batch_locate(vk, xs[:m], ps[:m], ctx) == [True] * m, m
    release(vk)


def test_cpp_mirror_verify_batch_locate(complex_zkey_bytes, golden):
    """Groth16::verify_batch_locate through groth16_bench (B2G_VERIFY_LOCATE=130): proofs 0, 65 and 129 have A negated, and
    the verdicts agree with the C++ host verifier over every proof"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, 'circom_compat_b200', 'host', 'groth16_bench')
    out = subprocess.check_output([exe, os.path.join(root, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'),
                                   'chain:%d' % int(golden['complex_zkey']['a']), '0'], text=True, env=dict(os.environ, B2G_VERIFY_LOCATE='130'))
    line = [l for l in out.splitlines() if l.startswith('verify_locate')][0]
    assert 'verify_locate 130 proofs (127 valid, 3 tampered): agree=1' in line, line
