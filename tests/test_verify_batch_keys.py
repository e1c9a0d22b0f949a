"""b2g_verify_batch_keys / Groth16.verify_batch_keys: the batch check of many keys in one device pass, one verdict per key.
Every verdict is compared with verify_batch on that key's batch with the same weights (the keyed call runs the same equation,
so the two agree bit for bit), and where stated with the per-key big-int model (tests/batch_keys_model.py).  Large key sets
are built with known discrete logs on the device (Context.fixed_base_g1 / g2)."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from batch_keys_model import verify_batch_keys_rlc
from batch_model import outside_b_proof, twist_point_outside_g2
from circom_compat_b200 import verifier as V
from circom_compat_b200 import ethereum as eth
from oracle import pyref as o
from test_verify_batch import _g1, _g2, _prep, _proof, _pts, _shape_key, _tampered, _weights

pytestmark = pytest.mark.gpu

P, R = V.P, o.R_MOD
_RINV = pow(1 << 256, -1, P)


# ---------------------------------------------------------------------------------------------- keys and proofs
def _canon(rows):
    """Montgomery rows of fixed_base_g1 / g2 -> canonical coordinates per row"""
    raw, w = np.ascontiguousarray(rows).tobytes(), rows.shape[1] // 4
    v = [int.from_bytes(raw[i:i + 32], 'little') * _RINV % P for i in range(0, len(raw), 32)]
    return [v[k * w:(k + 1) * w] for k in range(rows.shape[0])]


def _limbs(ks):
    return np.frombuffer(b''.join(k.to_bytes(32, 'little') for k in ks), dtype='<u8').copy()


def _device_keys(ctx, specs, seed):
    """specs = [(n_public, count)]: per spec (vk, inputs, proofs), a key with known discrete logs and `count` valid proofs,
    every point made on the device in one fixed-base call per group"""
    rng = random.Random(seed)
    plan, s1, s2 = [], [], []
    for n_public, count in specs:
        al, be, ga, de = (rng.randrange(1, R) for _ in range(4))
        ic = [rng.randrange(1, R) for _ in range(n_public + 1)]
        rows = []
        for _ in range(count):
            xs = [rng.randrange(R) for _ in range(n_public)]
            a, b = rng.randrange(1, R), rng.randrange(1, R)
            rows.append((xs, a, b, (a * b - al * be - _prep(ic, xs) * ga) * pow(de, -1, R) % R))
        plan.append((n_public, count))
        s1 += [al] + ic + [v for _, a, _, c in rows for v in (a, c)]
        s2 += [be, ga, de] + [b for _, _, b, _ in rows]
        plan[-1] += (rows,)
    g1 = [tuple(p) for p in _canon(ctx.fixed_base_g1(_limbs(s1)))]
    g2 = [((q[0], q[1]), (q[2], q[3])) for q in _canon(ctx.fixed_base_g2(_limbs(s2)))]
    out, i1, i2 = [], 0, 0
    for n_public, count, rows in plan:
        vk = V.VerifyingKey(g1[i1], g2[i2], g2[i2 + 1], g2[i2 + 2], g1[i1 + 1:i1 + 2 + n_public])
        i1 += 2 + n_public
        i2 += 3
        proofs = []
        for _ in rows:
            proofs.append(_proof(g1[i1], g2[i2], g1[i1 + 1]))
            i1 += 2
            i2 += 1
        out.append((vk, [xs for xs, _, _, _ in rows], proofs))
    return out


def _check(ctx, batches, weights=None, seed=0):
    """verify_batch_keys with explicit weights, compared with verify_batch per key with the same weights; returns the verdicts"""
    from circom_compat_b200 import Groth16
    rng = random.Random(seed)
    ws = weights or [_weights(rng, len(prs)) for _, _, prs in batches]
    got = Groth16.verify_batch_keys(batches, ctx, weights=ws)
    assert got == [Groth16.verify_batch(vk, ins, prs, ctx, weights=w) for (vk, ins, prs), w in zip(batches, ws)]
    return got


def _bad_c(p):
    a, b, c = _pts(p)
    return _proof(a, b, o.G1.add(c, o.G1_GEN))


@pytest.fixture(scope='module')
def bench_key(complex_zkey_bytes, golden):
    """the reference's bench key (2^14) and 40 proofs of chain witnesses a, a + 1, ..."""
    from circom_compat_b200 import Context, Groth16, fr_to_mont, read_zkey, release
    pk, cm = read_zkey(complex_zkey_bytes)
    cx = Context(0)
    a0 = int(golden['complex_zkey']['a'])
    rng = random.Random(1101)
    ws = [o.chain_witness(pk.n_vars, a0 + k) for k in range(40)]
    proofs = Groth16.create_proofs(pk, [(rng.randrange(R), rng.randrange(R)) for _ in ws], cm, [fr_to_mont(w) for w in ws], cx)
    release(cm)
    yield pk, [list(w[1:pk.n_public + 1]) for w in ws], proofs
    release(pk)
    cx.close()


@pytest.fixture(scope='module')
def small_keys(ctx):
    """device-made keys with 0, 1, 2, 100 and 129 public inputs, three proofs each"""
    from circom_compat_b200 import release
    keys = _device_keys(ctx, [(0, 3), (1, 3), (2, 3), (100, 3), (129, 3)], 1100)
    yield keys
    for vk, _, _ in keys:
        release(vk)


# ---------------------------------------------------------------------------------------------- valid calls
def test_mixed_keys_in_one_call(ctx, golden, test_zkey_bytes, bench_key, small_keys):
    from circom_compat_b200 import Proof, read_zkey, release
    pk, _ = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    xs = [int(x) for x in g['witness'][1:pk.n_public + 1]]
    golden_proofs = [Proof(bytes.fromhex(c['proof_hex'])) for c in g['proofs']]
    bpk, bins, bprs = bench_key
    batches = [(pk, [xs] * len(golden_proofs), golden_proofs), (bpk, bins[:33], bprs[:33])] + small_keys
    assert _check(ctx, batches, seed=1) == [True] * len(batches)
    release(pk)


def test_segment_shapes(ctx):
    """key sizes around the 64-record product CTA, the 128-record sum CTA, the 2 048-proof scalar chunk and above 4 096 (a
    third product level), next to an empty batch and one key in two batches; then a tampered proof in two of them"""
    from circom_compat_b200 import release
    sizes = [1, 63, 64, 65, 127, 128, 129, 2048, 2049, 4160, 130]
    keys = _device_keys(ctx, [(k % 3, n) for k, n in enumerate(sizes)], 1200)
    twice = keys[-1]
    batches = [k for k in keys[:-1]] + [(twice[0], twice[1][:65], twice[2][:65]), (keys[2][0], [], []),
                                        (twice[0], twice[1][65:], twice[2][65:])]
    assert _check(ctx, batches, seed=2) == [True] * len(batches)
    bad = list(batches)
    vk, ins, prs = bad[9]
    bad[9] = (vk, ins, prs[:-1] + [_bad_c(prs[-1])])                  # the last proof of the 4 160-proof key
    vk, ins, prs = bad[8]
    bad[8] = (vk, ins, [_bad_c(prs[0])] + prs[1:])                    # the first proof of the 2 049-proof key
    vk, ins, prs = bad[12]
    bad[12] = (vk, ins, prs[:-1] + [_bad_c(prs[-1])])                 # the second batch of the key given twice
    want = [True] * len(batches)
    want[8] = want[9] = want[12] = False
    assert _check(ctx, bad, seed=3) == want
    for vk, _, _ in keys:
        release(vk)


def test_a_thousand_keys_of_one_proof(ctx):
    from circom_compat_b200 import Groth16, release
    keys = _device_keys(ctx, [(k % 2, 1) for k in range(1000)], 1300)
    assert Groth16.verify_batch_keys(keys, ctx) == [True] * 1000
    bad = list(keys)
    for k in (0, 517, 999):
        vk, ins, prs = bad[k]
        bad[k] = (vk, ins, [_bad_c(prs[0])])
    assert _check(ctx, bad, seed=4) == [k not in (0, 517, 999) for k in range(1000)]
    for vk, _, _ in keys:
        release(vk)


def test_one_large_key_next_to_many_small_ones(ctx):
    """10 000 proofs of one key next to 300 keys of one to three proofs: the large key's reduction levels run next to the
    small keys' single CTAs"""
    from circom_compat_b200 import Groth16, release
    keys = _device_keys(ctx, [(1, 10000)] + [(k % 3, 1 + k % 3) for k in range(300)], 1400)
    assert Groth16.verify_batch_keys(keys, ctx) == [True] * 301
    bad = list(keys)
    vk, ins, prs = bad[0]
    bad[0] = (vk, ins, prs[:5000] + [_bad_c(prs[5000])] + prs[5001:])
    vk, ins, prs = bad[150]
    bad[150] = (vk, ins, prs[:-1] + [_bad_c(prs[-1])])
    assert _check(ctx, bad, seed=5) == [k not in (0, 150) for k in range(301)]
    for vk, _, _ in keys:
        release(vk)


# ---------------------------------------------------------------------------------------------- independence
def test_one_tampered_proof_changes_only_its_key(ctx, bench_key, small_keys):
    """every tampering kind of test_verify_batch.py, at the first and last proof of a key and in a key of one proof, among
    other keys (the bench key twice, small keys): exactly that key's verdict is False"""
    bpk, bins, bprs = bench_key
    outside = twist_point_outside_g2(random.Random(1500))
    one = small_keys[2]
    batches = [(bpk, bins[:6], bprs[:6]), (one[0], one[1][:1], one[2][:1]), (bpk, bins[6:10], bprs[6:10]), small_keys[1]]
    for kind in range(12):
        for key, pos in ((0, 0), (0, 5), (1, 0), (2, 3)):
            vk, ins, prs = batches[key]
            prev = prs[pos - 1] if len(prs) > 1 else bprs[20]            # kind 1 takes another proof's B
            xs, p = _tampered(kind, ins[pos], prs[pos], prev, outside)
            bad = list(batches)
            bad[key] = (vk, ins[:pos] + [xs] + ins[pos + 1:], prs[:pos] + [p] + prs[pos + 1:])
            assert _check(ctx, bad, seed=kind) == [k != key for k in range(4)], (kind, key, pos)


def test_b_outside_g2_fails_its_own_key(ctx, small_keys):
    """verify_many accepts the outside-G2 proof; the keyed call refuses its key only, and accepts the same key with B in G2"""
    from circom_compat_b200 import Groth16, release
    vk, xs, (a, b, c) = outside_b_proof(1600)
    bad, good = _proof(a, b, c), [_proof(a, _g2(k), c) for k in (3, 5)]
    assert Groth16.verify_many(vk, [xs], [bad], ctx) == [True]
    batches = [small_keys[0], (vk, [xs] * 3, good[:1] + [bad] + good[1:]), (vk, [xs] * 2, good)]
    assert _check(ctx, batches, seed=6) == [True, False, True]
    release(vk)


def test_every_tail_shape_per_key_matches_the_model(ctx):
    """gamma at infinity, delta at infinity, prepared inputs at infinity and sum r C at infinity, each in its own key of one
    call next to a plain key, then with the plain and gamma keys tampered: the device verdicts equal the big-int model"""
    from circom_compat_b200 import release
    rng = random.Random(1700)
    out = []
    vk, L, ic, r2 = _shape_key(11, 1)
    xs = [r2.randrange(R)]
    p = _prep(ic, xs)
    b = r2.randrange(1, R)
    out.append((vk, [xs], [_proof(_g1((L['al'] * L['be'] + p * L['ga']) * pow(b, -1, R) % R), _g2(b), None)]))      # r C = 0
    x0 = (-ic[0]) * pow(ic[1], -1, R) % R
    a, b = r2.randrange(1, R), r2.randrange(1, R)
    out.append((vk, [[x0]], [_proof(_g1(a), _g2(b), _g1((a * b - L['al'] * L['be']) * pow(L['de'], -1, R) % R))]))  # prepared = 0
    vk, L, ic, r2 = _shape_key(12, 1, gamma_inf=True)
    a, b = r2.randrange(1, R), r2.randrange(1, R)
    out.append((vk, [[r2.randrange(R)]], [_proof(_g1(a), _g2(b), _g1((a * b - L['al'] * L['be']) * pow(L['de'], -1, R) % R))]))
    vk, L, ic, r2 = _shape_key(13, 2, delta_inf=True)
    xs = [r2.randrange(R), r2.randrange(R)]
    b = r2.randrange(1, R)
    a = (L['al'] * L['be'] + _prep(ic, xs) * L['ga']) * pow(b, -1, R) % R
    out.append((vk, [xs], [_proof(_g1(a), _g2(b), _g1(r2.randrange(1, R)))]))
    vk, L, ic, r2 = _shape_key(14, 1)
    xs = [[r2.randrange(R)] for _ in range(2)]
    prs = []
    for x in xs:
        a, b = r2.randrange(1, R), r2.randrange(1, R)
        prs.append(_proof(_g1(a), _g2(b), _g1((a * b - L['al'] * L['be'] - _prep(ic, x) * L['ga']) * pow(L['de'], -1, R) % R)))
    out.append((vk, xs, prs))
    weights = [_weights(rng, len(p)) for _, _, p in out]
    pvks = [V.prepare_verifying_key(vk) for vk, _, _ in out]
    model = lambda bs: verify_batch_keys_rlc([(pvk, ins, prs) for pvk, (_, ins, prs) in zip(pvks, bs)], weights)
    assert _check(ctx, out, weights) == model(out) == [True] * 5
    bad = list(out)
    for k in (2, 4):
        vk, ins, prs = bad[k]
        bad[k] = (vk, ins, prs[:-1] + [_bad_c(prs[-1])])
    assert _check(ctx, bad, weights) == model(bad) == [True, True, False, True, False]
    for vk, _, _ in out[1:]:
        release(vk)


def test_weights_scale_their_own_proof_inside_one_key(ctx, small_keys):
    """C_3 + w_7 D and C_7 - w_3 D cancel in key 1's sum w_i C_i for exactly these weights: accepted with them, refused with
    fresh ones, and the other keys are unaffected"""
    from circom_compat_b200 import Groth16, release
    keys = _device_keys(ctx, [(2, 10)], 1800)
    vk, ins, prs = keys[0]
    rng = random.Random(1800)
    w = _weights(rng, 10)
    d = _g1(rng.randrange(1, R))
    (ai, bi, ci), (aj, bj, cj) = _pts(prs[3]), _pts(prs[7])
    bad = list(prs)
    bad[3] = _proof(ai, bi, o.G1.add(ci, o.G1.mul(d, w[7])))
    bad[7] = _proof(aj, bj, o.G1.add(cj, o.G1.neg(o.G1.mul(d, w[3]))))
    batches = [small_keys[1], (vk, ins, bad), small_keys[0]]
    others = [_weights(rng, 3), None, _weights(rng, 3)]
    assert _check(ctx, batches, [others[0], w, others[2]]) == [True, True, True]
    assert Groth16.verify_batch_keys(batches, ctx, weights=others) == [True, False, True]       # fresh weights for key 1
    swapped = list(w)
    swapped[3], swapped[7] = w[7], w[3]
    assert _check(ctx, batches, [others[0], swapped, others[2]]) == [True, False, True]
    release(vk)


# ---------------------------------------------------------------------------------------------- compressed proofs
def test_compressed_equals_decompress_then_keys(ctx, bench_key, small_keys):
    """verify_batch_keys_compressed equals decompress_proofs followed by verify_batch_keys, with a sign-flipped blob (it
    decodes to -A) and an undecodable blob (both flags set) in two of the keys"""
    from circom_compat_b200 import Groth16
    bpk, bins, bprs = bench_key
    batches = [(bpk, bins[:8], bprs[:8]), small_keys[3], small_keys[0], (bpk, bins[8:12], bprs[8:12])]
    blobs = [[eth.serialize_compressed(eth.Proof.from_proof(p)) for p in prs] for _, _, prs in batches]
    flipped = bytearray(blobs[0][2]); flipped[31] ^= 0x80
    blobs[0][2] = bytes(flipped)
    broken = bytearray(blobs[2][1]); broken[31] |= 0xC0
    blobs[2][1] = bytes(broken)
    rng = random.Random(1900)
    ws = [_weights(rng, len(b)) for b in blobs]
    got = Groth16.verify_batch_keys_compressed([(vk, ins, bl) for (vk, ins, _), bl in zip(batches, blobs)], ctx, weights=ws)
    decoded = [Groth16.decompress_proofs(bl, ctx) for bl in blobs]
    assert decoded[2][1] is None and all(p is not None for p in decoded[0])
    want = [False if any(p is None for p in dec) else None for dec in decoded]
    keyed = Groth16.verify_batch_keys([(vk, [x for x, p in zip(ins, dec) if p is not None], [p for p in dec if p is not None])
                                       for (vk, ins, _), dec in zip(batches, decoded)],
                                      ctx, weights=[[w for w, p in zip(wk, dec) if p is not None] for wk, dec in zip(ws, decoded)])
    want = [k if v is None else v for v, k in zip(want, keyed)]
    assert got == want == [False, True, False, True]


# ---------------------------------------------------------------------------------------------- errors and reuse
def test_errors_leave_the_context_usable(ctx, golden, test_zkey_bytes, small_keys):
    from circom_compat_b200 import B2gError, Groth16, fr_to_mont, read_zkey, release
    from circom_compat_b200 import _native as N
    vk, ins, prs = small_keys[2]
    assert Groth16.verify_batch_keys([], ctx) == []
    assert Groth16.verify_batch_keys([(vk, [], []), (vk, [], [])], ctx) == [True, True]
    with pytest.raises(V.MalformedVerifyingKey, match='key 1'):
        Groth16.verify_batch_keys([small_keys[2], (vk, [ins[0] + [1]], prs[:1])], ctx)
    with pytest.raises(ValueError, match='key 0'):
        Groth16.verify_batch_keys([(vk, ins, prs[:2])], ctx)
    with pytest.raises(ValueError):
        Groth16.verify_batch_keys([small_keys[2]], ctx, weights=[[1, 2, 3], [4]])
    with pytest.raises(B2gError, match='key 1') as e:
        Groth16.verify_batch_keys([small_keys[2], (vk, [[R, 1]] + ins[1:], prs)], ctx)
    assert e.value.code == -4
    with pytest.raises(B2gError, match='key 0') as e:
        Groth16.verify_batch_keys([small_keys[2]], ctx, weights=[[1, 0, 3]])
    assert e.value.code == -4
    # the C ABI
    L, h = N.lib(), ctx.vk_handle(vk)
    pub = np.frombuffer(b''.join(int(x).to_bytes(32, 'little') for xs in ins for x in xs), dtype=np.uint8).copy()
    pub_r = pub.copy(); pub_r[64:96] = np.frombuffer(R.to_bytes(32, 'little'), dtype=np.uint8)
    rows = np.frombuffer(b''.join(p.data for p in prs), dtype=np.uint8).copy()
    w = np.frombuffer(b''.join(k.to_bytes(16, 'little') for k in (5, 6, 7)), dtype=np.uint8).copy()
    w0 = w.copy(); w0[16:32] = 0
    ptr = lambda a: a.ctypes.data

    def table(*entries):
        return (N.KeyBatch * len(entries))(*[N.KeyBatch(hh and hh.value, n, 0, pb, pr, ww) for hh, n, pb, pr, ww in entries])

    ok = (h, 3, ptr(pub), ptr(rows), ptr(w))
    out = (C.c_uint8 * 2)()
    assert L.b2g_verify_batch_keys(ctx._h, 2, table(ok, ok), out) == 0 and list(out) == [1, 1]
    assert L.b2g_verify_batch_keys(ctx._h, 0, table(ok), out) == -2                                   # no keys
    assert L.b2g_verify_batch_keys(ctx._h, 2, table((h, 0, None, None, None), (h, 0, None, None, None)), out) == -2   # no proofs
    for bad in ((h, 3, None, ptr(rows), ptr(w)), (h, 3, ptr(pub), None, ptr(w)), (h, 3, ptr(pub), ptr(rows), None), (None, 3, ptr(pub), ptr(rows), ptr(w))):
        assert L.b2g_verify_batch_keys(ctx._h, 2, table(ok, bad), out) == -2
        assert b'key 1' in L.b2g_last_error()
    assert L.b2g_verify_batch_keys(ctx._h, 2, None, out) == -2
    assert L.b2g_verify_batch_keys(ctx._h, 2, table(ok, ok), None) == -2
    assert L.b2g_verify_batch_keys(ctx._h, 2, table(ok, (h, 3, ptr(pub), ptr(rows), ptr(w0))), out) == -4
    assert b'key 1: weight 1 is zero' in L.b2g_last_error()
    assert L.b2g_verify_batch_keys(ctx._h, 2, table((h, 3, ptr(pub_r), ptr(rows), ptr(w)), ok), out) == -4
    assert b'key 0: public input 0 of proof 1' in L.b2g_last_error()
    out[0] = out[1] = 0
    assert L.b2g_verify_batch_keys(ctx._h, 2, table((h, 0, None, None, None), ok), out) == 0 and list(out) == [1, 1]
    # a proof pending on the context
    pk, cm = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    case = g['proofs'][0]
    pending = Groth16.submit(pk, int(case['r']), int(case['s']), cm, fr_to_mont([int(x) for x in g['witness']]), ctx)
    with pytest.raises(B2gError) as e:
        Groth16.verify_batch_keys([small_keys[2]], ctx)
    assert e.value.code == -2
    assert pending.wait().data.hex() == case['proof_hex']
    release(pk); release(cm)


def test_interleaved_with_the_other_verifiers(ctx, small_keys):
    """the keyed call next to verify_many, verify_batch and verify_batch_locate on one context, growing and shrinking"""
    from circom_compat_b200 import Groth16, release
    big = _device_keys(ctx, [(1, 200), (2, 70)], 2000)
    (vk, ins, prs), (vk2, ins2, prs2) = big
    for n in (200, 3, 130, 1):
        keyed = [(vk, ins[:n], prs[:n]), (vk2, ins2[:min(n, 70)], prs2[:min(n, 70)]), small_keys[4]]
        assert Groth16.verify_batch_keys(keyed, ctx) == [True] * 3
        assert Groth16.verify_many(vk, ins[:n], prs[:n], ctx) == [True] * n
        assert Groth16.verify_batch(vk2, ins2[:min(n, 70)], prs2[:min(n, 70)], ctx)
        bad = prs[:n - 1] + [_bad_c(prs[n - 1])]
        assert Groth16.verify_batch_locate(vk, ins[:n], bad, ctx) == [True] * (n - 1) + [False]
        assert Groth16.verify_batch_keys([(vk, ins[:n], bad)] + keyed[1:], ctx) == [False, True, True]
    for k, _, _ in big:
        release(k)


def test_cpp_mirror_verify_batch_keys(complex_zkey_bytes, golden):
    """Groth16::verify_batch_keys through groth16_bench (B2G_VERIFY_KEYS=9): nine proofs in four batches of the bench key and
    an empty one, the second batch tampered; the verdicts equal the C++ host verifier's per batch"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, 'circom_compat_b200', 'host', 'groth16_bench')
    out = subprocess.check_output([exe, os.path.join(root, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'),
                                   'chain:%d' % int(golden['complex_zkey']['a']), '0'], text=True, env=dict(os.environ, B2G_VERIFY_KEYS='9'))
    line = [l for l in out.splitlines() if l.startswith('verify_keys')][0]
    assert 'verify_keys 9 proofs in 5 batches: device=10111 host=10111 agree=1' in line, line
