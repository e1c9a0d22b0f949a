"""b2g_verify_batch_keys_locate / Groth16.verify_batch_keys_locate: verify_batch_locate for many keys in one device pass, one
verdict per proof.  Every call is compared with verify_batch_locate on each batch alone with the same weights (the keyed call
runs the same groups and the same second pass, so the two agree bit for bit), and where stated with locate_model or with
verify_many AND the G2 membership of B.  Keys with known discrete logs come from _device_keys."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from batch_model import outside_b_proof, twist_point_outside_g2
from circom_compat_b200 import verifier as V
from circom_compat_b200 import ethereum as eth
from oracle import pyref as o
from test_verify_batch import _g2, _proof, _pts, _tampered, _weights
from test_verify_batch_keys import _bad_c, _device_keys, bench_key, small_keys  # noqa: F401
from test_verify_batch_locate import _cancelling_pair, _expected, _neg_a, locate_model

pytestmark = pytest.mark.gpu

P, R = V.P, o.R_MOD
GROUP = 64


def _check(ctx, batches, weights=None, seed=0, model=()):
    """verify_batch_keys_locate with explicit weights, compared with verify_batch_locate per batch with the same weights,
    and for the batches listed in `model` with locate_model; returns the verdicts"""
    from circom_compat_b200 import Groth16
    rng = random.Random(seed)
    ws = weights or [_weights(rng, len(prs)) for _, _, prs in batches]
    got = Groth16.verify_batch_keys_locate(batches, ctx, weights=ws)
    assert got == [Groth16.verify_batch_locate(vk, ins, prs, ctx, weights=w) for (vk, ins, prs), w in zip(batches, ws)]
    for k in model:
        vk, ins, prs = batches[k]
        assert got[k] == locate_model(Groth16.process_vk(vk), ins, prs, ws[k]), k
    return got


def _with(batch, pos, proof):
    vk, ins, prs = batch
    return vk, ins, prs[:pos] + [proof] + prs[pos + 1:]


def _release(keys):
    from circom_compat_b200 import release
    for vk, _, _ in keys:
        release(vk)


# ---------------------------------------------------------------------------------------------- valid and invalid calls
def test_mixed_keys_in_one_call(ctx, golden, test_zkey_bytes, bench_key, small_keys):
    """test.zkey's golden proofs, the 2^14 bench key and keys of 0 to 129 inputs in one call: all valid, then one bad proof
    in three of them; the verdicts of the golden and synthetic keys also equal the big-int model"""
    from circom_compat_b200 import Proof, read_zkey, release
    pk, _ = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    xs = [int(x) for x in g['witness'][1:pk.n_public + 1]]
    golden_proofs = [Proof(bytes.fromhex(c['proof_hex'])) for c in g['proofs']]
    bpk, bins, bprs = bench_key
    batches = [(pk, [xs] * len(golden_proofs), golden_proofs), (bpk, bins[:33], bprs[:33])] + small_keys
    assert _check(ctx, batches, seed=1) == [[True] * len(b[2]) for b in batches]
    bad = list(batches)
    bad[0] = _with(bad[0], 0, _neg_a(golden_proofs[0]))
    bad[1] = _with(bad[1], 32, _bad_c(bprs[32]))
    bad[6] = _with(bad[6], 1, _bad_c(small_keys[4][2][1]))          # the 129-input key
    want = [[True] * len(b[2]) for b in batches]
    want[0][0] = want[1][32] = want[6][1] = False
    assert _check(ctx, bad, seed=2, model=(0, 2, 3, 4, 5, 6)) == want
    release(pk)


def test_groups_restart_at_every_key(ctx):
    """batches of 1, 63, 64, 65 and 129 proofs side by side, then a tampered proof at the first and last position of every
    group of every key: only those proofs are False, so each key's groups start at its first proof"""
    sizes = [1, 63, 64, 65, 129]
    keys = _device_keys(ctx, [(k % 3, n) for k, n in enumerate(sizes)], 2100)
    assert _check(ctx, keys, seed=3) == [[True] * n for n in sizes]
    bad, want = [], []
    for (vk, ins, prs), n in zip(keys, sizes):
        edges = {e for g in range(0, n, GROUP) for e in (g, min(g + GROUP, n) - 1)}
        bad.append((vk, ins, [_bad_c(p) if i in edges else p for i, p in enumerate(prs)]))
        want.append([i not in edges for i in range(n)])
    assert _check(ctx, bad, seed=4) == want
    _release(keys)


def test_every_tampering_kind(ctx, bench_key, small_keys):
    """every tampering kind of test_verify_batch.py at the first and last proof of a key and in a key of one proof, among
    other keys: exactly that proof is False, and a malformed proof leaves its group's other verdicts True"""
    bpk, bins, bprs = bench_key
    outside = twist_point_outside_g2(random.Random(2200))
    one = small_keys[2]
    batches = [(bpk, bins[:6], bprs[:6]), (one[0], one[1][:1], one[2][:1]), (bpk, bins[6:10], bprs[6:10]), small_keys[1]]
    for kind in range(12):
        for key, pos in ((0, 0), (0, 5), (1, 0), (2, 3)):
            vk, ins, prs = batches[key]
            prev = prs[pos - 1] if len(prs) > 1 else bprs[20]            # kind 1 takes another proof's B
            xs, p = _tampered(kind, ins[pos], prs[pos], prev, outside)
            bad = list(batches)
            bad[key] = (vk, ins[:pos] + [xs] + ins[pos + 1:], prs[:pos] + [p] + prs[pos + 1:])
            want = [[not (k == key and i == pos) for i in range(len(b[2]))] for k, b in enumerate(batches)]
            assert _check(ctx, bad, seed=kind) == want, (kind, key, pos)


def test_b_outside_g2(ctx, small_keys):
    """verify_many accepts the outside-G2 proof; the keyed call refuses that proof only, in its group and next to other keys"""
    from circom_compat_b200 import Groth16, release
    vk, xs, (a, b, c) = outside_b_proof(2300)
    bad, good = _proof(a, b, c), [_proof(a, _g2(k), c) for k in range(3, 9)]
    assert Groth16.verify_many(vk, [xs], [bad], ctx) == [True]
    batches = [small_keys[0], (vk, [xs] * 4, good[:2] + [bad] + good[2:3]), (vk, [xs] * 3, good[3:])]
    assert _check(ctx, batches, seed=5) == [[True] * 3, [True, True, False, True], [True] * 3]
    release(vk)


def test_one_invalid_proof_in_every_group(ctx):
    """one invalid proof in every group of every key, with keys of 0 and 129 inputs next to each other: every group fails,
    every well-formed proof goes through the keyed second pass, and the verdicts equal verify_many AND B in G2 per key"""
    keys = _device_keys(ctx, [(0, 130), (129, 70), (1, 64), (2, 1)], 2400)
    rng = random.Random(2400)
    bad, want = [], []
    for vk, ins, prs in keys:
        n = len(prs)
        picks = {g + rng.randrange(min(GROUP, n - g)) for g in range(0, n, GROUP)}
        qs = [_neg_a(p) if i in picks else p for i, p in enumerate(prs)]
        bad.append((vk, ins, qs))
        want.append([i not in picks for i in range(n)])
    got = _check(ctx, bad, seed=6)
    assert got == want
    assert got == [_expected(ctx, vk, ins, prs) for vk, ins, prs in bad]
    _release(keys)


# ---------------------------------------------------------------------------------------------- launches and shapes
def test_launch_count_does_not_follow_the_keys(ctx):
    """1 000 one-proof keys, each proof invalid: the verdicts are right, and the call issues as many launches as a one-key
    call with a failing group and as a call of 10 such keys"""
    from circom_compat_b200 import Groth16
    keys = _device_keys(ctx, [(1 - k % 2, 1) for k in range(1000)], 2500)
    bad = [(vk, ins, [_neg_a(prs[0])]) for vk, ins, prs in keys]

    def delta(fn):
        fn()                                                            # loads the keys on the device
        before = ctx.launch_count()
        out = fn()
        return ctx.launch_count() - before, out

    d_many, got = delta(lambda: Groth16.verify_batch_keys_locate(bad, ctx))
    assert got == [[False]] * 1000
    d_ten, got = delta(lambda: Groth16.verify_batch_keys_locate(bad[:10], ctx))
    assert got == [[False]] * 10
    vk, ins, prs = bad[0]
    d_one, got = delta(lambda: Groth16.verify_batch_locate(vk, ins, prs, ctx))
    assert got == [False]
    assert d_many == d_ten == d_one, (d_many, d_ten, d_one)
    _release(keys)


def test_same_key_twice_empty_batches_and_a_large_key(ctx):
    """10 000 proofs of one key next to 300 small keys, with empty batches between full ones and one key in two batches"""
    keys = _device_keys(ctx, [(1, 10000)] + [(k % 3, 1 + k % 3) for k in range(300)], 2600)
    big_vk, big_ins, big_prs = keys[0]
    batches = [(big_vk, big_ins[:9000], big_prs[:9000]), (keys[5][0], [], [])] + keys[1:151] + \
              [(keys[7][0], [], []), (big_vk, big_ins[9000:], big_prs[9000:])] + keys[151:]
    got = _check(ctx, batches, seed=7)
    assert got == [[True] * len(b[2]) for b in batches]
    bad = list(batches)
    bad[0] = _with(bad[0], 5000, _neg_a(big_prs[5000]))
    assert batches[153][2] == big_prs[9000:]
    bad[153] = _with(bad[153], 999, _neg_a(big_prs[9999]))           # the large key's second batch
    vk, ins, prs = bad[100]
    bad[100] = (vk, ins, [_bad_c(p) for p in prs])
    want = [[True] * len(b[2]) for b in batches]
    want[0][5000] = want[153][999] = False
    want[100] = [False] * len(want[100])
    assert _check(ctx, bad, seed=8) == want
    _release(keys)


def test_weights_cancel_across_batches_but_not_in_the_keyed_call(ctx):
    """proofs i and j of one key in two batches, made invalid so that their errors cancel for the chosen weights: verify_batch
    over both batches together accepts them, but each gets its own batch's verdict in the keyed call"""
    from circom_compat_b200 import Groth16, release
    keys = _device_keys(ctx, [(2, 100)], 2700)
    vk, ins, prs = keys[0]
    rng = random.Random(2700)
    w = _weights(rng, 100)
    bad = _cancelling_pair(vk, ins, prs, 10, 80, w, rng)
    assert Groth16.verify_batch(vk, ins, bad, ctx, weights=w)
    batches = [(vk, ins[:50], bad[:50]), keys[0][:1] + (ins[50:], bad[50:])]
    want = [[k != 10 for k in range(50)], [k != 30 for k in range(50)]]
    assert _check(ctx, batches, [w[:50], w[50:]]) == want
    release(vk)


# ---------------------------------------------------------------------------------------------- compressed proofs
def test_compressed_equals_decompress_then_keyed_locate(ctx, bench_key, small_keys):
    """verify_batch_keys_locate_compressed equals decompress_proofs followed by verify_batch_keys_locate on the decoded rows
    (an undecodable blob as the 0xFF row), with a sign-flipped blob (it decodes to -A) and an undecodable blob"""
    from circom_compat_b200 import Groth16, Proof
    bpk, bins, bprs = bench_key
    batches = [(bpk, bins[:8], bprs[:8]), small_keys[3], small_keys[0], (bpk, bins[8:12], bprs[8:12])]
    blobs = [[eth.serialize_compressed(eth.Proof.from_proof(p)) for p in prs] for _, _, prs in batches]
    flipped = bytearray(blobs[0][2]); flipped[31] ^= 0x80
    blobs[0][2] = bytes(flipped)
    broken = bytearray(blobs[2][1]); broken[31] |= 0xC0
    blobs[2][1] = bytes(broken)
    rng = random.Random(2800)
    ws = [_weights(rng, len(b)) for b in blobs]
    comp = [(vk, ins, bl) for (vk, ins, _), bl in zip(batches, blobs)]
    got = Groth16.verify_batch_keys_locate_compressed(comp, ctx, weights=ws)
    assert got == [Groth16.verify_batch_locate_compressed(vk, ins, bl, ctx, weights=w) for (vk, ins, bl), w in zip(comp, ws)]
    decoded = [Groth16.decompress_proofs(bl, ctx) for bl in blobs]
    assert decoded[2][1] is None
    rows = [[d if d is not None else Proof(b'\xff' * 256) for d in dec] for dec in decoded]
    assert got == Groth16.verify_batch_keys_locate([(vk, ins, r) for (vk, ins, _), r in zip(batches, rows)], ctx, weights=ws)
    want = [[True] * len(b) for b in blobs]
    want[0][2] = want[2][1] = False
    assert got == want


# ---------------------------------------------------------------------------------------------- errors and reuse
def test_errors_leave_the_context_usable(ctx, golden, test_zkey_bytes, small_keys):
    from circom_compat_b200 import B2gError, Groth16, fr_to_mont, read_zkey, release
    from circom_compat_b200 import _native as N
    vk, ins, prs = small_keys[2]
    assert Groth16.verify_batch_keys_locate([], ctx) == []
    assert Groth16.verify_batch_keys_locate([(vk, [], []), (vk, [], [])], ctx) == [[], []]
    with pytest.raises(V.MalformedVerifyingKey, match='key 1'):
        Groth16.verify_batch_keys_locate([small_keys[2], (vk, [ins[0] + [1]], prs[:1])], ctx)
    with pytest.raises(ValueError, match='key 0'):
        Groth16.verify_batch_keys_locate([(vk, ins, prs[:2])], ctx)
    with pytest.raises(ValueError):
        Groth16.verify_batch_keys_locate([small_keys[2]], ctx, weights=[[1, 2, 3], [4]])
    with pytest.raises(ValueError):
        Groth16.verify_batch_keys_locate_compressed([(vk, ins[:1], [b'\x00' * 127])], ctx)
    with pytest.raises(B2gError, match='key 1') as e:
        Groth16.verify_batch_keys_locate([small_keys[2], (vk, [[R, 1]] + ins[1:], prs)], ctx)
    assert e.value.code == -4
    with pytest.raises(B2gError, match='key 0') as e:
        Groth16.verify_batch_keys_locate([small_keys[2]], ctx, weights=[[1, 0, 3]])
    assert e.value.code == -4
    # the C ABI, both forms
    L, h = N.lib(), ctx.vk_handle(vk)
    pub = np.frombuffer(b''.join(int(x).to_bytes(32, 'little') for xs in ins for x in xs), dtype=np.uint8).copy()
    pub_r = pub.copy(); pub_r[64:96] = np.frombuffer(R.to_bytes(32, 'little'), dtype=np.uint8)
    full = np.frombuffer(b''.join(p.data for p in prs), dtype=np.uint8).copy()
    comp = np.frombuffer(b''.join(eth.serialize_compressed(eth.Proof.from_proof(p)) for p in prs), dtype=np.uint8).copy()
    w = np.frombuffer(b''.join(k.to_bytes(16, 'little') for k in (5, 6, 7)), dtype=np.uint8).copy()
    w0 = w.copy(); w0[16:32] = 0
    ptr = lambda a: a.ctypes.data

    def table(*entries):
        return (N.KeyBatch * len(entries))(*[N.KeyBatch(hh and hh.value, n, 0, pb, pr, ww) for hh, n, pb, pr, ww in entries])

    for entry, rows in ((L.b2g_verify_batch_keys_locate, full), (L.b2g_verify_batch_keys_locate_compressed, comp)):
        ok = (h, 3, ptr(pub), ptr(rows), ptr(w))
        out = (C.c_uint8 * 6)()
        assert entry(ctx._h, 2, table(ok, ok), out) == 0 and list(out) == [1] * 6
        assert entry(ctx._h, 0, table(ok), out) == -2                                             # no keys
        assert entry(ctx._h, 2, table((h, 0, None, None, None), (h, 0, None, None, None)), out) == -2   # no proofs
        for bad in ((h, 3, None, ptr(rows), ptr(w)), (h, 3, ptr(pub), None, ptr(w)), (h, 3, ptr(pub), ptr(rows), None),
                    (None, 3, ptr(pub), ptr(rows), ptr(w))):
            assert entry(ctx._h, 2, table(ok, bad), out) == -2
            assert b'key 1' in L.b2g_last_error()
        assert entry(ctx._h, 2, None, out) == -2
        assert entry(ctx._h, 2, table(ok, ok), None) == -2
        assert entry(None, 2, table(ok, ok), out) == -2
        assert entry(ctx._h, 2, table(ok, (h, 3, ptr(pub), ptr(rows), ptr(w0))), out) == -4
        assert b'key 1: weight 1 is zero' in L.b2g_last_error()
        assert entry(ctx._h, 2, table((h, 3, ptr(pub_r), ptr(rows), ptr(w)), ok), out) == -4
        assert b'key 0: public input 0 of proof 1' in L.b2g_last_error()
        out = (C.c_uint8 * 6)()
        assert entry(ctx._h, 3, table((h, 0, None, None, None), ok, (h, 0, None, None, None)), out) == 0
        assert list(out) == [1, 1, 1, 0, 0, 0]                                                    # three bytes written
    # a proof pending on the context
    pk, cm = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    case = g['proofs'][0]
    pending = Groth16.submit(pk, int(case['r']), int(case['s']), cm, fr_to_mont([int(x) for x in g['witness']]), ctx)
    with pytest.raises(B2gError) as e:
        Groth16.verify_batch_keys_locate([small_keys[2]], ctx)
    assert e.value.code == -2
    assert pending.wait().data.hex() == case['proof_hex']
    assert Groth16.verify_batch_keys_locate([small_keys[2]], ctx) == [[True] * 3]
    release(pk); release(cm)


def test_interleaved_with_the_other_verifiers(ctx, small_keys):
    """the keyed locate call next to verify_many, verify_batch_keys and verify_batch_locate on one context, growing and
    shrinking"""
    from circom_compat_b200 import Groth16
    big = _device_keys(ctx, [(1, 200), (2, 70)], 2900)
    (vk, ins, prs), (vk2, ins2, prs2) = big
    for n in (200, 3, 130, 1):
        m = min(n, 70)
        bad = prs[:n - 1] + [_neg_a(prs[n - 1])]
        keyed = [(vk, ins[:n], bad), (vk2, ins2[:m], prs2[:m]), small_keys[4]]
        want = [[True] * (n - 1) + [False], [True] * m, [True] * 3]
        assert Groth16.verify_batch_keys_locate(keyed, ctx) == want
        assert Groth16.verify_many(vk, ins[:n], bad, ctx) == want[0]
        assert Groth16.verify_batch_keys(keyed, ctx) == [False, True, True]
        assert Groth16.verify_batch_locate(vk2, ins2[:m], prs2[:m], ctx) == want[1]
        assert Groth16.verify_batch_keys_locate(keyed[1:], ctx) == want[1:]
    _release(big)


def test_cpp_mirror_verify_batch_keys_locate(complex_zkey_bytes, golden):
    """Groth16::verify_batch_keys_locate through groth16_bench (B2G_VERIFY_KEYS_LOCATE=300): four batches of 75 proofs of the
    bench key and an empty one, A negated at group edges and batch ends; every verdict equals the C++ host verifier's"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, 'circom_compat_b200', 'host', 'groth16_bench')
    out = subprocess.check_output([exe, os.path.join(root, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'),
                                   'chain:%d' % int(golden['complex_zkey']['a']), '0'], text=True,
                                  env=dict(os.environ, B2G_VERIFY_KEYS_LOCATE='300'))
    line = [l for l in out.splitlines() if l.startswith('verify_keys_locate')][0]
    assert 'verify_keys_locate 300 proofs in 5 batches (288 valid, 12 tampered): agree=1' in line, line
