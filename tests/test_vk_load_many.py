"""b2g_vk_load_many / Groth16.load_verifying_keys: many verifying keys prepared on the device in one pass.  A batch-loaded
handle must hold what b2g_vk_load builds for the same key: the tests compare e(alpha, beta) byte for byte and the verifiers'
and the rerandomizer's results under both handles, with the host verifier as the reference for every verdict.  They also
cover the handles' shared allocation, the errors, the launch count and the keyed verifiers' single load call."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from circom_compat_b200 import _native as N
from circom_compat_b200 import verifier as V
from oracle import pyref as o
from test_verify_batch import _g1, _g2, _proof, _pts, _weights
from test_verify_batch_keys import _device_keys

P, R = V.P, o.R_MOD
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------- raw C ABI helpers
def _descs(vks):
    """b2g_vk_desc rows of the keys, and the arrays they point into"""
    from circom_compat_b200.groth16 import _vk_desc
    pairs = [_vk_desc(vk) for vk in vks]
    return (N.VkDesc * len(vks))(*[d for d, _ in pairs]), pairs


def _load_many(ctx, vks):
    descs, keep = _descs(vks)
    out = (C.c_void_p * len(vks))()
    assert N.lib().b2g_vk_load_many(ctx._h, len(vks), descs, out) == 0, N.lib().b2g_last_error()
    return [C.c_void_p(h) for h in out]


def _load_one(ctx, vk):
    descs, keep = _descs([vk])
    h = C.c_void_p()
    assert N.lib().b2g_vk_load(ctx._h, descs, C.byref(h)) == 0, N.lib().b2g_last_error()
    return h


def _free(hs):
    for h in hs:
        assert N.lib().b2g_vk_free(h) == 0


def _arr(data):
    return np.frombuffer(data, dtype=np.uint8).copy() if data else None


def _ptr(a):
    return a.ctypes.data if a is not None else None


def _pub(ins):
    return _arr(b''.join(int(x).to_bytes(32, 'little') for xs in ins for x in xs))


def _rows(prs):
    return _arr(b''.join(p.data for p in prs))


def _wbytes(ws):
    return _arr(b''.join(w.to_bytes(16, 'little') for w in ws))


def _alpha_beta(h):
    out = np.zeros(384, dtype=np.uint8)
    assert N.lib().b2g_vk_alpha_beta(h, out.ctypes.data) == 0
    return out.tobytes()


def _verify_many(ctx, h, ins, prs):
    out, pub, rows = np.zeros(len(prs), dtype=np.uint8), _pub(ins), _rows(prs)
    assert N.lib().b2g_verify_many(ctx._h, h, len(prs), _ptr(pub), _ptr(rows), out.ctypes.data) == 0
    return [bool(v) for v in out]


def _keys_call(ctx, entry, batches, ws):
    """b2g_verify_batch_keys (one verdict per batch) or b2g_verify_batch_keys_locate (one per proof) over [(handle, ins, prs)]"""
    keep = [(_pub(ins), _rows(prs), _wbytes(w)) for (_, ins, prs), w in zip(batches, ws)]
    table = (N.KeyBatch * len(batches))(*[N.KeyBatch(h.value, len(prs), 0, _ptr(pb), _ptr(rw), _ptr(wb))
                                           for (h, _, prs), (pb, rw, wb) in zip(batches, keep)])
    n = len(batches) if entry == 'b2g_verify_batch_keys' else sum(len(prs) for _, _, prs in batches)
    out = np.zeros(n, dtype=np.uint8)
    assert getattr(N.lib(), entry)(ctx._h, len(batches), table, out.ctypes.data) == 0, N.lib().b2g_last_error()
    return [bool(v) for v in out]


def _rerandomize(ctx, h, prs, r1s, r2s):
    rows, out, ok = _rows(prs), np.zeros(256 * len(prs), dtype=np.uint8), np.zeros(len(prs), dtype=np.uint8)
    f1, f2 = _arr(b''.join(r.to_bytes(32, 'little') for r in r1s)), _arr(b''.join(r.to_bytes(32, 'little') for r in r2s))
    assert N.lib().b2g_rerandomize_many(ctx._h, h, len(prs), _ptr(rows), _ptr(f1), _ptr(f2), out.ctypes.data, ok.ctypes.data) == 0
    return out.tobytes(), ok.tobytes()


# ---------------------------------------------------------------------------------------------- keys and proofs
def _key(seed, n_public, alpha_inf=False, gamma_inf=False, delta_inf=False):
    """a key with known discrete logs (a point at infinity has log 0) and three proofs: valid, A negated, a wrong input (C
    moved when there is no input)"""
    rng = random.Random(seed)
    al, be, ga, de = (rng.randrange(1, R) for _ in range(4))
    al, ga, de = 0 if alpha_inf else al, 0 if gamma_inf else ga, 0 if delta_inf else de
    ic = [rng.randrange(1, R) for _ in range(n_public + 1)]
    vk = V.VerifyingKey(_g1(al) if al else None, _g2(be), _g2(ga) if ga else None, _g2(de) if de else None, [_g1(k) for k in ic])
    ins, prs = [], []
    for j in range(3):
        xs = [rng.randrange(R) for _ in range(n_public)]
        prep = (ic[0] + sum(x * k for x, k in zip(xs, ic[1:]))) % R
        b = rng.randrange(1, R)
        if de:
            a = rng.randrange(1, R)
            c = (a * b - al * be - prep * ga) * pow(de, -1, R) % R
        else:
            c = rng.randrange(1, R)
            a = (al * be + prep * ga) * pow(b, -1, R) % R
        if j == 1:
            a = R - a
        ins.append(list(xs))
        prs.append(_proof(_g1(a) if a else None, _g2(b), _g1(c) if c else None))
        if j == 2:
            if n_public:
                ins[-1][0] = (xs[0] + 1) % R
            else:
                prs[-1] = _proof(_g1(a) if a else None, _g2(b), o.G1.add(_g1(c), o.G1_GEN))
    return vk, ins, prs


@pytest.fixture(scope='module')
def mixed_keys(golden, test_zkey_bytes):
    """n_public 0, 1, 2, 5 and 100; gamma, delta, both and alpha at infinity; test.zkey's key.  Each with its proofs and the
    host verifier's verdicts."""
    from circom_compat_b200 import Proof, read_zkey
    keys = [_key(10, 0), _key(11, 1), _key(12, 2), _key(13, 5), _key(14, 100), _key(15, 1, gamma_inf=True),
            _key(16, 2, delta_inf=True), _key(17, 1, gamma_inf=True, delta_inf=True), _key(18, 1, alpha_inf=True)]
    pk, _ = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    xs = [int(x) for x in g['witness'][1:pk.n_public + 1]]
    good = Proof(bytes.fromhex(g['proofs'][0]['proof_hex']))
    a, b, c = _pts(good)
    keys.append((pk, [xs, xs, [(xs[0] + 1) % R] + xs[1:]], [good, _proof(o.G1.neg(a), b, c), good]))
    out = []
    for vk, ins, prs in keys:
        pvk = V.prepare_verifying_key(vk)
        out.append((vk, ins, prs, [V.verify_with_processed_vk(pvk, x, p) for x, p in zip(ins, prs)]))
    return out


gpu = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------- the same state as b2g_vk_load
@gpu
def test_batch_loaded_handles_hold_what_the_one_key_load_builds(ctx, mixed_keys):
    """every key of the mixed set, plus two duplicates, in one call: each handle gives the bytes of e(alpha, beta) and the
    verify_many, verify_batch_keys_locate and rerandomize_proofs results of a one-key handle of the same key, and the verdicts
    are the host verifier's"""
    order = list(range(len(mixed_keys))) + [3, 0]                     # the same desc twice: its own handle each time
    many = _load_many(ctx, [mixed_keys[i][0] for i in order])
    one = [_load_one(ctx, mixed_keys[i][0]) for i in order]
    assert len({h.value for h in many}) == len(order)
    rng = random.Random(20)
    for t, i in enumerate(order):
        vk, ins, prs, host = mixed_keys[i]
        assert host[:2] == [True, False], i                            # with gamma at infinity the inputs do not count
        assert _alpha_beta(many[t]) == _alpha_beta(one[t]), i
        assert _verify_many(ctx, many[t], ins, prs) == _verify_many(ctx, one[t], ins, prs) == host, i
        r1s, r2s = [rng.randrange(1, R) for _ in prs], [rng.randrange(1, R) for _ in prs]
        assert _rerandomize(ctx, many[t], prs, r1s, r2s) == _rerandomize(ctx, one[t], prs, r1s, r2s), i
    ws = [_weights(rng, len(mixed_keys[i][2])) for i in order]
    for entry in ('b2g_verify_batch_keys_locate', 'b2g_verify_batch_keys'):
        got = _keys_call(ctx, entry, [(h, mixed_keys[i][1], mixed_keys[i][2]) for h, i in zip(many, order)], ws)
        assert got == _keys_call(ctx, entry, [(h, mixed_keys[i][1], mixed_keys[i][2]) for h, i in zip(one, order)], ws)
        want = [v for i in order for v in mixed_keys[i][3]] if entry.endswith('locate') else [all(mixed_keys[i][3]) for i in order]
        assert got == want, entry
    # the valid proofs alone pass the keyed batch check under every batch-loaded handle
    assert _keys_call(ctx, 'b2g_verify_batch_keys', [(h, mixed_keys[i][1][:1], mixed_keys[i][2][:1]) for h, i in zip(many, order)],
                      [w[:1] for w in ws]) == [True] * len(order)
    _free(many + one)


# ---------------------------------------------------------------------------------------------- lifetime
@gpu
def test_handles_of_one_call_are_freed_one_by_one_in_any_order(ctx):
    """64 keys in one call, freed in a shuffled order: after each free every key still held verifies its proof (and a
    tampered one fails), so no free releases memory another handle still uses"""
    keys = _device_keys(ctx, [(k % 3, 1) for k in range(64)], 30)
    hs = _load_many(ctx, [vk for vk, _, _ in keys])
    held = list(range(64))
    rng = random.Random(31)
    rng.shuffle(held)
    while held:
        k = held.pop()
        _free([hs[k]])
        if not held:
            break
        batches = [(hs[j], keys[j][1], keys[j][2]) for j in held]
        bad = held[len(held) // 2]
        a, b, c = _pts(keys[bad][2][0])
        batches[len(held) // 2] = (hs[bad], keys[bad][1], [_proof(o.G1.neg(a), b, c)])
        got = _keys_call(ctx, 'b2g_verify_batch_keys', batches, [_weights(rng, 1) for _ in held])
        assert got == [j != bad for j in held], len(held)


# ---------------------------------------------------------------------------------------------- errors
def _off_curve(p):
    return (p[0], (p[1] + 1) % P)


def _off_curve_g2(q):
    return (q[0], ((q[1][0] + 1) % P, q[1][1]))


@gpu
def test_errors_name_the_key_and_change_nothing(ctx):
    L = N.lib()
    keys = [vk for vk, _, _ in _device_keys(ctx, [(k % 3, 0) for k in range(6)], 40)]
    sentinel = [0x5151 + i for i in range(6)]

    def call(vks, n=None, patch=None):
        descs, keep = _descs(vks)
        if patch:
            patch(descs)
        out = (C.c_void_p * len(vks))(*sentinel[:len(vks)])
        rc = L.b2g_vk_load_many(ctx._h, len(vks) if n is None else n, descs, out)
        assert list(out) == sentinel[:len(vks)]                         # out is not written
        return rc, L.b2g_last_error().decode()

    def good_call():
        hs = _load_many(ctx, keys)
        _free(hs)

    assert call(keys, n=0) == (-2, 'b2g_vk_load_many: n_keys must be at least 1')
    good_call()
    for field in ('alpha_g1', 'beta_g2', 'gamma_g2', 'delta_g2', 'gamma_abc_g1'):
        rc, msg = call(keys, patch=lambda d: setattr(d[4], field, None))
        assert (rc, msg) == (-2, 'b2g_vk_load_many: key 4: null verifying-key field'), field
    good_call()
    assert L.b2g_vk_load_many(ctx._h, 2, None, (C.c_void_p * 2)()) == -2
    assert L.b2g_vk_load_many(None, 2, _descs(keys[:2])[0], (C.c_void_p * 2)()) == -2
    # an off-curve IC[2] in key 2 (G1 point 3: alpha comes first), then also an off-curve gamma in key 5: the lowest key is named
    bad = list(keys)
    vk = keys[2]
    bad[2] = V.VerifyingKey(vk.alpha_g1, vk.beta_g2, vk.gamma_g2, vk.delta_g2, vk.gamma_abc_g1[:2] + [_off_curve(vk.gamma_abc_g1[2])])
    assert call(bad) == (-4, 'b2g_vk_load_many: key 2: G1 point 3 of alpha_g1 / gamma_abc_g1 is not on the curve')
    vk = keys[5]
    bad[5] = V.VerifyingKey(vk.alpha_g1, vk.beta_g2, _off_curve_g2(vk.gamma_g2), vk.delta_g2, vk.gamma_abc_g1)
    assert call(bad) == (-4, 'b2g_vk_load_many: key 2: G1 point 3 of alpha_g1 / gamma_abc_g1 is not on the curve')
    assert call(bad[3:]) == (-4, 'b2g_vk_load_many: key 2: G2 point 1 of beta_g2 / gamma_g2 / delta_g2 is not on the curve')
    good_call()
    # G1 before G2 within a key, as b2g_vk_load checks them; b2g_vk_load's own messages name no key
    vk = keys[1]
    both = V.VerifyingKey(_off_curve(vk.alpha_g1), vk.beta_g2, _off_curve_g2(vk.gamma_g2), vk.delta_g2, vk.gamma_abc_g1)
    assert call([keys[0], both]) == (-4, 'b2g_vk_load_many: key 1: G1 point 0 of alpha_g1 / gamma_abc_g1 is not on the curve')
    descs, keep = _descs([both])
    h = C.c_void_p(0x77)
    assert L.b2g_vk_load(ctx._h, descs, C.byref(h)) == -4 and h.value == 0x77
    assert L.b2g_last_error() == b'G1 point 0 of alpha_g1 / gamma_abc_g1 is not on the curve'
    descs[0].delta_g2 = None
    assert L.b2g_vk_load(ctx._h, descs, C.byref(h)) == -2 and L.b2g_last_error() == b'null verifying-key field'
    good_call()


# ---------------------------------------------------------------------------------------------- launches
@gpu
def test_launch_count_does_not_follow_the_keys_or_inputs(ctx):
    grown = set()
    for n_public in (1, 7):
        keys = [vk for vk, _, _ in _device_keys(ctx, [(n_public, 0)] * 256, 50 + n_public)]
        for k in (1, 16, 256):
            descs, keep = _descs(keys[:k])
            out = (C.c_void_p * k)()
            before = ctx.launch_count()
            assert N.lib().b2g_vk_load_many(ctx._h, k, descs, out) == 0
            grown.add(ctx.launch_count() - before)
            _free([C.c_void_p(h) for h in out])
    assert grown == {4}, grown


# ---------------------------------------------------------------------------------------------- the Python mirror
@gpu
def test_keyed_verifier_loads_its_new_keys_in_one_call(ctx, monkeypatch):
    """verify_batch_keys over 64 fresh keys calls b2g_vk_load_many once and b2g_vk_load never; its verdicts equal those with
    the keys loaded one by one.  load_verifying_keys leaves nothing for the verifier to load."""
    from circom_compat_b200 import Groth16, release
    keys = _device_keys(ctx, [(k % 3, 2) for k in range(64)], 60)
    batches = list(keys)
    for k in (5, 40):
        vk, ins, prs = batches[k]
        a, b, c = _pts(prs[1])
        batches[k] = (vk, ins, [prs[0], _proof(o.G1.neg(a), b, c)])
    rng = random.Random(61)
    ws = [_weights(rng, 2) for _ in batches]
    L = N.lib()
    calls = {'b2g_vk_load_many': 0, 'b2g_vk_load': 0}
    for name in calls:
        real = getattr(L, name)

        def counted(*args, real=real, name=name):
            calls[name] += 1
            return real(*args)
        monkeypatch.setattr(L, name, counted)
    got = Groth16.verify_batch_keys(batches, ctx, weights=ws)
    assert calls == {'b2g_vk_load_many': 1, 'b2g_vk_load': 0}
    assert got == [k not in (5, 40) for k in range(64)]
    for vk, _, _ in keys:
        release(vk)
    for vk, _, _ in keys:
        ctx.vk_handle(vk)                                             # one by one
    assert calls == {'b2g_vk_load_many': 1, 'b2g_vk_load': 64}
    assert Groth16.verify_batch_keys(batches, ctx, weights=ws) == got
    assert Groth16.verify_batch_keys_locate(batches, ctx, weights=ws) == [[True, k not in (5, 40)] for k in range(64)]
    for vk, _, _ in keys:
        release(vk)
    Groth16.load_verifying_keys([vk for vk, _, _ in keys] + [keys[0][0]], ctx)
    assert calls == {'b2g_vk_load_many': 2, 'b2g_vk_load': 64}
    assert Groth16.verify_batch_keys(batches, ctx, weights=ws) == got
    assert calls == {'b2g_vk_load_many': 2, 'b2g_vk_load': 64}
    for vk, _, _ in keys:
        release(vk)


@gpu
def test_keyed_verifier_errors_keep_their_precedence(ctx):
    """two faulty batches: the error is the one the verifier raised when it loaded each batch's key as it reached the batch.
    After a failed check the keys of the batches before it are loaded; after a refused key none of the call's keys is."""
    from circom_compat_b200 import B2gError, Groth16, release
    from circom_compat_b200.groth16 import _VK_HANDLES
    keys = _device_keys(ctx, [(1, 1), (2, 1), (1, 1), (1, 1)], 70)
    vk = keys[1][0]
    off = V.VerifyingKey(vk.alpha_g1, vk.beta_g2, vk.gamma_g2, vk.delta_g2, vk.gamma_abc_g1[:2] + [_off_curve(vk.gamma_abc_g1[2])])
    off_batch = (off, keys[1][1], keys[1][2])
    arity = (keys[2][0], [keys[2][1][0] + [1]], keys[2][2])           # two inputs for a one-input key

    def loaded(vk):
        return (id(vk), ctx.device) in _VK_HANDLES

    # the off-curve key first: its load error wins
    with pytest.raises(B2gError) as e:
        Groth16.verify_batch_keys([keys[0], off_batch, keys[3], arity], ctx)
    assert e.value.code == -4
    assert e.value.msg == 'verify_batch_keys: key 1: G1 point 3 of alpha_g1 / gamma_abc_g1 is not on the curve'
    assert not loaded(keys[0][0]) and not loaded(off) and not loaded(keys[3][0])
    # the input-count error first: it wins, and nothing after it is loaded
    with pytest.raises(V.MalformedVerifyingKey, match='verify_batch_keys_locate: key 1: 2 public inputs for a key with 1'):
        Groth16.verify_batch_keys_locate([keys[0], arity, off_batch, keys[3]], ctx)
    assert loaded(keys[0][0]) and not loaded(off) and not loaded(keys[3][0])
    # a key refused in a later batch than its first use is named under its first use; an empty batch loads nothing
    with pytest.raises(B2gError) as e:
        Groth16.verify_batch_keys([(keys[3][0], [], []), keys[3], (off, [], []), off_batch, off_batch], ctx)
    assert e.value.msg == 'verify_batch_keys: key 3: G1 point 3 of alpha_g1 / gamma_abc_g1 is not on the curve'
    assert not loaded(keys[3][0])
    # load_verifying_keys names the key by its index in the list, and loads none
    with pytest.raises(B2gError) as e:
        Groth16.load_verifying_keys([keys[2][0], keys[3][0], keys[3][0], off], ctx)
    assert e.value.code == -4 and e.value.msg == 'key 3: G1 point 3 of alpha_g1 / gamma_abc_g1 is not on the curve'
    assert not loaded(keys[2][0]) and not loaded(keys[3][0])
    assert Groth16.verify_batch_keys([keys[2], keys[3]], ctx) == [True, True]
    for vk, _, _ in keys:
        release(vk)


# ---------------------------------------------------------------------------------------------- the C++ mirror
@gpu
def test_cpp_mirror_load_verifying_keys(complex_zkey_bytes, golden):
    """Groth16::load_verifying_keys over six copies of the bench key (four launches), then verify_batch_keys with proof i
    under copy i and A negated in proofs 1 and 4: the verdicts equal the C++ host verifier's"""
    exe = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench')
    out = subprocess.check_output([exe, os.path.join(ROOT, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'),
                                   'chain:%d' % int(golden['complex_zkey']['a']), '0'], text=True, env=dict(os.environ, B2G_LOAD_KEYS='6'))
    line = [l for l in out.splitlines() if l.startswith('load_keys')][0]
    assert 'load_keys 6 keys: held=1 load_launches=4 ' in line, line
    assert 'device=101101 host=101101 agree=1' in line, line


# ---------------------------------------------------------------------------------------------- without a GPU
def test_load_many_is_exported_and_declared():
    N.lib()
    assert 'b2g_vk_load_many' in N.EXPORTS
    assert hasattr(N.lib(), 'b2g_vk_load_many')
    hdr = open(os.path.join(ROOT, 'include', 'b2groth.h')).read()
    assert 'B2G_API int b2g_vk_load_many(b2g_ctx* ctx, uint32_t n_keys, const b2g_vk_desc* descs, b2g_vk** out);' in hdr


def _has_cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_cuda(), reason="checks the no-GPU failure mode")
def test_no_device_gives_a_device_error():
    """without a device there is no context to load into: load_verifying_keys fails with B2G_E_DEVICE, and the raw call
    without a context is refused before it touches a device"""
    from circom_compat_b200 import B2gError, Groth16
    vks = [_key(80, 0)[0], _key(81, 1)[0]]
    with pytest.raises(B2gError) as e:
        Groth16.load_verifying_keys(vks)
    assert e.value.code == -3
    descs, keep = _descs(vks[:1])
    assert N.lib().b2g_vk_load_many(None, 1, descs, (C.c_void_p * 1)()) == -2
