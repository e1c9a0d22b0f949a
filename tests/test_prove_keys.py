"""b2g_prove_keys / Groth16.create_proofs_keys: batches of witnesses under many proving keys in one device pass.  Every
key's batch must equal, byte for byte, Groth16.create_proofs on that key alone with the same (r, s) and witnesses."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from oracle import pyref as o
import prove_keys_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu


def _rs(rng, count):
    edge = [(0, 1), (1, 0), (o.R_MOD - 1, o.R_MOD - 1)]
    return [edge[k] if k < len(edge) else (rng.randrange(o.R_MOD), rng.randrange(o.R_MOD)) for k in range(count)]


class Key:
    """one key of the tests: (pk, matrices, reduction), satisfying witnesses (Montgomery) and their public inputs"""

    def __init__(self, pk, cm, red, ws, publics):
        self.pk, self.cm, self.red, self.ws, self.publics = pk, cm, red, ws, publics


def _expect(ctx, key, rs, ws):
    from circom_compat_b200 import Groth16
    return [p.data for p in Groth16.create_proofs(key.pk, rs, key.cm, ws, ctx, key.red)] if ws else []


def _prove_keys(ctx, keys, batches, group=None):
    """create_proofs_keys over a group of `keys` (loaded here unless given) -> one list of proof bytes per key"""
    from circom_compat_b200 import Groth16, release
    g = group or Groth16.load_proving_keys([(k.pk, k.cm, k.red) for k in keys], ctx)
    try:
        return [[p.data for p in ps] for ps in Groth16.create_proofs_keys(g, batches, ctx)]
    finally:
        if group is None:
            release(g)


def _check(ctx, keys, counts, seed=0, group=None):
    """counts[k] proofs under keys[k] (witness i of the key's list, cycled) against create_proofs per key"""
    rng = random.Random(seed)
    batches = []
    for k, n in zip(keys, counts):
        batches.append((_rs(rng, n), [k.ws[i % len(k.ws)] for i in range(n)]))
    got = _prove_keys(ctx, keys, batches, group)
    for k, (rs, ws), g in zip(keys, batches, got):
        assert g == _expect(ctx, k, rs, ws)
    return batches, got


@pytest.fixture(scope='module')
def keys(ctx, golden, test_zkey_bytes, complex_zkey_bytes):
    """test.zkey, the reference's 2^14 bench key, synthetic chain keys at 2^4 / 2^10 / 2^12 (two distinct 2^10 keys), a
    circom-like 2^13 key with a sparse B query, and LibsnarkReduction keys: a sparse circom-like 2^12 one and a dense
    2^10 chain"""
    from circom_compat_b200 import (read_zkey, fr_to_mont, synth, release, CircomReduction, LibsnarkReduction)
    out = {}
    pk, cm = read_zkey(test_zkey_bytes)
    w = [int(x) for x in golden['test_zkey']['witness']]
    out['test'] = Key(pk, cm, CircomReduction, [fr_to_mont(w)], [w[1:cm.num_instance_variables]])
    pk, cm = read_zkey(complex_zkey_bytes)
    a0 = int(golden['complex_zkey']['a'])
    ws = [o.chain_witness(pk.n_vars, a0 + k) for k in range(3)]
    out['bench'] = Key(pk, cm, CircomReduction, [fr_to_mont(v) for v in ws], [v[1:cm.num_instance_variables] for v in ws])

    def chain(n, seed=0xB200, flavour='circom'):
        circ = synth.chain_circuit(n)
        pk, _ = synth.setup(ctx, circ, seed=seed, flavour=flavour)
        ws = [synth.chain_witness(n, 3 + k) for k in range(3)]
        red = LibsnarkReduction if flavour == 'libsnark' else CircomReduction
        return Key(pk, circ.matrices(with_c=flavour == 'libsnark'), red, [fr_to_mont(v) for v in ws], [v[1:circ.num_inputs] for v in ws])

    out['c4'] = chain(1 << 4)
    out['c10'] = chain(1 << 10)
    out['c10b'] = chain(1 << 10, seed=0xB201)
    out['c12'] = chain(1 << 12)
    out['lib10'] = chain(1 << 10, seed=0xB202, flavour='libsnark')
    for name, log_n, flavour in (('sparse13', 13, 'circom'), ('lib12', 12, 'libsnark')):
        circ, w = synth.circomlike_circuit(log_n)
        pk, _ = synth.setup(ctx, circ, flavour=flavour)
        red = LibsnarkReduction if flavour == 'libsnark' else CircomReduction
        rng = random.Random(log_n)
        vs = [list(w)]
        for _ in range(2):                   # unsatisfied copies: their proofs are still deterministic
            v = list(w)
            for i in rng.sample(range(2, len(v)), len(v) // 3):
                v[i] = rng.randrange(o.R_MOD)
            vs.append(v)
        out[name] = Key(pk, circ.matrices(with_c=flavour == 'libsnark'), red, [fr_to_mont(v) for v in vs], [w[1:circ.num_inputs]])
    yield out
    for k in out.values():
        release(k.pk); release(k.cm)


# ---------------------------------------------------------------------------------------------- on the GPU
@gpu
def test_one_key_equals_create_proofs(ctx, golden, keys):
    """K = 1 on the reference bench key: the keyed call is create_proofs, and the golden (r, s) gives the golden bytes"""
    k = keys['bench']
    g = golden['complex_zkey']
    rs = [(int(g['r']), int(g['s']))] + _rs(random.Random(1), 2)
    got = _prove_keys(ctx, [k], [(rs, k.ws)])[0]
    assert got[0].hex() == g['proof_hex']
    assert got == _expect(ctx, k, rs, k.ws)


@gpu
def test_keys_of_one_size(ctx, keys):
    """two distinct 2^10 keys and a 2^10 LibsnarkReduction key: equal base counts, so no key is sorted at another's c"""
    _check(ctx, [keys['c10'], keys['c10b'], keys['lib10']], [3, 2, 3], seed=2)


@gpu
def test_mixed_domains(ctx, keys):
    """2^4 .. 2^14 in one group: every query at the 2^14 key's c, the small keys' rows after the large ones or before"""
    _check(ctx, [keys['c4'], keys['bench'], keys['c10'], keys['test'], keys['c12']], [2, 3, 1, 1, 2], seed=3)
    _check(ctx, [keys['c12'], keys['test'], keys['c4'], keys['bench']], [1, 2, 3, 1], seed=4)


@gpu
def test_reductions_and_b_queries_mixed(ctx, keys):
    """CircomReduction and LibsnarkReduction keys with sparse (compacted) and dense B queries in one group"""
    _check(ctx, [keys['sparse13'], keys['lib12'], keys['c12'], keys['lib10']], [3, 3, 2, 2], seed=5)
    _check(ctx, [keys['lib12'], keys['c4'], keys['sparse13']], [1, 2, 2], seed=6)


@gpu
def test_public_input_counts(ctx, keys):
    """test.zkey, the bench key and single-input synthetic keys side by side"""
    _check(ctx, [keys['test'], keys['bench'], keys['c10']], [2, 2, 2], seed=7)


@gpu
def test_counts_and_order(ctx, keys):
    """a key with no proofs (first, middle and last), a key with one proof, the same key twice, and the group permuted"""
    ks = [keys['c4'], keys['c10'], keys['sparse13'], keys['c10'], keys['test']]
    _check(ctx, ks, [0, 1, 2, 0, 3], seed=8)
    _check(ctx, ks, [2, 0, 1, 1, 0], seed=9)
    _check(ctx, ks[::-1], [1, 3, 0, 2, 1], seed=10)


@gpu
def test_total_crosses_scan_boundary(ctx, keys):
    """2^4 and 2^10 keys share c = 8 (128 buckets per proof): 8 proofs fill the single-CTA scan's 1024 threads with one bucket
    each, 9 give every thread two; and the 2^4 key's proofs leave the sort grid (sized by the 2^10 key) whole CTAs early"""
    from circom_compat_b200 import Groth16, release
    ks = [keys['c4'], keys['c10']]
    g = Groth16.load_proving_keys([(k.pk, k.cm, k.red) for k in ks], ctx)
    try:
        for counts in ([4, 4], [5, 4], [1, 8], [40, 1]):
            _check(ctx, ks, counts, seed=sum(counts), group=g)
    finally:
        release(g)


@gpu
def test_results_verify(ctx, keys):
    """every keyed proof passes verify_batch_keys under its key; a wrong public input is rejected for its key only"""
    from circom_compat_b200 import Groth16, Proof
    ks = [keys['test'], keys['bench'], keys['c12'], keys['lib10']]
    rng = random.Random(11)
    batches = [(_rs(rng, len(k.ws)), k.ws) for k in ks]
    got = _prove_keys(ctx, ks, batches)
    vb = [(k.pk, k.publics, [Proof(d) for d in ps]) for k, ps in zip(ks, got)]
    assert Groth16.verify_batch_keys(vb, ctx) == [True] * len(ks)
    bad = list(vb)
    pub = [list(x) for x in bad[2][1]]
    pub[1][0] = (pub[1][0] + 1) % o.R_MOD
    bad[2] = (bad[2][0], pub, bad[2][2])
    assert Groth16.verify_batch_keys(bad, ctx) == [True, True, False, True]


@gpu
def test_graph_direct_and_recapture(ctx, monkeypatch, keys):
    """direct launches (B2G_GRAPH=0) and the captured pass agree; one context re-captures per counts vector, grows its
    buffers and keeps proving single-key batches in between"""
    from circom_compat_b200 import Context, Groth16, release
    ks = [keys['c12'], keys['sparse13'], keys['c4']]
    monkeypatch.setenv('B2G_GRAPH', '0')
    direct = Context(0)
    monkeypatch.delenv('B2G_GRAPH')
    graph = Context(0)
    g = Groth16.load_proving_keys([(k.pk, k.cm, k.red) for k in ks], graph)
    try:
        _check(direct, ks, [2, 1, 3], seed=12, group=g)
        for counts in ([2, 1, 3], [1, 3, 0], [2, 1, 3]):
            _check(graph, ks, counts, seed=12, group=g)
            k = keys['bench']
            rs = _rs(random.Random(13), 2)
            assert _expect(graph, k, rs, k.ws[:2]) == _expect(ctx, k, rs, k.ws[:2])
    finally:
        release(g)
        direct.close(); graph.close()


@gpu
def test_dense_groups_share_the_witness_sort(ctx, keys):
    """with no sparse B query in the group, B1 and B2 read the L / A sort: adding a sparse key (with no proofs) adds exactly
    the B gather and the four launches of a third digit sort to the call, and both groups give create_proofs' bytes"""
    from circom_compat_b200 import Groth16, release
    dense = [keys['c10'], keys['c12'], keys['lib10']]
    launches = []
    for ks in (dense, dense + [keys['sparse13']]):
        g = Groth16.load_proving_keys([(k.pk, k.cm, k.red) for k in ks], ctx)
        try:
            counts = [2, 1, 2] + [0] * (len(ks) - 3)
            _check(ctx, ks, counts, seed=15, group=g)                      # also captures the pass
            before = ctx.launch_count()
            _check(ctx, ks, counts, seed=16, group=g)
            # _check also runs create_proofs per key: take those out with a second run of the same per-key calls
            mid = ctx.launch_count()
            for k, n in zip(ks, counts):
                _expect(ctx, k, _rs(random.Random(16), n), [k.ws[i % len(k.ws)] for i in range(n)])
            launches.append((mid - before) - (ctx.launch_count() - mid))
        finally:
            release(g)
    assert launches[1] - launches[0] == 5, launches


@gpu
def test_contexts_torn_down_after_keyed_calls(keys):
    """contexts that ran keyed passes (dense and sparse groups, captured and direct) are destroyed with their keyed buffers
    and graphs, one after another, and a fresh context still proves every key correctly"""
    from circom_compat_b200 import Context, Groth16, release
    ks = [keys['c4'], keys['sparse13'], keys['c10']]
    for i in range(3):
        cx = Context(0)
        g = Groth16.load_proving_keys([(k.pk, k.cm, k.red) for k in ks[:2 + i % 2]], cx)
        try:
            _check(cx, ks[:2 + i % 2], [2, 1, 1][:2 + i % 2], seed=20 + i, group=g)
        finally:
            release(g)
            cx.close()
    cx = Context(0)
    try:
        _check(cx, ks, [1, 2, 1], seed=23)
    finally:
        cx.close()


@gpu
def test_refusals_leave_the_context_usable(ctx, keys):
    """each refused input gives its code and message, and the context then proves correctly again"""
    from circom_compat_b200 import Context, Groth16, B2gError, release, _native as N
    L = N.lib()
    ks = [keys['c10'], keys['c4']]

    def good():
        _check(ctx, ks, [1, 2], seed=14)

    # a pk with another circuit's matrices (key 1 of the group: the 2^4 key with the 2^12 circuit's matrices)
    from circom_compat_b200.groth16 import _pk_desc
    (d0, k0), (d1, k1) = _pk_desc(keys['c10'].pk), _pk_desc(keys['c4'].pk)
    descs = (N.PkDesc * 2)(d0, d1)
    mats = (C.c_void_p * 2)(ctx.mat_handle(keys['c10'].cm, keys['c10'].pk.n_vars).value, ctx.mat_handle(keys['c12'].cm, keys['c12'].pk.n_vars).value)
    h = C.c_void_p()
    assert L.b2g_pk_group_load(ctx._h, 2, descs, mats, C.byref(h)) == N.B2G_E_SHAPE
    def last():
        return L.b2g_last_error().decode()

    assert last() == "b2g_pk_group_load: key 1: proving key and matrices disagree on n_vars" and not h.value
    good()
    # an empty group, null pointers, a sharded context
    assert L.b2g_pk_group_load(ctx._h, 0, None, None, C.byref(h)) == N.B2G_E_SHAPE
    assert last() == "b2g_pk_group_load: the group has no keys"
    assert L.b2g_pk_group_load(ctx._h, 2, None, mats, C.byref(h)) == N.B2G_E_SHAPE
    assert last() == "null pointer"
    sharded = Context(0, 0, 2)
    assert L.b2g_pk_group_load(sharded._h, 2, descs, mats, C.byref(h)) == N.B2G_E_SHAPE
    assert last() == "b2g_pk_group_load: a key group needs an unsharded context"
    sharded.close()
    with pytest.raises(ValueError):
        Groth16.load_proving_keys([], ctx)
    g = Groth16.load_proving_keys([(k.pk, k.cm, k.red) for k in ks], ctx)
    w = ks[0].ws[0]
    rr = np.zeros(4 * 65536, dtype=np.uint64)
    out = np.zeros(256 * 65536, dtype=np.uint8)

    def call(cx, counts, ptrs):
        cnt = np.array(counts, dtype=np.uint32)
        return L.b2g_prove_keys(cx._h, g._h, cnt.ctypes.data, rr.ctypes.data, rr.ctypes.data, ptrs, out.ctypes.data)

    try:
        one = (C.c_void_p * 1)(w.ctypes.data)
        cnt = np.array([1, 0], dtype=np.uint32)
        assert L.b2g_prove_keys(ctx._h, g._h, None, rr.ctypes.data, rr.ctypes.data, one, out.ctypes.data) == N.B2G_E_SHAPE
        assert last() == "null pointer"
        assert L.b2g_prove_keys(ctx._h, g._h, cnt.ctypes.data, rr.ctypes.data, None, one, out.ctypes.data) == N.B2G_E_SHAPE
        assert last() == "null pointer"
        assert call(ctx, [0, 0], one) == N.B2G_E_SHAPE
        assert last() == "b2g_prove_keys: the total count must be in [1, 65535]"
        many = (C.c_void_p * 65536)(*([w.ctypes.data] * 65536))
        assert call(ctx, [65535, 1], many) == N.B2G_E_SHAPE
        assert last() == "b2g_prove_keys: the total count must be in [1, 65535]"
        assert call(ctx, [2, 0], (C.c_void_p * 2)(w.ctypes.data, None)) == N.B2G_E_SHAPE
        assert last() == "null witness 1"
        good()
        sharded = Context(0, 0, 2)
        assert call(sharded, [1, 0], one) == N.B2G_E_SHAPE
        assert last() == "b2g_prove_keys needs an unsharded context"
        sharded.close()
        k = keys['bench']
        pending = Groth16.submit(k.pk, 1, 2, k.cm, k.ws[0], ctx)
        with pytest.raises(B2gError) as e:
            Groth16.create_proofs_keys(g, [([(1, 2)], [w]), ([], [])], ctx)
        assert e.value.code == N.B2G_E_SHAPE
        assert e.value.msg == "a submitted proof is still pending on this context: call b2g_prove_wait first"
        assert pending.wait().data == _expect(ctx, k, [(1, 2)], [k.ws[0]])[0]
        with pytest.raises(ValueError):
            Groth16.create_proofs_keys(g, [([(1, 2)], [w])], ctx)       # one batch per key
        with pytest.raises(ValueError) as v:
            Groth16.create_proofs_keys(g, [([(1, 2)], [w]), ([(1, 2)], [w])], ctx)   # a witness of the wrong length
        assert str(v.value) == "create_proofs_keys: key 1: full_assignment length != n_vars"
        assert Groth16.create_proofs_keys(g, [([], []), ([], [])], ctx) == [[], []]
        good()
    finally:
        release(g)


@gpu
def test_cpp_mirror_prove_keys(golden, keys, ctx):
    """Groth16T::create_proofs_keys through groth16_bench (B2G_PROVE_KEYS=3: copy k of the bench key proves chain:<a + k>
    with the golden (r, s)) gives create_proofs' bytes"""
    k = keys['bench']
    g = golden['complex_zkey']
    exe = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench')
    out = subprocess.check_output([exe, os.path.join(ROOT, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'), 'chain:%d' % int(g['a']), '1',
                                   '%x' % int(g['r']), '%x' % int(g['s'])], text=True, env=dict(os.environ, B2G_PROVE_KEYS='3'))
    lines = dict(l.split('=', 1) for l in out.splitlines() if l.startswith('keys['))
    rs = [(int(g['r']), int(g['s']))] * 3
    py = _expect(ctx, k, rs, k.ws[:3])
    assert [lines['keys[%d]' % i] for i in range(3)] == [d.hex() for d in py]
    assert py[0].hex() == g['proof_hex'] and 'first_identical=1' in out


# ---------------------------------------------------------------------------------------------- without a GPU
def _layout(bases, n_vars=None, n_dom=None, counts=None):
    """b2g_pk_group_layout -> (c per query, first rows per key, the three sorts' rows) or the refusal's message"""
    from circom_compat_b200 import _native as N
    K = len(bases)
    b = np.array(bases, dtype=np.uint32).reshape(-1)
    c = np.zeros(5, dtype=np.int32)
    rows = np.zeros(max(5 * K, 1), dtype=np.uint32)
    total = sum(counts) if counts else 0
    out = np.zeros(max(12 * total, 1), dtype=np.uint64) if counts and total <= 65535 else np.zeros(1, dtype=np.uint64)
    arrs = [np.array(x, dtype=np.uint32) if x is not None else None for x in (n_vars, n_dom, counts)]
    ptr = [a.ctypes.data if a is not None else None for a in arrs]
    rc = N.lib().b2g_pk_group_layout(K, b.ctypes.data if K else None, ptr[0], ptr[1], ptr[2], c.ctypes.data, rows.ctypes.data, out.ctypes.data)
    if rc != N.B2G_OK:
        return rc, N.lib().b2g_last_error().decode()
    cs = c.tolist()
    first = rows[:5 * K].reshape(K, 5).tolist()
    if not counts:
        return cs, first
    sorts = [[tuple(out[4 * (t * total + j):4 * (t * total + j) + 4].tolist()) for j in range(total)] for t in range(3)]
    return cs, first, sorts


def _random_group(rng, K):
    keys = []
    for _ in range(K):
        log_n = rng.randrange(2, 18)
        n_vars = rng.randrange(3, (1 << log_n) + 1)
        b = rng.choice([None, rng.randrange(0, n_vars)])
        keys.append((M.key_bases(1 << log_n, n_vars, b), n_vars, (1 << log_n) + rng.randrange(2)))
    return keys


@pytest.mark.parametrize('seed', range(6))
def test_layout_matches_model(seed):
    """windows, arena rows and per-proof rows of random groups (sizes 2^2 .. 2^17, sparse and dense B, zero counts) as the
    plain model computes them"""
    rng = random.Random(seed)
    keys = _random_group(rng, rng.randrange(1, 9))
    bases = [k[0] for k in keys]
    n_vars = [k[1] for k in keys]
    n_dom = [k[2] for k in keys]
    counts = [rng.choice([0, 1, 2, 5]) for _ in keys]
    counts[rng.randrange(len(keys))] += 1
    cs, rows = M.group_layout(bases)
    assert _layout(bases) == (cs, rows)
    got = _layout(bases, n_vars, n_dom, counts)
    assert got == (cs, rows, M.call_layout(cs, rows, bases, n_vars, n_dom, counts))


def test_layout_small_key_takes_the_large_keys_window():
    """a 2^4 key next to the 2^14 bench shape: every query at c = 13 (4096 buckets per proof), rows after the large key"""
    big, small = M.key_bases(1 << 14, 10002), M.key_bases(1 << 4, 16)
    cs, rows = _layout([big, small])
    assert cs == [13] * 5
    assert rows[1] == [v * M.nwin(13) for v in big]
    assert _layout([small]) == ([8] * 5, [[0] * 5])


def test_layout_refuses_2p31_rows():
    """two 2^27 domains: each H arena is 15 x 2^27 rows, together past the sign bit of an entry word"""
    from circom_compat_b200 import _native as N
    one = M.key_bases(1 << 27, 5)
    assert _layout([one])[0][0] == 17
    with pytest.raises(M.Refused):
        M.group_layout([one, one])
    rc, msg = _layout([one, one])
    assert rc == N.B2G_E_SHAPE and 'query H reach 2^31 rows' in msg


def test_layout_refuses_2p32_entries():
    """a call whose proofs x bases x windows of one sort reach 2^32 (one proof more than fits, with either key), and the
    total count bounds"""
    from circom_compat_b200 import _native as N
    bases = [M.key_bases(1 << 14, 10002), M.key_bases(1 << 12, 4096)]
    cs, rows = M.group_layout(bases)
    n, nw = 1 << 14, M.nwin(cs[0])                  # the H sort binds first: 2^14 bases per proof of key 0
    count = -(-(1 << 32) // (n * nw))
    for counts, ok in (([count - 1, 0], True), ([count, 0], False), ([count - 1, 40], False)):
        args = (bases, [10002, 4096], [1 << 14, 1 << 12], counts)
        if ok:
            M.call_layout(cs, rows, *args[:1], *args[1:])
            assert len(_layout(*args)) == 3
        else:
            with pytest.raises(M.Refused):
                M.call_layout(cs, rows, *args[:1], *args[1:])
            rc, msg = _layout(*args)
            assert rc == N.B2G_E_SHAPE
            assert msg == "b2g_prove_keys: proofs x bases x windows of query H reach 2^32 sorted entries; prove fewer per call"
    for counts in ([0, 0], [65535, 1]):
        rc, msg = _layout(bases, [10002, 4096], [1 << 14, 1 << 12], counts)
        assert rc == N.B2G_E_SHAPE and msg == "b2g_prove_keys: the total count must be in [1, 65535]"
    rc, msg = _layout([])
    assert rc == N.B2G_E_SHAPE and msg == "b2g_pk_group_load: the group has no keys"


def test_prove_keys_is_exported_and_declared():
    from circom_compat_b200 import _native as N
    hdr = open(os.path.join(ROOT, 'include', 'b2groth.h')).read()
    for name in ('b2g_pk_group_load', 'b2g_pk_group_free', 'b2g_prove_keys', 'b2g_pk_group_layout'):
        assert name in N.EXPORTS
        assert hasattr(N.lib(), name)
        assert f'B2G_API int {name}(' in hdr
