"""b2g_prove_many / Groth16.create_proofs: K witnesses of one circuit proved in one device pass.  Every batched proof must
equal, byte for byte, the single-proof call with the same (r_i, s_i, w_i) on the same key."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from oracle import pyref as o

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _singles(pk, cm, rs, ws, ctx, reduction=None):
    from circom_compat_b200 import Groth16, CircomReduction
    reduction = reduction or CircomReduction
    return [Groth16.create_proof_with_reduction_and_matrices(pk, r, s, cm, cm.num_instance_variables, cm.num_constraints, w, ctx, reduction).data
            for (r, s), w in zip(rs, ws)]


def _many(pk, cm, rs, ws, ctx, reduction=None):
    from circom_compat_b200 import Groth16, CircomReduction
    return [p.data for p in Groth16.create_proofs(pk, rs, cm, ws, ctx, reduction or CircomReduction)]


def _random_rs(rng, count):
    edge = [(0, 1), (1, 0), (o.R_MOD - 1, o.R_MOD - 1), (0, 0)]
    return [edge[k] if k < len(edge) else (rng.randrange(o.R_MOD), rng.randrange(o.R_MOD)) for k in range(count)]


@pytest.fixture(scope='module')
def complex_key(complex_zkey_bytes):
    from circom_compat_b200 import read_zkey, release
    pk, cm = read_zkey(complex_zkey_bytes)
    yield pk, cm
    release(pk); release(cm)


@pytest.fixture(scope='module')
def chain_witnesses(complex_key, golden):
    """Montgomery chain witnesses of the golden key: a = golden a + k"""
    from circom_compat_b200 import fr_to_mont
    pk, _ = complex_key
    a0 = int(golden['complex_zkey']['a'])
    return [fr_to_mont(o.chain_witness(pk.n_vars, a0 + k)) for k in range(33)]


@pytest.mark.parametrize('count', [1, 2, 7, 33])
def test_reference_bench_key_batches(ctx, golden, complex_key, chain_witnesses, count):
    """complex-circuit-10000-10000 (2^14, the reference's benches/groth16.rs key): distinct witnesses, (r, s) with 0, 1 and
    r - 1; the golden entry gives the golden bytes and two identical entries give identical proofs"""
    pk, cm = complex_key
    g = golden['complex_zkey']
    rng = random.Random(count)
    ws = [chain_witnesses[k] for k in range(count)]
    rs = _random_rs(rng, count)
    gi = count // 2                                                    # the golden entry sits mid-batch
    ws[gi], rs[gi] = chain_witnesses[0], (int(g['r']), int(g['s']))
    if count >= 2:                                                     # last entry repeats the golden one
        ws[-1], rs[-1] = ws[gi], rs[gi]
    got = _many(pk, cm, rs, ws, ctx)
    assert got[gi].hex() == g['proof_hex']
    if count >= 2:
        assert got[-1] == got[gi]
    assert got == _singles(pk, cm, rs, ws, ctx)
    if count >= 7:
        assert len(set(got)) == count - 1


@pytest.mark.parametrize('compact', [True, False])
def test_sparse_b_batches(ctx, monkeypatch, compact):
    """circom-like key at 2^13 whose B query is mostly infinity: the compacted B scalars of proof j sit at j * b_compact"""
    from circom_compat_b200 import fr_to_mont, synth, release
    circ, w = synth.circomlike_circuit(13)
    if not compact:
        monkeypatch.setenv('B2G_NO_B_COMPACT', '1')
    pk, td = synth.setup(ctx, circ)
    cm = circ.matrices()
    rng = random.Random(13)
    # the real witness, and copies with a share of the wires replaced: proofs of unsatisfied assignments are still deterministic
    ws = [list(w)]
    for k in range(4):
        v = list(w)
        for i in rng.sample(range(2, len(v)), len(v) // 3):
            v[i] = rng.randrange(o.R_MOD) if k % 2 else rng.randrange(2)
        ws.append(v)
    ws = [fr_to_mont(v) for v in ws]
    rs = _random_rs(rng, len(ws))
    assert _many(pk, cm, rs, ws, ctx) == _singles(pk, cm, rs, ws, ctx)
    release(pk); release(cm)


def _resolved_witness(circ, w, rng):
    """another satisfying assignment of a circuit whose rows each set one wire (C = one term, rows in dependency order, as
    synth.circomlike_circuit builds them): every wire no row sets is redrawn, then each row's target is recomputed, the
    public output included"""
    v = list(w)
    targets = set(np.asarray(circ.C[1]).tolist())
    for i in range(1, len(v)):
        if i not in targets:
            v[i] = rng.randrange(o.R_MOD)
    terms = {}
    for name, (rows, cols, vals) in zip('ABC', (circ.A, circ.B, circ.C)):
        for r_, c_, x in zip(np.asarray(rows).tolist(), np.asarray(cols).tolist(), vals):
            terms.setdefault((name, r_), []).append((c_, x))
    for k in range(circ.num_constraints):
        a = sum(x * v[c_] for c_, x in terms.get(('A', k), ())) % o.R_MOD
        b = sum(x * v[c_] for c_, x in terms.get(('B', k), ())) % o.R_MOD
        (col, x), = terms[('C', k)]
        v[col] = a * b * pow(x, -1, o.R_MOD) % o.R_MOD
    return v


def test_libsnark_reduction_batch_verifies(ctx):
    """five distinct satisfying witnesses (distinct public outputs) of a circom-like 2^12 circuit under LibsnarkReduction:
    a proof that reads another proof's a, b, c or h slice no longer equals its single proof nor verifies"""
    from circom_compat_b200 import Groth16, LibsnarkReduction, fr_to_mont, synth, release, Proof
    circ, w = synth.circomlike_circuit(12)
    pk, td = synth.setup(ctx, circ, flavour='libsnark')
    cm = circ.matrices(with_c=True)
    rng = random.Random(12)
    ws = [list(w)] + [_resolved_witness(circ, w, rng) for _ in range(4)]
    assert len({v[1] for v in ws}) == 5
    wms = [fr_to_mont(v) for v in ws]
    rs = _random_rs(rng, 5)
    got = _many(pk, cm, rs, wms, ctx, LibsnarkReduction)
    assert got == _singles(pk, cm, rs, wms, ctx, LibsnarkReduction)
    for d, v in zip(got, ws):
        assert Groth16.verify(pk, v[1:circ.num_inputs], Proof(d))
    assert not Groth16.verify(pk, ws[1][1:circ.num_inputs], Proof(got[0]))
    release(pk); release(cm)


@pytest.fixture(scope='module')
def chain10(ctx):
    from circom_compat_b200 import fr_to_mont, synth, release
    circ = synth.chain_circuit(1 << 10)
    pk, td = synth.setup(ctx, circ)
    cm = circ.matrices()
    dense = [fr_to_mont(synth.chain_witness(1 << 10, 3 + k)) for k in range(5)]
    zero = fr_to_mont(synth.chain_witness(1 << 10, 0))               # only w0 = 1
    yield pk, cm, dense, zero
    release(pk); release(cm)


def test_small_key_buckets_restart_per_proof(ctx, chain10):
    """2^10 key: c = 8, 128 buckets per proof, fewer than one reduce CTA spans, so several proofs share a reduce CTA's range
    unless the weights restart per proof; and a batch where all-zero witnesses leave a proof's buckets empty between full
    neighbours"""
    pk, cm, dense, zero = chain10
    rng = random.Random(10)
    rs = _random_rs(rng, 5)
    assert _many(pk, cm, rs, dense, ctx) == _singles(pk, cm, rs, dense, ctx)
    mixed = [dense[0], zero, dense[1], zero, dense[2]]
    assert _many(pk, cm, rs, mixed, ctx) == _singles(pk, cm, rs, mixed, ctx)


@pytest.fixture(scope='module')
def chain12(ctx):
    from circom_compat_b200 import fr_to_mont, synth, release
    circ = synth.chain_circuit(1 << 12)
    pk, td = synth.setup(ctx, circ)
    cm = circ.matrices()
    ws = [fr_to_mont(synth.chain_witness(1 << 12, 5 + k)) for k in range(3)] + [fr_to_mont(synth.chain_witness(1 << 12, 0))]
    rs = _random_rs(random.Random(12), 4)
    expect = _singles(pk, cm, rs, ws, ctx)
    yield pk, cm, ws, rs, expect
    release(pk); release(cm)


@pytest.mark.parametrize('env', [
    {'B2G_MSM_C': '8', 'B2G_MSM_REDUCE_CHUNK': '1'},
    {'B2G_MSM_C': '8', 'B2G_MSM_REDUCE_CHUNK': '1000'},
    {'B2G_MSM_C': '13', 'B2G_MSM_REDUCE_CHUNK': '1'},
    {'B2G_MSM_C': '13', 'B2G_MSM_REDUCE_CHUNK': '1000'},
    {'B2G_MSM_CHUNK': '1'},
    {'B2G_MSM_CHUNK': '97', 'B2G_MSM_CHUNK_G2': '193'},
], ids=lambda e: ','.join(f'{k[8:]}={v}' for k, v in e.items()))
def test_bucket_layout_variants(monkeypatch, chain12, env):
    """window sizes, reduce chunks and run lengths whose runs straddle proof boundaries over count * nb buckets: a fresh
    context (and key tables) built under each setting"""
    from circom_compat_b200 import Context, release
    pk, cm, ws, rs, expect = chain12
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    release(pk)                                                        # B2G_MSM_C is read when the key's tables are built
    cx = Context(0)
    try:
        assert _many(pk, cm, rs, ws, cx) == expect
    finally:
        cx.close()
        release(pk)


def test_graph_direct_regrowth_and_recapture(ctx, monkeypatch, golden, complex_key, chain_witnesses):
    """direct launches (B2G_GRAPH=0) and the captured graph agree on a batch; one context runs count 3 -> 5 -> 3 -> single
    -> 3, re-capturing per count and growing its buffers once"""
    from circom_compat_b200 import Context
    pk, cm = complex_key
    g = golden['complex_zkey']
    rs = _random_rs(random.Random(35), 5)
    ws = chain_witnesses[:5]
    expect = _singles(pk, cm, rs, ws, ctx)
    monkeypatch.setenv('B2G_GRAPH', '0')
    direct = Context(0)
    monkeypatch.delenv('B2G_GRAPH')
    graph = Context(0)
    assert _many(pk, cm, rs[:3], ws[:3], direct) == expect[:3]
    for n in (3, 5, 3):
        assert _many(pk, cm, rs[:n], ws[:n], graph) == expect[:n]
    assert _singles(pk, cm, [(int(g['r']), int(g['s']))], [chain_witnesses[0]], graph)[0].hex() == g['proof_hex']
    assert _many(pk, cm, rs[2:5], ws[2:5], graph) == expect[2:5]
    direct.close(); graph.close()


def test_2p20_batch_closed_form(ctx):
    """two 2^20 chain proofs in one pass (31 M sorted entries per witness query) against the trapdoor closed form"""
    from circom_compat_b200 import fr_to_mont, synth, release
    circ = synth.chain_circuit(1 << 20)
    pk, td = synth.setup(ctx, circ)
    cm = circ.matrices()
    wl = [synth.chain_witness(1 << 20, a) for a in (3, 11)]
    rs = [(0x1234567890abcdef, 0xfedcba0987654321), (o.R_MOD - 1, 1)]
    got = _many(pk, cm, rs, [fr_to_mont(w) for w in wl], ctx)
    from circom_compat_b200 import Proof
    from oracle import cref as c
    for d, w, (r, s) in zip(got, wl, rs):
        da, db, dc = synth.expected_proof_dlogs_independent(td, circ, w, r, s)
        ea = c.limbs_to_ints(c.fq_from_mont(c.fixed_base_g1(c.ints_to_limbs([da, dc]))))
        eb = c.limbs_to_ints(c.fq_from_mont(c.fixed_base_g2(c.ints_to_limbs([db]))))
        p = Proof(d)
        assert p.a == (ea[0], ea[1]) and p.c == (ea[2], ea[3]) and p.b == ((eb[0], eb[1]), (eb[2], eb[3]))
    release(pk); release(cm)


def _pick_c(n):
    # msm.cuh msm_pick_c
    if n >= 3 << 18: return 17
    if n >= 1 << 19: return 16
    if n >= 1 << 15: return 15
    if n >= 1 << 13: return 13
    if n >= 1 << 11: return 11
    return max(8, n.bit_length() - 1 - 3)


def test_errors_leave_the_context_usable(ctx, golden, complex_key, chain_witnesses):
    from circom_compat_b200 import Context, B2gError, _native as N
    pk, cm = complex_key
    g = golden['complex_zkey']
    L = N.lib()
    ph, mh = ctx.pk_handle(pk), ctx.mat_handle(cm, pk.n_vars)
    w = chain_witnesses[0]

    def call(cx_h, count, ptrs):
        rr = np.zeros(4 * max(count, 1), dtype=np.uint64)
        out = np.zeros(256 * max(count, 1), dtype=np.uint8)
        return L.b2g_prove_many(cx_h, ph, mh, count, rr.ctypes.data, rr.ctypes.data, ptrs, out.ctypes.data)

    def last():
        return L.b2g_last_error().decode()

    one = (C.c_void_p * 1)(w.ctypes.data)
    rr = np.zeros(4, dtype=np.uint64)
    out = np.zeros(256, dtype=np.uint8)
    assert L.b2g_prove_many(ctx._h, ph, mh, 1, None, rr.ctypes.data, one, out.ctypes.data) == N.B2G_E_SHAPE
    assert last() == "null pointer"
    assert L.b2g_prove_many(ctx._h, ph, mh, 1, rr.ctypes.data, rr.ctypes.data, None, out.ctypes.data) == N.B2G_E_SHAPE
    assert last() == "null pointer"
    for count in (0, 65536):
        assert call(ctx._h, count, one) == N.B2G_E_SHAPE
        assert last() == "b2g_prove_many: count must be in [1, 65535]"
    assert call(ctx._h, 2, (C.c_void_p * 2)(w.ctypes.data, None)) == N.B2G_E_SHAPE
    assert last() == "null witness 1"
    from circom_compat_b200 import Groth16
    sharded = Context(0, 0, 2)
    with pytest.raises(B2gError) as e:
        Groth16.create_proofs(pk, [(1, 2)], cm, [w], sharded)
    assert e.value.code == N.B2G_E_SHAPE
    assert e.value.msg == "a whole proof (b2g_prove, b2g_prove_many) needs an unsharded context; use b2g_prove_partial/finish"
    sharded.close()
    pending = Groth16.submit(pk, int(g['r']), int(g['s']), cm, w, ctx)
    assert call(ctx._h, 1, one) == N.B2G_E_SHAPE
    assert last() == "a submitted proof is still pending on this context: call b2g_prove_wait first"
    assert pending.wait().data.hex() == g['proof_hex']
    # a count at which the witness queries (n_vars - 1 bases each) reach 2^32 sorted entries
    n = pk.n_vars - 1
    c = _pick_c(n)
    nwin = -(-255 // c)
    count = -(-(1 << 32) // (n * nwin))
    assert count <= 65535
    many = (C.c_void_p * count)(*([w.ctypes.data] * count))
    assert call(ctx._h, count, many) == N.B2G_E_SHAPE
    assert last() == "b2g_prove_many: count x bases x windows of a query reaches 2^32 sorted entries; prove fewer per call"
    p = _many(pk, cm, [(int(g['r']), int(g['s']))] * 2, [w, w], ctx)
    assert p[0].hex() == g['proof_hex'] and p[1] == p[0]


def test_cpp_mirror_create_proofs(golden, complex_key, chain_witnesses, ctx):
    """Groth16T::create_proofs through groth16_bench (B2G_MANY=3: chain witnesses a, a + 1, a + 2 with the golden (r, s))
    gives the same bytes as the Python path"""
    pk, cm = complex_key
    g = golden['complex_zkey']
    exe = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench')
    out = subprocess.check_output([exe, os.path.join(ROOT, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'), 'chain:%d' % int(g['a']), '1',
                                   '%x' % int(g['r']), '%x' % int(g['s'])], text=True, env=dict(os.environ, B2G_MANY='3'))
    lines = dict(l.split('=', 1) for l in out.splitlines() if l.startswith('many['))
    rs = [(int(g['r']), int(g['s']))] * 3
    py = _many(pk, cm, rs, chain_witnesses[:3], ctx)
    assert [lines['many[%d]' % i] for i in range(3)] == [d.hex() for d in py]
    assert py[0].hex() == g['proof_hex'] and 'first_identical=1' in out
