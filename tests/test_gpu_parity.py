"""GPU parity tests: every call goes through the C ABI (libb2groth.so) and is compared bit-for-bit with the oracle
(oracle/cref.c restatement, oracle/pyref.py big-int) on the same inputs.  Integer work => exact equality."""
import hashlib
import os
import random

import numpy as np
import pytest

from oracle import cref as c
from oracle import msm_digits as md
from oracle import pyref as o
from oracle import xyzz as X

pytestmark = pytest.mark.gpu


def _rand_fe(rng, n, mod, extra=()):
    vals = [rng.randrange(mod) for _ in range(n)] + list(extra)
    return vals


# ------------------------------------------------------------------------------------------------ field layer
@pytest.mark.parametrize('field', ['fq', 'fr'])
def test_field_ops(ctx, field):
    rng = random.Random(11)
    mod = o.Q_MOD if field == 'fq' else o.R_MOD
    to_m = c.fq_to_mont if field == 'fq' else c.fr_to_mont
    from_m = c.fq_from_mont if field == 'fq' else c.fr_from_mont
    base = 0 if field == 'fq' else 3
    edge = [0, 1, 2, mod - 1, mod - 2, (1 << 253), (1 << 254) % mod, mod >> 1]
    a = _rand_fe(rng, 3000, mod, edge + edge)
    b = _rand_fe(rng, 3000, mod, edge + edge[::-1])
    am, bm = to_m(c.ints_to_limbs(a)), to_m(c.ints_to_limbs(b))
    assert c.limbs_to_ints(from_m(ctx.test_op(base + 0, am, bm))) == [x * y % mod for x, y in zip(a, b)]
    assert c.limbs_to_ints(from_m(ctx.test_op(base + 1, am, bm))) == [(x + y) % mod for x, y in zip(a, b)]
    assert c.limbs_to_ints(from_m(ctx.test_op(base + 2, am, bm))) == [(x - y) % mod for x, y in zip(a, b)]
    nz = [x for x in a if x][:64]
    inv = ctx.test_op(6 if field == 'fq' else 7, to_m(c.ints_to_limbs(nz)))
    assert c.limbs_to_ints(from_m(inv)) == [pow(x, -1, mod) for x in nz]


def _raw_residues(rng, n, mod):
    """Raw Montgomery residues (any integer < mod) with extreme limb patterns mixed in."""
    pat = [0, 1, 0xffffffff, 0xfffffffe, 0x80000000, 0x7fffffff]
    out = [0, 1, mod - 1, mod - 2, mod >> 1, (1 << 253) - 1, 1 << 253]
    while len(out) < n:
        if rng.random() < 0.5:
            out.append(rng.randrange(mod))
        else:
            v = sum(rng.choice(pat + [rng.getrandbits(32)]) << (32 * i) for i in range(8)) % mod
            out.append(v)
    return out[:n]


def test_lazy_reduction_blocks(ctx):
    """sqr / mul_wide / redc / mul_sub and the Fq2 routines built on them, on raw residues: out = x*y*R^-1 mod q."""
    rng = random.Random(77)
    q = o.Q_MOD
    rinv = pow(1 << 256, -1, q)
    n = 4000
    x, y = _raw_residues(rng, n, q), _raw_residues(rng, n, q)[::-1]
    xl, yl = c.ints_to_limbs(x), c.ints_to_limbs(y)
    assert c.limbs_to_ints(ctx.test_op(14, xl, yl)) == [a * a * rinv % q for a in x]
    assert c.limbs_to_ints(ctx.test_op(15, xl, yl)) == [(a * b - b * b) * rinv % q for a, b in zip(x, y)]
    assert c.limbs_to_ints(ctx.test_op(16, xl, yl)) == [a * b * rinv % q for a, b in zip(x, y)]
    assert c.limbs_to_ints(ctx.test_op(0, xl, yl)) == [a * b * rinv % q for a, b in zip(x, y)]
    # Fq2 = Fq[u]/(u^2+1): elements are consecutive pairs
    x2 = list(zip(x[0::2], x[1::2])); y2 = list(zip(y[0::2], y[1::2]))

    def mul2(a, b):
        return ((a[0] * b[0] - a[1] * b[1]) * rinv % q, (a[0] * b[1] + a[1] * b[0]) * rinv % q)

    def flat(v):
        return [t for pair in v for t in pair]

    assert c.limbs_to_ints(ctx.test_op(17, xl, yl)) == flat([mul2(a, b) for a, b in zip(x2, y2)])
    assert c.limbs_to_ints(ctx.test_op(18, xl, yl)) == flat([mul2(a, a) for a in x2])
    exp = []
    for a, b in zip(x2, y2):
        p1, p2 = mul2(a, b), mul2(b, (a[1], a[0]))
        exp.append(((p1[0] - p2[0]) % q, (p1[1] - p2[1]) % q))
    assert c.limbs_to_ints(ctx.test_op(19, xl, yl)) == flat(exp)
    # the inlined Karatsuba the G2 accumulation runs (row products); pairs such as (q-1, q-2) make a0 + a1 close to 2q
    assert c.limbs_to_ints(ctx.test_op(28, xl, yl)) == flat([mul2(a, b) for a, b in zip(x2, y2)])
    # Fq::mul_wide over its whole input range: a < 2^255 (Karatsuba passes a0 + a1 < 2q), b any 256-bit value
    m = 0xffffffff
    wa = [0, 1, q - 1, q, 2 * q - 2, 2 * q - 1, (1 << 255) - 1, 1 << 254, (1 << 255) - (1 << 224), (m >> 1) << 224]
    wb = [(1 << 256) - 1, 0, 1, (1 << 256) - 1, (1 << 256) - 1, q - 1, (1 << 256) - 1, (1 << 256) - 1, m, 1 << 255]
    while len(wa) < 3000:
        wa.append(sum(rng.choice([0, 1, m, m - 1, 0x80000000, 0x7fffffff, rng.getrandbits(32)]) << (32 * i) for i in range(8)) % (1 << 255)
                  if rng.random() < 0.5 else rng.randrange(1 << 255))
        wb.append(sum(rng.choice([0, 1, m, m - 1, 0x80000000, rng.getrandbits(32)]) << (32 * i) for i in range(8))
                  if rng.random() < 0.5 else rng.getrandbits(256))
    got = c.limbs_to_ints(ctx.test_op(29, c.ints_to_limbs(wa), c.ints_to_limbs(wb)))
    assert [lo | (hi << 256) for lo, hi in zip(got[0::2], got[1::2])] == [a * b for a, b in zip(wa, wb)]


def test_group_ops(ctx):
    rng = random.Random(5)
    n = 200
    ka = [rng.randrange(1, o.R_MOD) for _ in range(n)]
    kb = [rng.randrange(1, o.R_MOD) for _ in range(n)]
    kb[0] = ka[0]                      # P + P  -> doubling branch
    kb[1] = o.R_MOD - ka[1]            # P + (-P) -> infinity
    pa, pb = c.fixed_base_g1(c.ints_to_limbs(ka)), c.fixed_base_g1(c.ints_to_limbs(kb))
    pa[2] = 0; pb[3] = 0; pa[4] = 0; pb[4] = 0      # infinities on either / both sides
    exp = np.stack([c.add_g1(x, y) for x, y in zip(pa, pb)])
    assert np.array_equal(ctx.test_op(8, pa, pb), exp)          # full XYZZ addition
    assert np.array_equal(ctx.test_op(12, pa, pb), exp)         # mixed addition
    assert np.array_equal(ctx.test_op(10, pa), np.stack([c.add_g1(x, x) for x in pa]))
    qa, qb = c.fixed_base_g2(c.ints_to_limbs(ka[:60])), c.fixed_base_g2(c.ints_to_limbs(kb[:60]))
    qa[2] = 0; qb[3] = 0
    exp2 = np.stack([c.add_g2(x, y) for x, y in zip(qa, qb)])
    assert np.array_equal(ctx.test_op(9, qa, qb), exp2)
    assert np.array_equal(ctx.test_op(13, qa, qb), exp2)
    assert np.array_equal(ctx.test_op(11, qa), np.stack([c.add_g2(x, x) for x in qa]))
    # Curve::add / madd / dbl on raw XYZZ records (ops 20-25): projective operands on every exceptional branch, the result
    # checked as a record (ZZ^3 = ZZZ^2, X = x ZZ, Y = y ZZZ), not through an affine conversion
    for g2, rows in ((False, pa[5:12]), (True, qa[5:12])):
        pts = [X.aff(r, g2) for r in rows]
        curve = o.G2 if g2 else o.G1
        cases = X.addition_cases(rng, g2, pts)
        zs = X.z_values(rng, g2)
        acc = np.stack([X.record(P, z, g2) for _, P, z, _ in cases])
        q_rec = np.stack([X.record(Q, zs[(i + 3) % len(zs)], g2) for i, (_, _, _, Q) in enumerate(cases)])   # projective q too
        q_aff = np.stack([X.aff_row(Q, g2) for _, _, _, Q in cases])
        base = 23 if g2 else 20
        for op, b, exp in ((base, q_rec, [curve.add(P, Q) for _, P, _, Q in cases]),
                           (base + 1, q_aff, [curve.add(P, Q) for _, P, _, Q in cases]),
                           (base + 2, None, [curve.add(P, P) for _, P, _, _ in cases])):
            out = ctx.test_op(op, acc, b)
            bad = [(i, cases[i][0], err) for i in range(len(cases)) if (err := X.check_record(out[i], exp[i], g2))]
            assert not bad, (op, len(bad), bad[:6])


def test_fixed_base(ctx):
    rng = random.Random(2)
    ks = [0, 1, 2, o.R_MOD - 1] + [rng.randrange(o.R_MOD) for _ in range(300)]
    lim = c.ints_to_limbs(ks)
    assert np.array_equal(ctx.fixed_base_g1(lim), c.fixed_base_g1(lim))
    assert np.array_equal(ctx.fixed_base_g2(lim[:80]), c.fixed_base_g2(lim[:80]))


# ------------------------------------------------------------------------------------------------ NTT
# 21 / 22: the >= 2^21 pass schedule (block pass + two 2-D strided passes of <= 7 index bits, ntt.cu ntt_domain_create) that the
# 2^22 configuration (BASELINE.json config 4) runs; 1..4 run the one-stage-per-barrier kernel, 5 and up the radix-8 register rounds
@pytest.mark.parametrize('log_n', [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 16, 20, 21, 22])
def test_ntt_plain(ctx, log_n):
    rng = np.random.default_rng(log_n)
    n = 1 << log_n
    vals = c.fr_to_mont(c.ints_to_limbs([int(x) for x in rng.integers(0, 2**62, n)]))      # any residues will do
    vals = c.fr_mul(vals, vals[::-1].copy())                                                 # spread over the field
    assert np.array_equal(ctx.ntt(vals), c.ntt(vals))
    assert np.array_equal(ctx.ntt(vals, inverse=True), c.ntt(vals, inverse=True))


# every pass shape of ntt_domain_create: the radix-2 kernel (B2G_NTT_RADIX2=1), small tiles (many strided passes, partial
# rounds), 2-D strided tiles (B2G_NTT_MAXK), 512- and 2048-element tiles at sizes where they are not the default
@pytest.mark.parametrize('env', [dict(B2G_NTT_RADIX2='1'), dict(B2G_NTT_TL='5'), dict(B2G_NTT_TL='6', B2G_NTT_MAXK='2'),
                                 dict(B2G_NTT_TL='7', B2G_NTT_MAXK='4'), dict(B2G_NTT_TL='9'), dict(B2G_NTT_TL='11'),
                                 dict(B2G_NTT_MAXK='5'), dict(B2G_NTT_RADIX2='1', B2G_NTT_MAXK='5')],
                         ids=lambda e: ','.join('%s=%s' % (k[8:], v) for k, v in e.items()))
@pytest.mark.parametrize('log_n', [9, 13, 17])
def test_ntt_pass_schedules(ctx, monkeypatch, env, log_n):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(1000 + log_n)
    n = 1 << log_n
    vals = c.fr_to_mont(c.ints_to_limbs([int(x) for x in rng.integers(0, 2**62, n)]))
    vals = c.fr_mul(vals, vals[::-1].copy())
    assert np.array_equal(ctx.ntt(vals), c.ntt(vals))
    assert np.array_equal(ctx.ntt(vals, inverse=True), c.ntt(vals, inverse=True))


@pytest.mark.parametrize('env', [dict(B2G_NTT_RADIX2='1'), dict(B2G_NTT_TL='6', B2G_NTT_MAXK='3'), dict(B2G_NTT_TL='11'), dict(B2G_NTT_MAXK='5')],
                         ids=lambda e: ','.join('%s=%s' % (k[8:], v) for k, v in e.items()))
def test_witness_map_pass_schedules(ctx, monkeypatch, env):
    # the fused chain (DIF passes, DIF + coset scale + DIT block pass, DIT passes + h = a*b - c) under every pass shape,
    # CircomReduction and LibsnarkReduction, against oracle/cref.c
    from circom_compat_b200 import CircomReduction, LibsnarkReduction, fr_to_mont, synth, release
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    log_n = 13
    circ = synth.chain_circuit(1 << log_n); w = synth.chain_witness(1 << log_n)
    wm = fr_to_mont(w)
    cm = circ.matrices()
    h = CircomReduction.witness_map_from_matrices(cm, circ.num_inputs, circ.num_constraints, wm, ctx)
    assert np.array_equal(h, c.witness_map(cm.num_constraints, circ.num_inputs, circ.n_vars, cm.a, cm.b, wm))
    release(cm)
    cm3 = circ.matrices(with_c=True)
    h = LibsnarkReduction.witness_map_from_matrices(cm3, circ.num_inputs, circ.num_constraints, wm, ctx)
    assert np.array_equal(h, c.witness_map_libsnark(cm3.num_constraints, cm3.num_instance_variables, cm3.a, cm3.b, cm3.c, wm))
    release(cm3)


def test_ntt_linearity_large(ctx):
    # size-independent property at the headline size: NTT(a + b) = NTT(a) + NTT(b), iNTT(NTT(a)) = a
    log_n = 20
    n = 1 << log_n
    rng = np.random.default_rng(99)
    raw = rng.integers(0, 2**63, (2, n, 4), dtype=np.uint64); raw[..., 3] &= (1 << 60) - 1   # < r
    a, b = raw[0], raw[1]
    fa, fb = ctx.ntt(a), ctx.ntt(b)
    s = ctx.test_op(4, a, b)
    assert np.array_equal(ctx.ntt(s), ctx.test_op(4, fa, fb))
    assert np.array_equal(ctx.ntt(fa, inverse=True), a)


# ------------------------------------------------------------------------------------------------ MSM
def _msm_case(rng, n, dist):
    ks = [rng.randrange(1, o.R_MOD) for _ in range(n)]
    if dist == 'uniform':
        sc = [rng.randrange(o.R_MOD) for _ in range(n)]
    elif dist == 'circomlike':      # 60 % bits, 20 % small, 20 % wide
        sc = [rng.randrange(2) if (u := rng.random()) < 0.6 else (rng.randrange(1 << 32) if u < 0.8 else rng.randrange(o.R_MOD)) for _ in range(n)]
    elif dist == 'ones':
        sc = [1] * n
    elif dist == 'same':
        v = rng.randrange(o.R_MOD); sc = [v] * n
    else:
        sc = [0] * n
    return ks, sc


@pytest.mark.parametrize('n,dist', [(1, 'uniform'), (2, 'uniform'), (3, 'ones'), (33, 'uniform'), (257, 'zeros'), (1000, 'circomlike'),
                                    (4096, 'uniform'), (5000, 'same'), (70000, 'uniform'), (70000, 'circomlike'), (70000, 'ones')])
def test_msm_g1(ctx, n, dist):
    rng = random.Random(n * 7 + len(dist))
    ks, sc = _msm_case(rng, n, dist)
    bases = c.fixed_base_g1(c.ints_to_limbs(ks))
    if n > 40:
        bases[5] = 0; bases[9] = bases[8]; sc[8] = 5; sc[9] = o.R_MOD - 5; sc[0] = 0; sc[1] = 1; sc[2] = o.R_MOD - 1
    scl = c.ints_to_limbs(sc)
    exp = c.msm_g1(bases, scl)
    assert np.array_equal(ctx.msm_g1(bases, scl), exp)
    assert np.array_equal(ctx.msm_g1(bases, c.fr_to_mont(scl), scalars_mont=True), exp)


@pytest.mark.parametrize('n,dist', [(1, 'uniform'), (3, 'ones'), (300, 'circomlike'), (5000, 'uniform'), (5000, 'same'), (40000, 'circomlike')])
def test_msm_g2(ctx, n, dist):
    rng = random.Random(n * 13 + len(dist))
    ks, sc = _msm_case(rng, n, dist)
    bases = c.fixed_base_g2(c.ints_to_limbs(ks))
    if n > 40:
        bases[5] = 0; bases[9] = bases[8]; sc[8] = 5; sc[9] = o.R_MOD - 5
    scl = c.ints_to_limbs(sc)
    assert np.array_equal(ctx.msm_g2(bases, scl), c.msm_g2(bases, scl))


def test_msm_small_chunks_exercise_fragments(ctx, monkeypatch):
    # tiny runs (B2G_MSM_CHUNK) force buckets to straddle many threads, including the whole-CTA fold path
    rng = random.Random(77)
    n = 6000
    ks, sc = _msm_case(rng, n, 'circomlike')
    bases = c.fixed_base_g1(c.ints_to_limbs(ks)); scl = c.ints_to_limbs(sc)
    exp = c.msm_g1(bases, scl)
    for chunk in ('1', '2', '3', '7'):
        monkeypatch.setenv('B2G_MSM_CHUNK', chunk)
        assert np.array_equal(ctx.msm_g1(bases, scl), exp), chunk
    # the bulk-copied entry slab around its size limit (128 runs x 96 entries = 48 KB per CTA): up to 96 entries per run it
    # is staged, from 97 the runs read the entry list directly; the entry count is not a multiple of 4, so the last CTA's
    # slab is partial and its copy is rounded up
    monkeypatch.setenv('B2G_MSM_C', '11')
    m = md.partial_slab_prefix(sc, 11)
    exp_m = c.msm_g1(bases[:m], scl[:m])
    for chunk in ('1', '64', '96', '97'):
        monkeypatch.setenv('B2G_MSM_CHUNK', chunk)
        assert np.array_equal(ctx.msm_g1(bases[:m], scl[:m]), exp_m), chunk
    # the weighted bucket sum with every per-thread bucket count, at two window sizes
    monkeypatch.delenv('B2G_MSM_CHUNK')
    for cw in ('8', '13'):
        monkeypatch.setenv('B2G_MSM_C', cw)
        for rchunk in ('1', '3', '7', '1000'):
            monkeypatch.setenv('B2G_MSM_REDUCE_CHUNK', rchunk)
            assert np.array_equal(ctx.msm_g1(bases, scl), exp), (cw, rchunk)
    monkeypatch.delenv('B2G_MSM_REDUCE_CHUNK')
    # buckets spanning exactly MSM_BIG_FRAGS runs (msm_fold_kernel) and one more (msm_fold_big_kernel), starting on and off
    # a run boundary; then four equal points in runs of two: each fragment is 2P in projective form, the fold doubles it
    monkeypatch.setenv('B2G_MSM_C', '8')
    sc2, ch = md.fold_boundary_scalars(rng)
    monkeypatch.setenv('B2G_MSM_CHUNK', str(ch))
    bases2 = c.fixed_base_g1(c.ints_to_limbs([rng.randrange(1, o.R_MOD) for _ in range(len(sc2))]))
    scl2 = c.ints_to_limbs(sc2)
    assert np.array_equal(ctx.msm_g1(bases2, scl2), c.msm_g1(bases2, scl2))
    monkeypatch.setenv('B2G_MSM_CHUNK', '2')
    for v in (3, rng.randrange(o.R_MOD)):
        b4, s4 = np.stack([bases2[0]] * 4), c.ints_to_limbs([v] * 4)
        assert np.array_equal(ctx.msm_g1(b4, s4), c.msm_g1(b4, s4)), v


def test_msm_g1_two_entry_buckets(ctx):
    """Buckets that hold exactly two points make the XYZZ mixed addition's exceptional cases deterministic: P + P (the
    doubling branch), P + (-P) (sum at infinity), P + infinity and infinity + infinity; then four equal points."""
    rng = random.Random(4242)
    k = rng.randrange(1, o.R_MOD)
    P = c.fixed_base_g1(c.ints_to_limbs([k]))[0]
    Pn = c.fixed_base_g1(c.ints_to_limbs([o.R_MOD - k]))[0]                    # -P
    inf = np.zeros_like(P)
    for sv in (1, 5, rng.randrange(o.R_MOD), o.R_MOD - 1):
        scl = c.ints_to_limbs([sv, sv])
        for pair in ((P, P), (P, Pn), (P, inf), (inf, P), (inf, inf)):
            bases = np.stack(pair)
            assert np.array_equal(ctx.msm_g1(bases, scl), c.msm_g1(bases, scl)), sv
    bases = np.stack((P, P, P, P)); scl = c.ints_to_limbs([3, 3, 3, 3])
    assert np.array_equal(ctx.msm_g1(bases, scl), c.msm_g1(bases, scl))


def test_msm_truncation_rule(ctx):
    rng = random.Random(3)
    bases = c.fixed_base_g1(c.ints_to_limbs([rng.randrange(1, o.R_MOD) for _ in range(50)]))
    sc = c.ints_to_limbs([rng.randrange(o.R_MOD) for _ in range(31)])
    assert np.array_equal(ctx.msm_g1(bases, sc), c.msm_g1(bases[:31], sc))
    assert not ctx.msm_g1(bases[:0], sc[:0]).any()


# ------------------------------------------------------------------------------------------------ witness map + proofs
def test_witness_map_and_proofs_test_zkey(ctx, golden, test_zkey_bytes):
    # verify_proof_with_zkey_without_r1cs (src/zkey.rs:875-919) with pinned r, s
    from circom_compat_b200 import read_zkey, Groth16, CircomReduction, fr_to_mont, fr_from_mont
    pk, cm = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    w = [int(x) for x in g['witness']]
    wm = fr_to_mont(w)
    h = CircomReduction.witness_map_from_matrices(cm, cm.num_instance_variables, cm.num_constraints, wm, ctx)
    assert [str(x) for x in fr_from_mont(h)] == g['h']
    z = o.read_zkey(test_zkey_bytes)
    for i, case in enumerate(g['proofs']):
        p = Groth16.create_proof_with_reduction_and_matrices(pk, int(case['r']), int(case['s']), cm, cm.num_instance_variables,
                                                             cm.num_constraints, wm, ctx)
        assert p.data.hex() == case['proof_hex'], i
        if i == 0:
            # src/zkey.rs:868-872: process_vk + verify_with_processed_vk on the product's own host verifier; the oracle's
            # (differently built) pairing must agree
            pvk = Groth16.process_vk(pk)
            assert Groth16.verify_with_processed_vk(pvk, w[1:cm.num_instance_variables], p)
            assert not Groth16.verify_with_processed_vk(pvk, [34], p)
            assert o.verify(z, w[1:cm.num_instance_variables], (p.a, p.b, p.c))


def test_witness_map_and_proof_complex_zkey(ctx, golden, complex_zkey_bytes):
    # the reference's bench workload (benches/groth16.rs:13-85): 10 000-constraint chain, domain 2^14
    from circom_compat_b200 import read_zkey, Groth16, CircomReduction, fr_to_mont
    pk, cm = read_zkey(complex_zkey_bytes)
    g = golden['complex_zkey']
    w = o.chain_witness(pk.n_vars, g['a'])
    wm = fr_to_mont(w)
    h = CircomReduction.witness_map_from_matrices(cm, cm.num_instance_variables, cm.num_constraints, wm, ctx)
    hc = c.fr_from_mont(h)
    assert [str(x) for x in c.limbs_to_ints(hc[:4])] == g['h_head']
    assert hashlib.sha256(np.ascontiguousarray(hc).tobytes()).hexdigest() == g['h_sha256_canon_le']
    p = Groth16.create_proof_with_reduction_and_matrices(pk, int(g['r']), int(g['s']), cm, cm.num_instance_variables, cm.num_constraints, wm, ctx)
    assert p.data.hex() == g['proof_hex']


def _synthetic(ctx, kind, log_n):
    from circom_compat_b200 import synth
    if kind == 'chain':
        circ = synth.chain_circuit(1 << log_n); w = synth.chain_witness(1 << log_n)
    else:
        circ, w = synth.circomlike_circuit(log_n)
    pk, td = synth.setup(ctx, circ)
    return circ, w, pk, td


def _oracle_key(pk, cm):
    za = dict(n_vars=pk.n_vars, n_public=pk.n_public, domain_size=pk.domain_size, num_constraints=cm.num_constraints, a_csr=cm.a, b_csr=cm.b)
    for name in ('alpha_g1', 'beta_g1', 'delta_g1', 'beta_g2', 'delta_g2', 'a_query', 'b_g1_query', 'b_g2_query', 'l_query', 'h_query'):
        za[name] = np.ascontiguousarray(getattr(pk, name), dtype=np.uint64)
    return za


@pytest.mark.parametrize('kind,log_n', [('chain', 12), ('circomlike', 13), ('chain', 16)])
def test_synthetic_proof_vs_oracle_and_trapdoor(ctx, kind, log_n):
    # BASELINE.json config 2 (2^16, MSM + NTT correctness vs CPU) and smaller shapes
    from circom_compat_b200 import Groth16, CircomReduction, fr_to_mont, fr_from_mont, synth
    circ, w, pk, td = _synthetic(ctx, kind, log_n)
    cm = circ.matrices()
    # spot-check GPU-generated bases against the oracle's fixed-base multiplication
    rng = random.Random(log_n)
    for i in [0, 1, pk.n_vars - 1] + [rng.randrange(pk.n_vars) for _ in range(20)]:
        assert np.array_equal(pk.a_query[i], c.fixed_base_g1(c.ints_to_limbs([td.a_t[i]]))[0])
        assert np.array_equal(pk.b_g2_query[i], c.fixed_base_g2(c.ints_to_limbs([td.b_t[i]]))[0])
    wm = fr_to_mont(w)
    r, s = rng.randrange(o.R_MOD), rng.randrange(o.R_MOD)
    h = CircomReduction.witness_map_from_matrices(cm, circ.num_inputs, circ.num_constraints, wm, ctx)
    p = Groth16.create_proof_with_reduction_and_matrices(pk, r, s, cm, circ.num_inputs, circ.num_constraints, wm, ctx)
    pb, h_ref = c.prove(_oracle_key(pk, cm), r, s, wm, want_h=True)
    assert np.array_equal(h, h_ref)
    assert p.data == pb
    da, db, dc = synth.expected_proof_dlogs(td, w, fr_from_mont(h), r, s, circ.num_inputs)
    assert o.G1.mul(o.G1_GEN, da) == p.a and o.G2.mul(o.G2_GEN, db) == p.b and o.G1.mul(o.G1_GEN, dc) == p.c
    # and the form that takes no h at all: H term = (a(tau) b(tau) - c(tau)) / delta straight from the trapdoor
    assert synth.expected_proof_dlogs_independent(td, circ, w, r, s) == (da, db, dc)


def test_submit_wait_pipelines_proofs_on_one_thread(golden, complex_zkey_bytes):
    """b2g_prove_submit / b2g_prove_wait: three contexts, one host thread, proofs with different (r, s) in flight at once
    (the captured proof graph is replayed with new r, s and witness each time); results equal the synchronous call's."""
    from circom_compat_b200 import read_zkey, Groth16, fr_to_mont, Context, B2gError
    pk, cm = read_zkey(complex_zkey_bytes)
    g = golden['complex_zkey']
    wm = fr_to_mont(o.chain_witness(pk.n_vars, g['a']))
    ctxs = [Context(0) for _ in range(3)]
    rs = [(int(g['r']), int(g['s'])), (5, 7), (0, 11), (o.R_MOD - 1, 3), (int(g['r']), int(g['s'])), (1, 0)]
    expect = [Groth16.create_proof_with_reduction_and_matrices(pk, r, s, cm, cm.num_instance_variables, cm.num_constraints, wm, ctxs[0]).data for r, s in rs]
    assert expect[0].hex() == g['proof_hex'] and expect[4] == expect[0] and len(set(expect)) == 5
    pend, got = {}, []
    for k, (r, s) in enumerate(rs):
        j = k % 3
        if j in pend:
            got.append(pend.pop(j).wait().data)
        pend[j] = Groth16.submit(pk, r, s, cm, wm, ctxs[j])
    with pytest.raises(B2gError):                                  # one pending proof per context
        Groth16.submit(pk, 1, 1, cm, wm, ctxs[0])
    for j in (0, 1, 2):
        got.append(pend.pop(j).wait().data)
    assert got == expect
    for cx in ctxs:
        cx.close()


def test_graph_and_direct_launch_paths_agree(golden, complex_zkey_bytes, monkeypatch):
    """The captured proof graph (default) and direct launches (B2G_GRAPH=0 at context creation) are the same pipeline: same
    golden bytes; a context switches keys (re-capture on a new key uid) and comes back."""
    from circom_compat_b200 import read_zkey, Groth16, fr_to_mont, Context
    pk, cm = read_zkey(complex_zkey_bytes)
    g = golden['complex_zkey']
    wm = fr_to_mont(o.chain_witness(pk.n_vars, g['a']))
    monkeypatch.setenv('B2G_GRAPH', '0')
    direct = Context(0)
    monkeypatch.delenv('B2G_GRAPH')
    graph = Context(0)
    for cx in (direct, graph, graph, direct):
        p = Groth16.create_proof_with_reduction_and_matrices(pk, int(g['r']), int(g['s']), cm, cm.num_instance_variables, cm.num_constraints, wm, cx)
        assert p.data.hex() == g['proof_hex']
    t = direct.last_timings()
    assert t['witness_map'] > 0 and t['msm_b2'] > 0                  # interior phase timers exist only without the graph
    assert graph.last_timings()['msm_b2'] < 0.05 < graph.last_timings()['total']     # no interior events inside the graph
    # another key on the same contexts, then the first one again
    from circom_compat_b200 import synth
    circ = synth.chain_circuit(1 << 10); w2 = synth.chain_witness(1 << 10)
    pk2, td = synth.setup(graph, circ); cm2 = circ.matrices()
    p2 = Groth16.create_proof_with_reduction_and_matrices(pk2, 3, 4, cm2, circ.num_inputs, circ.num_constraints, fr_to_mont(w2), graph)
    assert p2.data == c.prove(_oracle_key(pk2, cm2), 3, 4, fr_to_mont(w2))
    p = Groth16.create_proof_with_reduction_and_matrices(pk, int(g['r']), int(g['s']), cm, cm.num_instance_variables, cm.num_constraints, wm, graph)
    assert p.data.hex() == g['proof_hex']
    direct.close(); graph.close()


def test_sparse_b_compaction_matches_uncompacted(ctx, monkeypatch):
    """Keys whose B query is mostly points at infinity (real circom keys; here the circom-like circuit: B touches 768 of ~9 000
    wires) are proved over the compacted B bases with their own scalar sort; same bytes as with compaction disabled and as the
    CPU oracle, also when the shard ranges cut the key in three."""
    from circom_compat_b200 import Groth16, fr_to_mont, synth, release, Context
    circ, w = synth.circomlike_circuit(13)
    pk, td = synth.setup(ctx, circ)
    nb = int(np.count_nonzero(np.asarray(pk.b_g1_query).reshape(pk.n_vars, -1).any(axis=1)))
    assert nb * 5 < pk.n_vars                                          # sparse enough for the compacted path
    cm = circ.matrices()
    wm = fr_to_mont(w)
    r, s = 0xabcdef0123, 0x456789
    ref = c.prove(_oracle_key(pk, cm), r, s, wm)
    p1 = Groth16.create_proof_with_reduction_and_matrices(pk, r, s, cm, circ.num_inputs, circ.num_constraints, wm, ctx)
    parts, ctxs = [], []
    for rank in range(3):
        cx = Context(0, rank, 3); ctxs.append(cx)
        parts.append(Groth16.prove_partial(pk, cm, wm, cx))
    p3 = Groth16.prove_finish(pk, np.stack(parts), r, s, ctxs[0])
    release(pk)
    monkeypatch.setenv('B2G_NO_B_COMPACT', '1')
    p2 = Groth16.create_proof_with_reduction_and_matrices(pk, r, s, cm, circ.num_inputs, circ.num_constraints, wm, ctx)
    assert p1.data == ref and p2.data == ref and p3.data == ref
    release(pk); release(cm)
    for cx in ctxs:
        cx.close()


def test_sharded_proof_equals_whole_proof(golden, complex_zkey_bytes):
    # base-range sharding on one device: 3 shard contexts, partials folded in rank order
    from circom_compat_b200 import read_zkey, Groth16, fr_to_mont, Context
    pk, cm = read_zkey(complex_zkey_bytes)
    g = golden['complex_zkey']
    wm = fr_to_mont(o.chain_witness(pk.n_vars, g['a']))
    parts, ctxs = [], []
    for rank in range(3):
        cx = Context(0, rank, 3); ctxs.append(cx)
        parts.append(Groth16.prove_partial(pk, cm, wm, cx))
    p = Groth16.prove_finish(pk, np.stack(parts), int(g['r']), int(g['s']), ctxs[1])
    assert p.data.hex() == g['proof_hex']
    for cx in ctxs:
        cx.close()


def test_error_behaviour(ctx, test_zkey_bytes, complex_zkey_bytes):
    from circom_compat_b200 import read_zkey, Groth16, fr_to_mont, B2gError, _native as N
    import ctypes as C
    pk, cm = read_zkey(test_zkey_bytes)
    with pytest.raises(ValueError) as v:
        Groth16.create_proof_with_reduction_and_matrices(pk, 1, 1, cm, cm.num_instance_variables, cm.num_constraints, fr_to_mont([1, 2, 3]), ctx)
    assert str(v.value) == "full_assignment length != n_vars"
    with pytest.raises(B2gError) as e:
        ctx.test_op(99, np.zeros((1, 4), dtype=np.uint64))            # unknown op: B2G_E_SHAPE, nothing launched
    assert e.value.code == -2 and e.value.msg == "bad arguments"
    # b2g_prove: null pointers, and a key with another circuit's matrices
    L = N.lib()
    w = fr_to_mont([1, 33, 3, 11])
    rr = np.zeros(4, dtype=np.uint64)
    out = np.zeros(256, dtype=np.uint8)
    pkc, cmc = read_zkey(complex_zkey_bytes)
    ph, mh, mhc = ctx.pk_handle(pk), ctx.mat_handle(cm, pk.n_vars), ctx.mat_handle(cmc, pkc.n_vars)
    assert L.b2g_prove(ctx._h, ph, mh, None, rr.ctypes.data, w.ctypes.data, out.ctypes.data) == N.B2G_E_SHAPE
    assert L.b2g_last_error().decode() == "null pointer"
    assert L.b2g_prove(ctx._h, ph, mh, rr.ctypes.data, rr.ctypes.data, None, out.ctypes.data) == N.B2G_E_SHAPE
    assert L.b2g_last_error().decode() == "null witness 0"
    assert L.b2g_prove(ctx._h, ph, mhc, rr.ctypes.data, rr.ctypes.data, w.ctypes.data, out.ctypes.data) == N.B2G_E_SHAPE
    assert L.b2g_last_error().decode() == "proving key and matrices disagree on n_vars"
    # a sharded context refuses the whole-proof entry point, a whole context refuses foreign shards' keys
    from circom_compat_b200 import Context
    cx = Context(0, 0, 2)
    with pytest.raises(B2gError) as e:
        Groth16.create_proof_with_reduction_and_matrices(pk, 1, 1, cm, cm.num_instance_variables, cm.num_constraints, w, cx)
    assert e.value.code == N.B2G_E_SHAPE
    assert e.value.msg == "a whole proof (b2g_prove, b2g_prove_many) needs an unsharded context; use b2g_prove_partial/finish"
    cx.close()
    # domain limit: next_pow2(num_constraints + num_inputs) must leave room for the doubled domain (qap.rs:31,63-66)
    from circom_compat_b200 import PolynomialDegreeTooLarge, ConstraintMatrices
    import numpy as _np
    huge = ConstraintMatrices(2, 2, (1 << 27) + 1, 0, 0, 0, (_np.zeros((1 << 27) + 2, dtype=_np.uint32), _np.zeros(0, dtype=_np.uint32), _np.zeros((0, 4), dtype=_np.uint64)),
                              (_np.zeros((1 << 27) + 2, dtype=_np.uint32), _np.zeros(0, dtype=_np.uint32), _np.zeros((0, 4), dtype=_np.uint64)))
    with pytest.raises(PolynomialDegreeTooLarge):
        ctx.mat_handle(huge, 4)


def test_cpp_host_mirror_proves_golden(golden, tmp_path):
    """C++ host layer (read_zkey -> Groth16::create_proof_with_reduction_and_matrices, the shape of benches/groth16.rs)
    reproduces the golden proof bytes; .wtns input and the host-computed chain witness."""
    import struct, subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, 'circom_compat_b200', 'host', 'groth16_bench')
    g = golden['complex_zkey']
    out = subprocess.check_output([exe, os.path.join(root, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'), 'chain:%d' % g['a'], '2',
                                   '%x' % int(g['r']), '%x' % int(g['s'])], text=True, env=dict(os.environ, B2G_INFLIGHT='3'))
    assert 'proof=' + g['proof_hex'] in out and 'verified=1' in out      # C++ process_vk + verify_with_processed_vk
    assert 'pipelined (3 in flight' in out and 'identical=1' in out      # Groth16::prove_batch: submit / wait on three contexts
    gt = golden['test_zkey']
    w = [int(x) for x in gt['witness']]
    wt = tmp_path / 'w.wtns'
    sec1 = struct.pack('<I', 32) + o.R_MOD.to_bytes(32, 'little') + struct.pack('<I', len(w))
    sec2 = b''.join(x.to_bytes(32, 'little') for x in w)
    wt.write_bytes(b'wtns' + struct.pack('<II', 2, 2) + struct.pack('<IQ', 1, len(sec1)) + sec1 + struct.pack('<IQ', 2, len(sec2)) + sec2)
    case = gt['proofs'][0]
    out = subprocess.check_output([exe, os.path.join(root, 'tests', 'golden', 'test.zkey'), str(wt), '1', '%x' % int(case['r']), '%x' % int(case['s'])], text=True)
    assert 'proof=' + case['proof_hex'] in out


# ------------------------------------------------------------------------------------------------ BASELINE.json sizes
def _dot_mod_r(a, b):
    return sum(x * y for x, y in zip(a, b)) % o.R_MOD


def test_msm_g1_2p20_closed_form(ctx):
    # config 3 size: 2^20 G1 bases [k_i]G against uniform and circom-like scalars; expected = [sum s_i k_i]G
    n = 1 << 20
    rng = random.Random(0xB200)
    ks = [rng.randrange(1, o.R_MOD) for _ in range(n)]
    bases = ctx.fixed_base_g1(c.ints_to_limbs(ks))
    for dist in ('uniform', 'circomlike'):
        _, sc = _msm_case(rng, n, dist)
        got = ctx.msm_g1(bases, c.ints_to_limbs(sc))
        exp = ctx.fixed_base_g1(c.ints_to_limbs([_dot_mod_r(ks, sc)]))[0]
        assert np.array_equal(got, exp), dist
        assert np.array_equal(got, c.fixed_base_g1(c.ints_to_limbs([_dot_mod_r(ks, sc)]))[0])


def test_msm_g2_2p20_stress(ctx):
    # config 5: G2 stress, 2^20 G2 bases (the B2-query shape), uniform (seed 0x62) and circom-like scalars
    n = 1 << 20
    rng = random.Random(0x62)
    ks = [rng.randrange(1, o.R_MOD) for _ in range(n)]
    bases = ctx.fixed_base_g2(c.ints_to_limbs(ks))
    for dist in ('uniform', 'circomlike'):
        _, sc = _msm_case(rng, n, dist)
        got = ctx.msm_g2(bases, c.ints_to_limbs(sc))
        assert np.array_equal(got, c.fixed_base_g2(c.ints_to_limbs([_dot_mod_r(ks, sc)]))[0]), dist


def test_headline_2p20_proof_closed_form(ctx):
    # config 3: the headline workload itself (chain, domain 2^20): proof == trapdoor closed form (O(n) big-int + 3 oracle muls)
    from circom_compat_b200 import Groth16, CircomReduction, fr_to_mont, fr_from_mont, synth, release
    circ = synth.chain_circuit(1 << 20); w = synth.chain_witness(1 << 20)
    pk, td = synth.setup(ctx, circ)
    cm = circ.matrices()
    wm = fr_to_mont(w)
    r, s = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
    h = CircomReduction.witness_map_from_matrices(cm, circ.num_inputs, circ.num_constraints, wm, ctx)
    p = Groth16.create_proof_with_reduction_and_matrices(pk, r, s, cm, circ.num_inputs, circ.num_constraints, wm, ctx)
    # (1) the witness map against the CPU oracle, bit for bit, at the headline size
    assert np.array_equal(h, c.witness_map(cm.num_constraints, circ.num_inputs, circ.n_vars, cm.a, cm.b, wm))
    # (2) the proof against the trapdoor closed form that uses NO h (H term = (a(tau) b(tau) - c(tau)) / delta): a wrong h
    #     cannot move this expectation.  (3) the h-based form must agree with it (checks h . h_t == the same quantity).
    da, db, dc = synth.expected_proof_dlogs_independent(td, circ, w, r, s)
    assert synth.expected_proof_dlogs(td, w, fr_from_mont(h), r, s, circ.num_inputs) == (da, db, dc)
    _assert_proof_is(p, da, db, dc)
    release(pk); release(cm)


def _assert_proof_is(p, da, db, dc):
    ea = c.limbs_to_ints(c.fq_from_mont(c.fixed_base_g1(c.ints_to_limbs([da, dc]))))
    eb = c.limbs_to_ints(c.fq_from_mont(c.fixed_base_g2(c.ints_to_limbs([db]))))
    assert p.a == (ea[0], ea[1]) and p.c == (ea[2], ea[3]) and p.b == ((eb[0], eb[1]), (eb[2], eb[3]))


@pytest.fixture(scope='module')
def chain22():
    from circom_compat_b200 import fr_to_mont, synth
    circ = synth.chain_circuit(1 << 22); w = synth.chain_witness(1 << 22)
    return circ, w, circ.matrices(), fr_to_mont(w)


def test_witness_map_2p22_vs_oracle(ctx, chain22):
    # BASELINE.json config 4's domain: qap.rs:23-88 on 2^22 rows (the three-pass NTT schedule), bit-exact vs oracle/cref.c
    from circom_compat_b200 import CircomReduction, release
    circ, w, cm, wm = chain22
    h = CircomReduction.witness_map_from_matrices(cm, circ.num_inputs, circ.num_constraints, wm, ctx)
    assert np.array_equal(h, c.witness_map(cm.num_constraints, circ.num_inputs, circ.n_vars, cm.a, cm.b, wm))
    release(cm)


def test_config4_2p22_base_sharded_proof_closed_form(chain22):
    # BASELINE.json config 4: 2^22-constraint chain, MSM bases sharded by range over every visible GPU (at least two
    # shard contexts; both on GPU 0 when the box has one), 768-byte partials folded in rank order.  Expected proof =
    # trapdoor closed form that does not use h (benches/groth16.rs:69-84 shape, qap.rs:30-32 domain rule).
    import torch
    from circom_compat_b200 import Groth16, Context, synth, release_all
    circ, w, cm, wm = chain22
    ngpu = max(1, torch.cuda.device_count())
    shards = max(2, ngpu)
    setup_ctx = Context(0)
    pk, td = synth.setup(setup_ctx, circ)
    setup_ctx.close()
    r, s = 0x1234567890abcdef1234567890abcdef, 0xfedcba0987654321fedcba0987654321
    parts, ctxs = [], []
    for rank in range(shards):
        cx = Context(rank % ngpu, rank, shards); ctxs.append(cx)
        parts.append(Groth16.prove_partial(pk, cm, wm, cx, r, s))
    p = Groth16.prove_finish(pk, np.stack(parts), r, s, ctxs[0])
    assert Groth16.prove_finish(pk, np.stack(parts), r, s, ctxs[-1]).data == p.data      # every rank obtains the same bytes
    _assert_proof_is(p, *synth.expected_proof_dlogs_independent(td, circ, w, r, s))
    release_all()
    for cx in ctxs:
        cx.close()


def test_gpu_setup_prove_verify_flow(ctx):
    """tests/groth16.rs:11-41 flow on the GPU: generate_random_parameters_with_reduction -> prove -> verify (oracle pairing),
    and the wrong-public-input negative of tests/groth16.rs:42-74."""
    from circom_compat_b200 import Groth16, fr_to_mont, synth, release
    circ, w = synth.circomlike_circuit(8)
    rng = random.Random(1234)
    pk = Groth16.generate_random_parameters_with_reduction(circ, rng, ctx)
    cm = circ.matrices()
    p = Groth16.prove(pk, cm, fr_to_mont(w), rng, ctx)
    vk = _vk_from_pk(pk)
    assert vk.gamma_g2 != o.G2_GEN                                   # gamma is random here, not 1
    # tests/groth16.rs:33-37: Groth16::verify(&vk, &inputs, &proof) on the product's verifier; oracle pairing as cross-check
    assert Groth16.verify(pk, w[1:circ.num_inputs], p)
    assert not Groth16.verify(pk, [(w[1] + 1) % o.R_MOD], p)
    assert o.verify(vk, w[1:circ.num_inputs], (p.a, p.b, p.c))
    release(pk); release(cm)


# ------------------------------------------------------------------------------------------------ LibsnarkReduction + R1CS route
def _vk_from_pk(pk):
    vk = o.ZKey()
    def g1(a): return o._g1_from(np.ascontiguousarray(a).tobytes())
    def g2(a): return o._g2_from(np.ascontiguousarray(a).tobytes())
    vk.alpha_g1, vk.beta_g2, vk.gamma_g2, vk.delta_g2 = g1(pk.alpha_g1), g2(pk.beta_g2), g2(pk.gamma_g2), g2(pk.delta_g2)
    vk.ic = [g1(x) for x in pk.gamma_abc_g1]
    return vk


@pytest.mark.parametrize('log_n', [3, 9, 11, 14])
def test_libsnark_witness_map_vs_oracle(ctx, log_n):
    from circom_compat_b200 import LibsnarkReduction, fr_to_mont, synth, release
    circ, w = synth.circomlike_circuit(log_n)
    cm = circ.matrices(with_c=True)
    wm = fr_to_mont(w)
    h = LibsnarkReduction.witness_map_from_matrices(cm, circ.num_inputs, circ.num_constraints, wm, ctx)
    ref = c.witness_map_libsnark(cm.num_constraints, cm.num_instance_variables, cm.a, cm.b, cm.c, wm)
    assert np.array_equal(h, ref)
    assert not h[-1].any()                                     # deg h <= n - 2
    release(cm)


def test_r1cs_route_setup_prove_verify(ctx):
    """/root/reference/tests/groth16.rs:11-41 (mycircuit) and :75-105 (circuit2) with their real circom fixtures:
    R1CS file -> matrices, snarkjs witness, Groth16<Bn254> = LibsnarkReduction setup -> prove -> verify; :42-74 negative."""
    from circom_compat_b200 import R1CSFile, R1CS, read_wtns, Groth16, LibsnarkReduction, fr_to_mont, fr_from_mont, release
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    rng = random.Random(99)
    for r1cs_name, witness in (('mycircuit.r1cs', [1, 33, 3, 11]), ('circuit2.r1cs', None)):
        r = R1CS.from_file(R1CSFile.new(open(os.path.join(root, 'tests', 'golden', r1cs_name), 'rb').read()))
        w = witness or read_wtns(open(os.path.join(root, 'tests', 'golden', 'circuit2_witness.wtns'), 'rb').read())
        circ = r.to_circuit()
        cm = circ.matrices(with_c=True)
        pk = Groth16.generate_random_parameters_with_reduction(circ, rng, ctx, LibsnarkReduction)
        assert len(pk.h_query) == circ.domain_size - 1
        wm = fr_to_mont(w)
        p = Groth16.prove(pk, cm, wm, rng, ctx, LibsnarkReduction)
        pvk = Groth16.process_vk(pk)
        assert Groth16.verify_with_processed_vk(pvk, w[1:r.num_inputs], p), r1cs_name
        assert not Groth16.verify_with_processed_vk(pvk, [(w[1] + 1) % o.R_MOD] + w[2:r.num_inputs], p)
        assert o.verify(_vk_from_pk(pk), w[1:r.num_inputs], (p.a, p.b, p.c)), r1cs_name
        # the witness map behind it is the oracle's
        h = LibsnarkReduction.witness_map_from_matrices(cm, r.num_inputs, len(r.constraints), wm, ctx)
        ni, nw, cons = r.num_inputs, r.num_variables, [tuple([(v, i) for i, v in lc] for lc in con) for con in r.constraints]
        href = o.libsnark_witness_map_from_matrices([c_[0] for c_ in cons], [c_[1] for c_ in cons], [c_[2] for c_ in cons], ni, len(cons), w)
        assert fr_from_mont(h) == href
        release(pk); release(cm)


def test_libsnark_proof_matches_cpu_oracle_bytes(ctx):
    # same key, witness, r, s: GPU proof bytes == CPU oracle (libsnark h fed to the shared proof assembly)
    from circom_compat_b200 import Groth16, LibsnarkReduction, fr_to_mont, synth, release
    circ, w = synth.circomlike_circuit(12)
    pk, td = synth.setup(ctx, circ, flavour='libsnark')
    cm = circ.matrices(with_c=True)
    wm = fr_to_mont(w)
    r, s = 0x1234567, 0x7654321
    p = Groth16.create_proof_with_reduction_and_matrices(pk, r, s, cm, circ.num_inputs, circ.num_constraints, wm, ctx, LibsnarkReduction)
    href = c.fr_from_mont(c.witness_map_libsnark(cm.num_constraints, cm.num_instance_variables, cm.a, cm.b, cm.c, wm))
    hi = c.limbs_to_ints(href)
    da, db, dc = synth.expected_proof_dlogs(td, w, hi[:len(td.h_t)], r, s, circ.num_inputs)
    assert o.G1.mul(o.G1_GEN, da) == p.a and o.G2.mul(o.G2_GEN, db) == p.b and o.G1.mul(o.G1_GEN, dc) == p.c
    release(pk); release(cm)


def _p2p_worker(rank, world, port, q):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    os.environ['MASTER_ADDR'] = '127.0.0.1'; os.environ['MASTER_PORT'] = str(port)
    os.environ['B2G_P2P_TIMEOUT_MS'] = '15000'                   # a broken exchange fails instead of spinning
    import json
    import torch
    import torch.distributed as dist
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from circom_compat_b200 import read_zkey, Groth16, fr_to_mont, Context, sharding
        from oracle import pyref
        g = json.load(open(os.path.join(root, 'tests', 'golden', 'golden_vectors.json')))['complex_zkey']
        pk, cm = read_zkey(os.path.join(root, 'tests', 'golden', 'complex-circuit-10000-10000.zkey'))
        wm = fr_to_mont(pyref.chain_witness(pk.n_vars, g['a']))
        dev = rank % torch.cuda.device_count()
        ctx = Context(dev, rank, world)
        ctx.prepare(pk, cm)                                      # before the wiring: the exchange arena is sized for this domain
        sharding.connect_p2p(ctx, dist)                          # CUDA-IPC handles over gloo
        dist.barrier()
        ok = True
        for _ in range(3):                                       # several epochs: both exchange slots are reused
            p = Groth16.prove_sharded_p2p(pk, cm, int(g['r']), int(g['s']), wm, ctx)
            ok = ok and p.data.hex() == g['proof_hex']
        q.put((rank, ok))
        dist.barrier()
        ctx.close()
    except Exception as e:                                       # noqa: BLE001
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('world', [2, 4])
def test_sharded_proof_fused_peer_memory_exchange(world):
    """b2g_prove_sharded_p2p, one process per shard (one GPU each if the box has them, else all on GPU 0): each rank publishes
    its partial MSM results with a system-scope release and folds its peers' partials straight out of their HBM (CUDA IPC
    mapping) inside the captured proof graph; every rank must produce the golden proof.  world = 4 also runs the SPLIT
    witness map: a, b, c transformed on ranks 0, 1, 2, every rank forming its slice of h = a*b - c from peer memory."""
    import torch.multiprocessing as mp
    mpc = mp.get_context('spawn')
    q = mpc.Queue()
    port = 29600 + (os.getpid() % 300) + world
    procs = [mpc.Process(target=_p2p_worker, args=(r, world, port, q)) for r in range(world)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=240) for _ in range(world))
    [p.join(timeout=30) for p in procs]
    assert res == [(r, True) for r in range(world)], res


def test_off_curve_key_point_is_rejected(ctx, test_zkey_bytes):
    # the reference panics in G1Affine::new on an off-curve zkey point (src/zkey.rs:347); the ABI returns B2G_E_INPUT
    from circom_compat_b200 import read_zkey, Groth16, fr_to_mont, B2gError, release
    pk, cm = read_zkey(test_zkey_bytes)
    pk.a_query = pk.a_query.copy(); pk.a_query[2, 0] ^= 1          # flip one bit of a coordinate
    with pytest.raises(B2gError) as e:
        Groth16.create_proof_with_reduction_and_matrices(pk, 1, 1, cm, cm.num_instance_variables, cm.num_constraints, fr_to_mont([1, 33, 3, 11]), ctx)
    assert e.value.code == -4 and 'not on the curve' in str(e.value)
    pk2, _ = read_zkey(test_zkey_bytes)
    pk2.b_g2_query = pk2.b_g2_query.copy(); pk2.b_g2_query[3, 5] ^= 4
    with pytest.raises(B2gError) as e:
        ctx.pk_handle(pk2)
    assert e.value.code == -4
    release(cm)


def test_load_time_validation(ctx, test_zkey_bytes, monkeypatch):
    """What b2g_pk_load / b2g_matrices_load refuse: off-curve alpha / delta / query[0] (the reference's G1Affine::new and
    G2Affine::new validate every point, src/zkey.rs:340-360), malformed CSR row pointers
    and an out-of-range window override."""
    from circom_compat_b200 import read_zkey, B2gError, ConstraintMatrices
    for field, idx in (('alpha_g1', (0, 1)), ('delta_g1', (0, 0)), ('delta_g2', (0, 3)), ('a_query', (0, 2)), ('b_g2_query', (0, 9)), ('beta_g2', (0, 0))):
        pk, _ = read_zkey(test_zkey_bytes)
        arr = getattr(pk, field).copy(); arr[idx] ^= 2; setattr(pk, field, arr)
        if field in ('a_query', 'b_g2_query') and not arr[0].any():
            continue                                              # query[0] at infinity in this key: nothing to corrupt
        with pytest.raises(B2gError) as e:
            ctx.pk_handle(pk)
        assert e.value.code == -4 and 'not on the curve' in str(e.value), field
    from circom_compat_b200 import synth
    cm = synth.chain_circuit(8).matrices()                        # 6 rows, one entry each: rowptr = 0..6
    for rowptr in ([1, 1, 2, 3, 4, 5, 6], [0, 2, 1, 3, 4, 5, 6]):
        bad = ConstraintMatrices(cm.num_instance_variables, cm.num_witness_variables, cm.num_constraints, cm.a_num_non_zero, cm.b_num_non_zero, 0,
                                 (np.array(rowptr, dtype=np.uint32), cm.a[1], cm.a[2]), cm.b)
        with pytest.raises(B2gError) as e:
            ctx.mat_handle(bad, 8)
        assert e.value.code == -2 and 'row' in str(e.value), rowptr
    monkeypatch.setenv('B2G_MSM_C', '5')
    with pytest.raises(B2gError) as e:
        ctx.msm_g1(c.fixed_base_g1(c.ints_to_limbs([1, 2, 3])), c.ints_to_limbs([1, 2, 3]))
    assert e.value.code == -2 and 'B2G_MSM_C' in str(e.value)


# ------------------------------------------------------------------------------------------------ edge cases
def _prove_both(ctx, circ, w, r, s, td_seed=7):
    """GPU proof and CPU-oracle proof on a fresh synthetic key; returns (gpu bytes, oracle bytes, pk, td)"""
    from circom_compat_b200 import Groth16, fr_to_mont, synth, release
    pk, td = synth.setup(ctx, circ, seed=td_seed)
    cm = circ.matrices()
    wm = fr_to_mont(w)
    p = Groth16.create_proof_with_reduction_and_matrices(pk, r, s, cm, circ.num_inputs, circ.num_constraints, wm, ctx)
    ref = c.prove(_oracle_key(pk, cm), r, s, wm)
    release(pk); release(cm)
    return p, ref


def test_edge_zero_witness_and_zero_blinding(ctx):
    # squaring chain with a = 0: every wire except the constant is 0 -> all MSM scalars but one vanish (empty buckets,
    # infinity partial results); r = s = 0 removes every delta term and skips B1 (prover.rs: r == 0)
    from circom_compat_b200 import synth, Groth16, Context, fr_to_mont, release
    circ = synth.chain_circuit(1 << 10)
    w = synth.chain_witness(1 << 10, 0)
    assert w[0] == 1 and not any(w[1:])
    cases = ((0, 0), (0, 5), (7, 0), (o.R_MOD - 1, o.R_MOD - 1))
    for r, s in cases:
        p, ref = _prove_both(ctx, circ, w, r, s)
        assert p.data == ref, (r, s)
    # the same scalars through the host-exchange sharded route: three shard contexts, prove_finish scales every rank's
    # A / B1 partial itself; with (r, s) given to prove_partial, prove_finish reuses the precomputation started there
    pk, td = synth.setup(ctx, circ)
    cm = circ.matrices()
    wm = fr_to_mont(w)
    shards = [Context(0, rank, 3) for rank in range(3)]
    for r, s in cases:
        ref = c.prove(_oracle_key(pk, cm), r, s, wm)
        for early in ((None, None), (r, s)):
            parts = np.stack([Groth16.prove_partial(pk, cm, wm, cx, *early) for cx in shards])
            assert Groth16.prove_finish(pk, parts, r, s, shards[0]).data == ref, (r, s, early)
    release(pk); release(cm)
    for cx in shards:
        cx.close()


def test_edge_no_witness_variables_and_tiny_domains(ctx):
    # n_vars == num_inputs: the L query is empty (msm over zero terms = infinity); domains of size 2 and 4
    from circom_compat_b200 import synth
    one = [1]
    circ = synth.Circuit(2, 2, 1, (np.array([0]), np.array([1]), one), (np.array([0]), np.array([0]), one), (np.array([0]), np.array([1]), one))   # w1 * 1 = w1
    w = [1, 5]
    assert circ.domain_size == 4
    p, ref = _prove_both(ctx, circ, w, 3, 4)
    assert p.data == ref
    circ1 = synth.Circuit(1, 1, 1, (np.array([0]), np.array([0]), one), (np.array([0]), np.array([0]), one), (np.array([0]), np.array([0]), one))  # 1 * 1 = 1
    assert circ1.domain_size == 2
    p, ref = _prove_both(ctx, circ1, [1], 9, 11)
    assert p.data == ref


@pytest.mark.parametrize('m', [1022, 1023, 1024])
def test_edge_domain_boundaries(ctx, m):
    # domain = next_pow2(num_constraints + num_inputs) (qap.rs:30-31): 1022 + 2 = 1024 exactly, 1023 + 2 and 1024 + 2 -> 2048
    from circom_compat_b200 import synth
    circ = synth.chain_circuit(m + 2)
    assert circ.num_constraints == m and circ.domain_size == (1024 if m == 1022 else 2048)
    p, ref = _prove_both(ctx, circ, synth.chain_witness(m + 2, 3), 0xabcdef, 0x123456)
    assert p.data == ref


def test_edge_ragged_rows_and_repeated_columns(ctx):
    # rows with 0, 1 and many terms, repeated wire indices and explicit zero coefficients in A / B (evaluate_constraint just sums)
    from circom_compat_b200 import synth, CircomReduction, fr_to_mont, release
    rng = random.Random(31)
    n_vars, li, m = 40, 3, 29
    w = [1] + [rng.randrange(o.R_MOD) for _ in range(n_vars - 1)]
    rows_a, cols_a, vals_a, rows_b, cols_b, vals_b = [], [], [], [], [], []
    for i in range(m):
        for (rows, cols, vals, k) in ((rows_a, cols_a, vals_a, i % 7), (rows_b, cols_b, vals_b, (i * 3) % 5)):
            for _ in range(k):                                   # k = 0 -> empty row
                rows.append(i); cols.append(rng.randrange(n_vars)); vals.append(rng.choice([0, 1, o.R_MOD - 1, rng.randrange(o.R_MOD)]))
    circ = synth.Circuit(n_vars, li, m, (np.array(rows_a), np.array(cols_a), vals_a), (np.array(rows_b), np.array(cols_b), vals_b),
                         (np.array([], dtype=np.int64), np.array([], dtype=np.int64), []))
    cm = circ.matrices()
    wm = fr_to_mont(w)
    h = CircomReduction.witness_map_from_matrices(cm, li, m, wm, ctx)
    href = c.witness_map(m, li, n_vars, cm.a, cm.b, wm)
    assert np.array_equal(h, href)
    A = [[] for _ in range(m)]; B = [[] for _ in range(m)]
    for r_, c_, v in zip(rows_a, cols_a, vals_a): A[r_].append((v, c_))
    for r_, c_, v in zip(rows_b, cols_b, vals_b): B[r_].append((v, c_))
    assert c.limbs_to_ints(c.fr_from_mont(h)) == o.witness_map_from_matrices(A, B, li, m, w)
    release(cm)


def test_proofs_of_the_reference_witness_kats(ctx, golden, test_zkey_bytes):
    """The witnesses the reference's witness-calculator tests pin for mycircuit (src/witness/witness_calculator.rs:260-298:
    multiplier_1/2/3; 2 and 3 carry scalars a few units below r) proved with the reference's test.zkey: proof bytes equal the
    big-int oracle's and verify against the public input circuit.rs:18-26 derives from the witness."""
    from circom_compat_b200 import read_zkey, Groth16, fr_to_mont
    pk, cm = read_zkey(test_zkey_bytes)
    z = o.read_zkey(test_zkey_bytes)
    r, s = int(golden['r']), int(golden['s'])
    pvk = Groth16.process_vk(pk)
    for wit in golden['witness_kats']['multiplier']:
        w = [int(x) for x in wit]
        p = Groth16.create_proof_with_reduction_and_matrices(pk, r, s, cm, cm.num_instance_variables, cm.num_constraints, fr_to_mont(w), ctx)
        A, B, C = o.prove(z, r, s, w)
        assert p.data == o.proof_to_bytes(A, B, C)
        assert Groth16.verify_with_processed_vk(pvk, w[1:cm.num_instance_variables], p)
        assert not Groth16.verify_with_processed_vk(pvk, [(w[1] + 1) % o.R_MOD], p)
