"""G2 bucket accumulation runs one chain per lane pair (msm.cu msm_accumulate_g2_kernel).  Tiny runs make buckets straddle
many pairs, so the fragment records (each lane stores half of one) and the whole-CTA fold of buckets with many fragments
are exercised, against oracle/cref.c.  Single lane-pair additions and runs (test ops 26 / 27) are checked as raw XYZZ
records in big-int arithmetic (oracle/xyzz.py)."""
import random

import numpy as np
import pytest

from circom_compat_b200.groth16 import TEST_PAIR_RUN
from oracle import cref as c
from oracle import msm_digits as md
from oracle import pyref as o
from oracle import xyzz as X

pytestmark = pytest.mark.gpu


def _entry(E, sign):
    """a signed entry (16 words of affine point, 4 words of sign) whose effective point is E: with the sign bit set it
    stores -E, which the lane pair negates back"""
    e = np.zeros(20, dtype=np.uint64)
    e[:16] = X.aff_row(o.G2.neg(E) if sign else E, True)
    e[16] = sign
    return e


def _g2_points(rng, n):
    return [X.aff(r, True) for r in c.fixed_base_g2(c.ints_to_limbs([rng.randrange(1, o.R_MOD) for _ in range(n)]))]


def test_g2_pair_madd_exceptional_cases(ctx):
    """G2Pair::madd onto projective, affine and empty accumulators: generic sum, acc == q (doubling), acc == -q (infinity),
    q at infinity, both at infinity; each with the entry's sign bit clear and set.  Adjacent rows (lane pairs of one warp)
    take different branches."""
    rng = random.Random(2026)
    pts = _g2_points(rng, 6)
    acc, ent, exp, labels = [], [], [], []
    for label, P, z, Q in X.addition_cases(rng, True, pts):
        for sign in (0, 1):
            acc.append(X.record(P, z, True)); ent.append(_entry(Q, sign))
            exp.append(o.G2.add(P, Q)); labels.append((label, sign))
    out = ctx.test_op(26, np.stack(acc), np.stack(ent))
    bad = [(i, labels[i], err) for i in range(len(exp)) if (err := X.check_record(out[i], exp[i], True, strict_inf=True))]
    assert not bad, (len(bad), bad[:6])


def test_g2_pair_runs(ctx):
    """One lane pair folds TEST_PAIR_RUN signed entries from empty, as one run of the accumulation kernel: doubling on a
    projective accumulator, infinity in mid-run and a restart, points at infinity, and random runs, interleaved so that the
    pairs of one warp diverge."""
    rng = random.Random(77)
    G = o.G2
    pool = _g2_points(rng, 12)
    P, Q, R, A, B, C = pool[:6]
    PQ, ABC = G.add(P, Q), G.sum([A, B, C])
    heads = [[P, Q, PQ], [P, Q, G.neg(PQ), R], [P, G.neg(P), P], [None, P, None], [P, P, P], [A, B, C, ABC],
             [A, B, C, G.neg(ABC), P], [None, None], [P, G.neg(P), G.neg(P), P], []]
    runs = []
    for _ in range(6):
        for head in heads:
            seq = list(head) + [rng.choice(pool + [None]) for _ in range(TEST_PAIR_RUN - len(head))]
            runs.append(seq)
    rows = np.stack([np.concatenate([_entry(E, rng.randrange(2)) for E in seq]) for seq in runs])
    out = ctx.test_op(27, rows)
    bad = [(i, err) for i, seq in enumerate(runs) if (err := X.check_record(out[i], G.sum(seq), True, strict_inf=True))]
    assert not bad, (len(bad), bad[:6])


def test_msm_g2_small_chunks_exercise_fragments(ctx, monkeypatch):
    rng = random.Random(91)
    n = 3000
    ks = [rng.randrange(1, o.R_MOD) for _ in range(n)]
    # circom-like: 60 % bits, 20 % small, 20 % wide
    sc = [rng.randrange(2) if (u := rng.random()) < 0.6 else (rng.randrange(1 << 32) if u < 0.8 else rng.randrange(o.R_MOD))
          for _ in range(n)]
    bases = c.fixed_base_g2(c.ints_to_limbs(ks))
    bases[5] = 0                                   # a table point at infinity
    bases[9] = bases[8]; sc[8] = 5; sc[9] = o.R_MOD - 5    # a base used twice: P and -P land in one bucket
    scl = c.ints_to_limbs(sc)
    exp = c.msm_g2(bases, scl)
    for chunk in ('1', '2', '3', '7'):
        monkeypatch.setenv('B2G_MSM_CHUNK_G2', chunk)
        assert np.array_equal(ctx.msm_g2(bases, scl), exp), chunk
    # two-entry buckets make the pair's exceptional cases deterministic: P + P (doubling), P + (-P), P + infinity
    monkeypatch.delenv('B2G_MSM_CHUNK_G2')
    k = rng.randrange(1, o.R_MOD)
    Q = c.fixed_base_g2(c.ints_to_limbs([k]))[0]
    Qn = c.fixed_base_g2(c.ints_to_limbs([o.R_MOD - k]))[0]
    s2 = c.ints_to_limbs([7, 7])
    for pair in ((Q, Q), (Q, Qn), (Q, np.zeros_like(Q)), (np.zeros_like(Q), Q)):
        b2 = np.stack(pair)
        assert np.array_equal(ctx.msm_g2(b2, s2), c.msm_g2(b2, s2))
    # four equal points in runs of two: each fragment is 2Q in projective form and the fold takes add's doubling branch
    monkeypatch.setenv('B2G_MSM_CHUNK_G2', '2')
    for v in (3, rng.randrange(o.R_MOD)):
        b4, s4 = np.stack([Q] * 4), c.ints_to_limbs([v] * 4)
        assert np.array_equal(ctx.msm_g2(b4, s4), c.msm_g2(b4, s4)), v
    # buckets spanning MSM_BIG_FRAGS and MSM_BIG_FRAGS + 1 runs, on and off a run boundary
    monkeypatch.setenv('B2G_MSM_C', '8')
    sc_f, ch = md.fold_boundary_scalars(rng)
    monkeypatch.setenv('B2G_MSM_CHUNK_G2', str(ch))
    b_f = c.fixed_base_g2(c.ints_to_limbs([rng.randrange(1, o.R_MOD) for _ in range(len(sc_f))]))
    s_f = c.ints_to_limbs(sc_f)
    assert np.array_equal(ctx.msm_g2(b_f, s_f), c.msm_g2(b_f, s_f))
    # run lengths from one entry to 193 on a prefix whose entry count is not a multiple of 4: at 64 and 192 the last run is
    # cut short
    monkeypatch.setenv('B2G_MSM_C', '11')
    m = md.partial_slab_prefix(sc, 11)
    exp_m = c.msm_g2(bases[:m], scl[:m])
    for chunk in ('1', '3', '64', '192', '193'):
        monkeypatch.setenv('B2G_MSM_CHUNK_G2', chunk)
        assert np.array_equal(ctx.msm_g2(bases[:m], scl[:m]), exp_m), chunk
    monkeypatch.delenv('B2G_MSM_CHUNK_G2')
    # the weighted bucket sum with one and with all buckets per thread
    for cw in ('8', '13'):
        monkeypatch.setenv('B2G_MSM_C', cw)
        for rchunk in ('1', '1000'):
            monkeypatch.setenv('B2G_MSM_REDUCE_CHUNK', rchunk)
            assert np.array_equal(ctx.msm_g2(bases, scl), exp), (cw, rchunk)
