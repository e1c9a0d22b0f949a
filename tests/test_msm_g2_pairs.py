"""G2 bucket accumulation runs one chain per lane pair (msm.cu msm_accumulate_g2_kernel).  Tiny runs make buckets straddle
many pairs, so the fragment records (each lane stores half of one) and the whole-CTA fold of buckets with many fragments
are exercised, against oracle/cref.c."""
import random

import numpy as np
import pytest

from oracle import cref as c
from oracle import pyref as o

pytestmark = pytest.mark.gpu


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
    scl = c.ints_to_limbs([7, 7])
    for pair in ((Q, Q), (Q, Qn), (Q, np.zeros_like(Q)), (np.zeros_like(Q), Q)):
        bases = np.stack(pair)
        assert np.array_equal(ctx.msm_g2(bases, scl), c.msm_g2(bases, scl))
