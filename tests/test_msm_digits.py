"""Signed-digit windows of the MSM (msm.cu msm_window_bits / msm_digit_at) at every window size B2G_MSM_C accepts.

The CPU test checks the restated shortcut against the full carry chain (oracle/msm_digits.py); the GPU test runs G1 and G2
MSMs at each window size on scalars whose windows sit on the values where the shortcut's walk decides a carry."""
import functools
import random

import numpy as np
import pytest

from oracle import cref as c
from oracle import msm_digits as md
from oracle import pyref as o

WINDOWS = list(range(8, 23))


def _uniform(rng, n):
    return [rng.randrange(o.R_MOD) for _ in range(n)]


def _circomlike(rng, n):            # 60 % bits, 20 % small, 20 % wide
    return [rng.randrange(2) if (u := rng.random()) < 0.6 else (rng.randrange(1 << 32) if u < 0.8 else rng.randrange(o.R_MOD))
            for _ in range(n)]


@pytest.mark.parametrize('cw', WINDOWS)
def test_digit_shortcut_matches_carry_chain(cw):
    rng = random.Random(cw)
    h = 1 << (cw - 1)
    nw = md.nwin(cw)
    # no carry out of the top window for ANY k < r: its raw bits are at most (r-1) >> (c (nwin-1)), plus a carry of one
    assert ((o.R_MOD - 1) >> (cw * (nw - 1))) + 1 < h
    assert nw * cw >= 255 and md.nwin(cw) == len(md.make_digits(0, cw))
    edge = md.digit_edge_scalars(cw, rng)
    # the generator reaches what it promises: runs of h-1 of every depth that end at the bottom of the scalar
    for depth in range(1, nw):
        assert any(all(md.window_bits(k, cw, w) == h - 1 for w in range(depth)) for k in edge), depth
    for k in edge + _uniform(rng, 300) + [0, 1, h - 1, h, (1 << cw) - 1]:
        d = md.device_digits(k, cw)
        assert d == md.make_digits(k, cw), hex(k)
        assert sum(x << (cw * w) for w, x in enumerate(d)) == k
        assert all(-h <= x < h for x in d)


def test_digit_walk_depth_is_observable():
    # a walk limited to two windows would mis-carry here: windows 0..2 = h-1, h-1, h (bottom up), so window 3 takes a carry
    # that only the third window down decides
    cw = 8
    h = 1 << (cw - 1)
    k = h | ((h - 1) << cw) | ((h - 1) << (2 * cw))
    assert md.digit_at(k, cw, 3) == 1 and md.make_digits(k, cw)[3] == 1


# ------------------------------------------------------------------------------------------------ the MSM at every window size
@functools.lru_cache(maxsize=None)
def _bases(g2, n):
    rng = random.Random(0xD161 + g2)
    ks = [rng.randrange(1, o.R_MOD) for _ in range(n)]
    return (c.fixed_base_g2 if g2 else c.fixed_base_g1)(c.ints_to_limbs(ks))


@pytest.mark.gpu
@pytest.mark.parametrize('cw', WINDOWS)
def test_msm_every_window_size(ctx, monkeypatch, cw):
    monkeypatch.setenv('B2G_MSM_C', str(cw))
    rng = random.Random(100 + cw)
    edge = md.digit_edge_scalars(cw, rng)
    n = 3000
    assert len(edge) < n
    sc = edge + _circomlike(rng, n - len(edge))
    bases = _bases(False, n)
    scl = c.ints_to_limbs(sc)
    exp = c.msm_g1(bases, scl)
    assert np.array_equal(ctx.msm_g1(bases, scl), exp)
    assert np.array_equal(ctx.msm_g1(bases, c.fr_to_mont(scl), scalars_mont=True), exp)
    if cw in (8, 12, 16, 17, 22):
        n2 = 800
        assert len(edge) < n2
        sc2 = edge + _circomlike(rng, n2 - len(edge))
        bases2 = _bases(True, n2)
        scl2 = c.ints_to_limbs(sc2)
        assert np.array_equal(ctx.msm_g2(bases2, scl2), c.msm_g2(bases2, scl2))
