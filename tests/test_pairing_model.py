"""The big-int model of the device pairing (oracle/pairing_model.py) against the host verifier, and the constants
csrc/pairing.cuh pins against the model.  CPU only."""
import os
import random
import re

from circom_compat_b200 import verifier as V
from oracle import pairing_model as M
from oracle import pyref as o

P, R = V.P, o.R_MOD
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rand_f12(rng):
    return tuple(tuple((rng.randrange(P), rng.randrange(P)) for _ in range(3)) for _ in range(2))


def _g1(k):
    return o.G1.mul(o.G1_GEN, k)


def _g2(k):
    return o.G2.mul(o.G2_GEN, k)


def test_hard_part_is_the_exact_exponent():
    phi = P ** 4 - P ** 2 + 1
    assert phi % R == 0
    assert M.hard_chain_exponent() % phi == phi // R          # not a multiple: results are bit-identical to the host's


def test_loop_digits_and_frobenius_constants():
    assert sum(d * 2 ** i for i, d in enumerate(reversed(M.ATE_NAF))) == 6 * M.X + 2 == V.ATE_LOOP_COUNT
    assert all(M.ATE_NAF[i] == 0 or M.ATE_NAF[i + 1] == 0 for i in range(len(M.ATE_NAF) - 1))
    assert len(M.prepare_g2(o.G2_GEN)) == len(M.ATE_NAF) - 1 + sum(1 for d in M.ATE_NAF[1:] if d) + 2
    rng = random.Random(1)
    f = _rand_f12(rng)
    for k in (1, 2, 3):
        assert M.frobenius(f, k) == V.f12_pow(f, P ** k)
    q = _g2(5)                                                  # the twist Frobenius constants are the tower's
    assert (M.TWIST_FROB_X, M.TWIST_FROB_Y, M.TWIST_FROB2_X, M.TWIST_FROB2_Y) == (M.FROB[1][2], M.FROB[1][3], M.FROB[2][2], M.FROB[2][3])
    assert V.g2_on_curve(M.twist_frobenius(q)) and V.g2_on_curve(M.twist_frobenius2_neg(q))


def test_tower_pieces():
    rng = random.Random(2)
    f = _rand_f12(rng)
    assert M.f12_sqr(f) == V.f12_mul(f, f)
    c0, c3, c4 = [(rng.randrange(P), rng.randrange(P)) for _ in range(3)]
    assert M.mul_by_034(f, c0, c3, c4) == V.f12_mul(f, ((c0, V.F2_ZERO, V.F2_ZERO), (c3, c4, V.F2_ZERO)))
    g = V.f12_mul(V.f12_conj(f), V.f12_inv(f))
    g = V.f12_mul(M.frobenius(g, 2), g)
    assert M.cyclotomic_sqr(g) == V.f12_mul(g, g)
    assert M.exp_by_x(g) == V.f12_pow(g, M.X)


def test_projective_lines_are_scaled_affine_lines():
    """the doubling / addition coefficients at P are the host's affine line times an Fq2 factor, and the points agree"""
    q, t = _g2(3), _g2(11)
    px, py = _g1(7)
    tp = (t[0], t[1], V.F2_ONE)
    t2, l = M.dbl_step(tp)
    (a0, a1, a3), t2a = V._line_and_step(t, t, px, py)
    k = V.f2_mul(V.f2_scale(l[0], py), V.f2_inv((a0, 0)))       # the factor, from the w^0 coefficient
    assert V.f2_mul(a1, k) == V.f2_scale(l[1], px) and V.f2_mul(a3, k) == l[2]
    zi = V.f2_inv(t2[2])
    assert (V.f2_mul(t2[0], zi), V.f2_mul(t2[1], zi)) == t2a
    t3, l = M.add_step(tp, q)
    (a0, a1, a3), t3a = V._line_and_step(t, q, px, py)
    k = V.f2_mul(V.f2_scale(l[0], py), V.f2_inv((a0, 0)))
    assert V.f2_mul(a1, k) == V.f2_scale(l[1], px) and V.f2_mul(a3, k) == l[2]
    zi = V.f2_inv(t3[2])
    assert (V.f2_mul(t3[0], zi), V.f2_mul(t3[1], zi)) == t3a


def test_final_exponentiation_matches_host():
    rng = random.Random(3)
    for f in [_rand_f12(rng), _rand_f12(rng), V.miller_loop([(_g1(5), _g2(9))]), M.miller_loop([(_g1(2), _g2(3))])]:
        assert M.final_exponentiation(f) == V.final_exponentiation(f)


def test_pairing_matches_host_and_is_bilinear():
    rng = random.Random(4)
    assert M.pairing(o.G1_GEN, o.G2_GEN) == V.pairing(o.G1_GEN, o.G2_GEN)
    a, b = rng.randrange(1, R), rng.randrange(1, R)
    pa, qb = _g1(a), _g2(b)
    e = M.pairing(pa, qb)
    assert e == V.pairing(pa, qb)
    assert e == V.f12_pow(M.pairing(o.G1_GEN, o.G2_GEN), a * b % R)
    assert M.pairing(None, qb) == V.F12_ONE == M.pairing(pa, None)


def test_batched_verdict_matches_host(golden, test_zkey_bytes):
    from circom_compat_b200 import Proof, read_zkey
    pk, _ = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    xs = [int(x) for x in g['witness'][1:pk.n_public + 1]]
    good = Proof(bytes.fromhex(g['proofs'][0]['proof_hex']))
    c = o.G1.add(good.c, o.G1_GEN)
    bad = Proof(good.data[:192] + c[0].to_bytes(32, 'little') + c[1].to_bytes(32, 'little'))
    big = Proof((good.a[0] + P).to_bytes(32, 'little') + good.data[32:])        # a coordinate >= p
    pvk = V.prepare_verifying_key(pk)
    want = [V.verify_with_processed_vk(pvk, xs, p) for p in (good, bad, big)]
    assert want == [True, False, True]                                          # the host reduces the coordinate
    assert M.verify_batch(pvk, [xs] * 3, [good, bad, big]) == [True, False, False]


def _header_words(name):
    src = open(os.path.join(ROOT, 'circom_compat_b200', 'csrc', 'pairing.cuh')).read()
    body = re.search(name + r'\[[^=]*=\s*\{(.*?)\};', src, re.S).group(1)
    return [int(t.rstrip('u'), 0) for t in re.findall(r'-?0x[0-9a-f]+u|-?\d+', body)]


def test_pinned_constants_match_the_model():
    frob = [w for k in (1, 2, 3) for e in range(1, 6) for c in M.FROB[k][e] for w in M.mont_limbs(c)]
    assert _header_words('PAIRING_FROB') == frob
    b3 = V.f2_scale(V.TWIST_B, 3)
    assert _header_words('PAIRING_TWIST_B3') == M.mont_limbs(b3[0]) + M.mont_limbs(b3[1])
    assert _header_words('PAIRING_INV2') == M.mont_limbs((P + 1) // 2)
    assert _header_words('PAIRING_ATE_NAF') == M.ATE_NAF[1:]
    src = open(os.path.join(ROOT, 'circom_compat_b200', 'csrc', 'pairing.cuh')).read()
    assert 'PAIRING_X = 0x%xull' % M.X in src
    assert 'ATE_LINES = %d + %d + 2' % (len(M.ATE_NAF) - 1, sum(1 for d in M.ATE_NAF[1:] if d)) in src
