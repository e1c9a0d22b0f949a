"""The big-int model of b2g_verify_batch (tests/batch_model.py), checked on the CPU: the G2 membership test the device runs
against the order test, and the random-linear-combination batch equation against valid, tampered and cancelling proofs."""
import random

from batch_model import g2_in_subgroup, outside_b_proof, twist_point_outside_g2, verify_batch_rlc
from circom_compat_b200 import verifier as V
from oracle import pyref as o

P, R = V.P, o.R_MOD


# ---------------------------------------------------------------------------------------------- helpers
def _g1(k):
    return o.G1.mul(o.G1_GEN, k)


def _g2(k):
    return o.G2.mul(o.G2_GEN, k)


def _synthetic(n_public, seed, count):
    """a key with known discrete logs and `count` valid proofs as (A, B, C) tuples"""
    rng = random.Random(seed)
    al, be, ga, de = (rng.randrange(1, R) for _ in range(4))
    ic = [rng.randrange(1, R) for _ in range(n_public + 1)]
    vk = V.VerifyingKey(_g1(al), _g2(be), _g2(ga), _g2(de), [_g1(k) for k in ic])
    inputs, proofs = [], []
    for _ in range(count):
        xs = [rng.randrange(R) for _ in range(n_public)]
        a, b = rng.randrange(1, R), rng.randrange(1, R)
        prep = (ic[0] + sum(x * k for x, k in zip(xs, ic[1:]))) % R
        c = (a * b - al * be - prep * ga) * pow(de, -1, R) % R
        inputs.append(xs)
        proofs.append((_g1(a), _g2(b), _g1(c)))
    return V.prepare_verifying_key(vk), inputs, proofs


# ---------------------------------------------------------------------------------------------- tests
def test_g2_membership_agrees_with_the_order_check():
    rng = random.Random(43)
    inside = [_g2(rng.randrange(1, R)) for _ in range(4)] + [o.G2_GEN]
    outside = [twist_point_outside_g2(rng) for _ in range(5)]
    for q in inside + outside:
        assert V.g2_on_curve(q)
        assert g2_in_subgroup(q) == (o.G2.mul(q, R - 1) == o.G2.neg(q))
    assert all(g2_in_subgroup(q) for q in inside) and not any(g2_in_subgroup(q) for q in outside)
    assert g2_in_subgroup(None)


def test_batch_model_accepts_valid_and_refuses_a_tampered_proof():
    rng = random.Random(44)
    for n_public in (0, 2):
        pvk, inputs, proofs = _synthetic(n_public, 50 + n_public, 3)
        assert all(V.verify_with_processed_vk(pvk, xs, p) for xs, p in zip(inputs, proofs))
        weights = [rng.getrandbits(128) | 1 for _ in proofs]
        assert verify_batch_rlc(pvk, inputs, proofs, weights)
        a, b, c = proofs[1]
        bad = proofs[:1] + [(a, b, o.G1.add(c, o.G1_GEN))] + proofs[2:]
        assert not verify_batch_rlc(pvk, inputs, bad, weights)
        if n_public:
            assert not verify_batch_rlc(pvk, [inputs[0], [(inputs[1][0] + 1) % R, inputs[1][1]], inputs[2]], proofs, weights)


def test_batch_model_refuses_b_outside_g2_and_coordinates_above_p():
    pvk, inputs, proofs = _synthetic(1, 60, 2)
    a, b, c = proofs[0]
    outside = twist_point_outside_g2(random.Random(60))
    assert not verify_batch_rlc(pvk, inputs, [(a, outside, c), proofs[1]], [1, 1])
    assert not verify_batch_rlc(pvk, inputs, [((a[0] + P, a[1]), b, c), proofs[1]], [1, 1])


def test_cancelling_pair_needs_random_weights():
    """C_1 + D and C_2 - D: each proof is invalid, the sum of the C is unchanged"""
    pvk, inputs, proofs = _synthetic(1, 70, 3)
    d = _g1(12345)
    (a1, b1, c1), (a2, b2, c2) = proofs[0], proofs[1]
    bad = [(a1, b1, o.G1.add(c1, d)), (a2, b2, o.G1.add(c2, o.G1.neg(d))), proofs[2]]
    assert not V.verify_with_processed_vk(pvk, inputs[0], bad[0]) and not V.verify_with_processed_vk(pvk, inputs[1], bad[1])
    assert verify_batch_rlc(pvk, inputs, bad, [1, 1, 1])
    rng = random.Random(71)
    assert not verify_batch_rlc(pvk, inputs, bad, [rng.getrandbits(128) | 1 for _ in bad])


def test_b_outside_g2_fails_the_batch_where_the_pairing_holds():
    """A at infinity removes e(A, B); C is solved so that the rest equals e(alpha, beta).  The host verifier accepts the proof,
    and only the G2 membership test makes the model refuse it: with a B in G2 instead, the same proof passes"""
    vk, xs, proof = outside_b_proof(80)
    pvk = V.prepare_verifying_key(vk)
    assert V.verify_with_processed_vk(pvk, xs, proof) and not g2_in_subgroup(proof[1])
    assert not verify_batch_rlc(pvk, [xs], [proof], [3])
    a, b, c = proof
    b_in = o.G2.mul(o.G2_GEN, 5)
    assert V.verify_with_processed_vk(pvk, xs, (a, b_in, c)) and verify_batch_rlc(pvk, [xs], [(a, b_in, c)], [3])
