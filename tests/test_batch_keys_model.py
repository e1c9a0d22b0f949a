"""The per-key model of b2g_verify_batch_keys (tests/batch_keys_model.py), checked on the CPU against the host verifier: valid
batches under several keys, the same key twice and an empty batch are True; a tampered proof or a B outside G2 makes its own
key's verdict False and no other."""
import random

from batch_keys_model import verify_batch_keys_rlc
from batch_model import outside_b_proof
from circom_compat_b200 import verifier as V
from oracle import pyref as o
from test_batch_model import _synthetic

R = o.R_MOD


def _host(batches):
    """the host verifier's verdict per batch: every proof passes verify_with_processed_vk"""
    return [all(V.verify_with_processed_vk(pvk, xs, p) for xs, p in zip(ins, prs)) for pvk, ins, prs in batches]


def test_keys_model_agrees_with_the_host_verifier():
    rng = random.Random(90)
    k0, k1, k2 = _synthetic(0, 90, 2), _synthetic(1, 91, 1), _synthetic(2, 92, 2)
    batches = [k0, k1, k2, (k2[0], k2[1][:1], k2[2][:1]), (k1[0], [], [])]     # k2's key twice; an empty batch
    weights = [[rng.getrandbits(128) | 1 for _ in prs] for _, _, prs in batches]
    assert verify_batch_keys_rlc(batches, weights) == _host(batches) == [True] * 5
    pvk, ins, prs = k2
    a, b, c = prs[1]
    bad = list(batches)
    bad[2] = (pvk, ins, [prs[0], (a, b, o.G1.add(c, o.G1_GEN))])
    assert verify_batch_keys_rlc(bad, weights) == _host(bad) == [True, True, False, True, True]
    pvk, ins, prs = k1
    bad = list(batches)
    bad[1] = (pvk, [[(ins[0][0] + 1) % R]], prs)
    assert verify_batch_keys_rlc(bad, weights) == _host(bad) == [True, False, True, True, True]


def test_keys_model_refuses_b_outside_g2_in_its_own_key_only():
    """the host verifier accepts the outside-G2 proof; the model refuses its key and keeps the others"""
    vk, xs, proof = outside_b_proof(93)
    pvk = V.prepare_verifying_key(vk)
    good = _synthetic(1, 94, 1)
    batches = [good, (pvk, [xs], [proof])]
    assert _host(batches) == [True, True]
    assert verify_batch_keys_rlc(batches, [[5], [7]]) == [True, False]
