"""Big-int model of b2g_verify_batch (csrc/verify.cu), shared by tests/test_batch_model.py (CPU) and tests/test_verify_batch.py
(GPU).  TEST INFRASTRUCTURE ONLY.  It restates the G2 membership test the device runs and the random-linear-combination batch
equation
    prod e(r_i A_i, B_i) * e(sum r_i C_i, -delta) * e(s_0 IC[0] + sum_j s_j IC[j], -gamma) == e(alpha, beta)^s_0,
    s_0 = sum r_i, s_j = sum r_i x_ij (mod r)."""
from circom_compat_b200 import verifier as V
from oracle import pairing_model as M
from oracle import pyref as o

P, R = V.P, o.R_MOD


def _psi(q):
    return None if q is None else M.twist_frobenius(q)


def g2_in_subgroup(q) -> bool:
    """[x + 1] Q + psi([x] Q) + psi^2([x] Q) == psi^3([2x] Q) for Q on the twist (psi: the twist Frobenius)"""
    if q is None:
        return True
    xq = o.G2.mul(q, M.X)
    lhs = o.G2.add(o.G2.add(o.G2.add(xq, q), _psi(xq)), _psi(_psi(xq)))
    return lhs == _psi(_psi(_psi(o.G2.add(xq, xq))))


def verify_batch_rlc(pvk, inputs_list, proofs, weights) -> bool:
    """the verdict b2g_verify_batch computes for these weights (proof coordinates canonical; one >= p fails the batch)"""
    vk = pvk.vk
    pairs, rc = [], None
    for w, proof in zip(weights, proofs):
        a, b, c = V._proof_points(proof)
        coords = [v for pt in (a, c) if pt is not None for v in pt] + ([v for xy in b for v in xy] if b is not None else [])
        if any(v >= P for v in coords) or not (V.g1_on_curve(a) and V.g1_on_curve(c) and V.g2_on_curve(b)):
            return False
        if not g2_in_subgroup(b):
            return False
        pairs.append((V.g1_mul(a, w) if a is not None else None, b))
        rc = V.g1_add(rc, V.g1_mul(c, w) if c is not None else None)
    n_public = len(vk.gamma_abc_g1) - 1
    s = [sum(weights) % R] + [sum(w * xs[j] for w, xs in zip(weights, inputs_list)) % R for j in range(n_public)]
    prep = None
    for k, base in zip(s, vk.gamma_abc_g1):
        prep = V.g1_add(prep, V.g1_mul(base, k) if base is not None else None)
    f = V.miller_loop(pairs + [(rc, pvk.delta_g2_neg), (prep, pvk.gamma_g2_neg)])
    return V.final_exponentiation(f) == V.f12_pow(pvk.alpha_g1_beta_g2, s[0])


def twist_point_outside_g2(rng):
    """a random point on the twist; outside G2 with overwhelming probability (the cofactor is about p)"""
    while True:
        x = (rng.randrange(P), rng.randrange(P))
        y = o._fq2_sqrt(V.f2_add(V.f2_mul(V.f2_sqr(x), x), V.TWIST_B))
        if y is not None:
            return (x, y)


def outside_b_proof(seed):
    """(vk, inputs, (A, B, C)) with A at infinity, B on the twist but outside G2 and C solved so that the pairing equation
    holds: the host verifier and verify_many accept it, and only the G2 membership test can refuse it"""
    import random
    rng = random.Random(seed)
    al, be, ga, de = (rng.randrange(1, R) for _ in range(4))
    ic = [rng.randrange(1, R) for _ in range(2)]
    g1, g2 = (lambda k: o.G1.mul(o.G1_GEN, k)), (lambda k: o.G2.mul(o.G2_GEN, k))
    vk = V.VerifyingKey(g1(al), g2(be), g2(ga), g2(de), [g1(k) for k in ic])
    xs = [rng.randrange(R)]
    c = -(al * be + (ic[0] + xs[0] * ic[1]) * ga) * pow(de, -1, R) % R
    return vk, xs, (None, twist_point_outside_g2(rng), g1(c))
