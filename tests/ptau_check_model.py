"""Big-int model of b2g_powers_check (include/b2groth.h): the point rules, then the random linear combination of the
ratio rules, with the oracle's scalar products and the host pairing of verifier.py; a maker of small ceremonies by the
oracle's products, and the shifted-sum identities the check relies on.  Written from the check's definition, not from the
kernels."""
import numpy as np

from circom_compat_b200.zkey import Q_MOD, R_MOD


ARRAYS = ('tau_g1', 'tau_g2', 'alpha_tau_g1', 'beta_tau_g1', 'beta_g2')
_MONT_R_INV = pow(1 << 256, -1, Q_MOD)


def point_of(row, g2):
    """(raw Montgomery words as ints, canonical affine point or None for all-zero)"""
    raw = np.ascontiguousarray(row, dtype='<u8').tobytes()
    words = [int.from_bytes(raw[k:k + 32], 'little') for k in range(0, len(raw), 32)]
    c = [w * _MONT_R_INV % Q_MOD for w in words]
    if not any(words):
        return words, None
    return words, (((c[0], c[1]), (c[2], c[3])) if g2 else (c[0], c[1]))


def point_rule(row, g2, gen) -> int:
    """the first rule the point breaks: 1 a coordinate >= p, 2 off its curve, 3 at infinity, 4 outside G2, 5 not the generator
    (only with gen); 0 when it passes"""
    from batch_model import g2_in_subgroup
    from oracle import pyref as o
    words, pt = point_of(row, g2)
    if any(w >= Q_MOD for w in words):
        return 1
    if not (o.G2 if g2 else o.G1).on_curve(pt):
        return 2
    if pt is None:
        return 3
    if g2 and not g2_in_subgroup(pt):
        return 4
    if gen and pt != (o.G2_GEN if g2 else o.G1_GEN):
        return 5
    return 0


def prefix_arrays(powers, log_n):
    n = 1 << log_n
    counts = (2 * n - 1, n, n, n, 1)
    return [np.asarray(getattr(powers, name))[:c] for name, c in zip(ARRAYS, counts)]


def check(powers, log_n, challenges):
    """(ok, rule, array name, index): the verdict b2g_powers_check gives for these challenges (rho, sigma, pi, kappa, eps)"""
    from circom_compat_b200 import verifier as V
    from oracle import pyref as o
    arrays = prefix_arrays(powers, log_n)
    pts = []
    for a, (name, arr) in enumerate(zip(ARRAYS, arrays)):
        g2 = name in ('tau_g2', 'beta_g2')
        for i, row in enumerate(arr):
            rule = point_rule(row, g2, a in (0, 1) and i == 0)
            if rule:
                return False, rule, name, i
        pts.append([point_of(row, g2)[1] for row in arr])
    T, U, A, B, (b2,) = pts
    rho, sigma, pi, kappa, eps = challenges
    n = 1 << log_n
    S = {k: X for k, X in zip('TUAB', (T, U, A, B))}
    G = {k: (o.G2 if k == 'U' else o.G1) for k in 'TUAB'}
    sums = {k: G[k].sum([G[k].mul(x, pow(rho, i, R_MOD)) for i, x in enumerate(S[k])]) for k in 'TUAB'}
    g1 = o.G1

    def sub(c, x, y):
        return c.add(x, c.neg(y))
    p_hi = g1.sum([sub(g1, sums['T'], T[0]), g1.mul(sub(g1, sums['A'], A[0]), sigma), g1.mul(sub(g1, sums['B'], B[0]), pi),
                   g1.mul(B[0], eps)])
    x_t = sub(g1, sums['T'], g1.mul(T[2 * n - 2], pow(rho, 2 * n - 2, R_MOD)))
    x_a = sub(g1, sums['A'], g1.mul(A[n - 1], pow(rho, n - 1, R_MOD)))
    x_b = sub(g1, sums['B'], g1.mul(B[n - 1], pow(rho, n - 1, R_MOD)))
    p_lo = g1.mul(g1.sum([x_t, g1.mul(x_a, sigma), g1.mul(x_b, pi)]), rho)
    q3 = sub(o.G2, sums['U'], U[0])
    q4 = sub(o.G2, sums['U'], o.G2.mul(U[n - 1], pow(rho, n - 1, R_MOD)))
    pairs = [(p_hi, U[0]), (g1.neg(p_lo), U[1]), (g1.mul(T[0], kappa), q3), (g1.neg(g1.mul(T[1], kappa * rho)), q4),
             (g1.neg(g1.mul(T[0], eps)), b2)]
    ok = V.final_exponentiation(V.miller_loop(pairs)) == V.F12_ONE
    return (True, 0, None, None) if ok else (False, 6, None, None)


class CpuCeremony:
    """the arrays of a ceremony of size 2^power for (tau, alpha, beta) on the standard generators, by the oracle's scalar
    products (small powers only), with the fields of ptau.read_ptau's result"""

    def __init__(self, power, tau, alpha, beta):
        from circom_compat_b200.groth16 import _mont_points
        from oracle import pyref as o
        n = 1 << power
        self.power = self.ceremony_power = power
        t = [pow(tau, i, R_MOD) for i in range(2 * n - 1)]
        self.tau_g1 = _mont_points([o.G1.mul(o.G1_GEN, v) for v in t], False).reshape(-1, 8)
        self.tau_g2 = _mont_points([o.G2.mul(o.G2_GEN, v) for v in t[:n]], True).reshape(-1, 16)
        self.alpha_tau_g1 = _mont_points([o.G1.mul(o.G1_GEN, alpha * v) for v in t[:n]], False).reshape(-1, 8)
        self.beta_tau_g1 = _mont_points([o.G1.mul(o.G1_GEN, beta * v) for v in t[:n]], False).reshape(-1, 8)
        self.beta_g2 = _mont_points([o.G2.mul(o.G2_GEN, beta)], True).reshape(-1, 16)


def shifted_sums(xs, rho):
    """(sum_{i<M-1} rho^i X_{i+1}, sum_{i<M-1} rho^i X_i) for integers X_i (discrete logs), and the same from S_X alone"""
    m = len(xs)
    s = sum(pow(rho, i, R_MOD) * x for i, x in enumerate(xs)) % R_MOD
    direct = (sum(pow(rho, i, R_MOD) * xs[i + 1] for i in range(m - 1)) % R_MOD,
              sum(pow(rho, i, R_MOD) * xs[i] for i in range(m - 1)) % R_MOD)
    from_s = (pow(rho, -1, R_MOD) * (s - xs[0]) % R_MOD, (s - pow(rho, m - 1, R_MOD) * xs[m - 1]) % R_MOD)
    return direct, from_s
