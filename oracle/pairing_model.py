"""Big-int model of the device pairing (circom_compat_b200/csrc/pairing.cuh) and batched verifier (csrc/verify.cu).
TEST INFRASTRUCTURE ONLY.

It restates, step by step, what the device computes, on the same Fq2 -> Fq6 -> Fq12 tower as the host verifier
(u^2 = -1, v^3 = 9 + u, w^2 = v; an Fq12 is ((c0.c0, c0.c1, c0.c2), (c1.c0, c1.c1, c1.c2)) of Fq2):
  - Miller loop over the signed digits of 6x + 2 with homogeneous projective line steps on the twist (no inversion), the
    line f * (c0 py + c1 px w + c2 w^3) as the sparse product `mul_by_034`, then the two Frobenius lines pi(Q), -pi^2(Q);
  - the prepared coefficient list of a fixed G2 argument (one (c0, c1, c2) triple per step, in loop order);
  - the final exponentiation: easy part conj(f) / f then g^(p^2) g, hard part as the exact decomposition
    (p^4 - p^2 + 1) / r = l3 p^3 + l2 p^2 + l1 p + l0 in x and p (Scott et al.), three exp-by-x chains on
    Granger-Scott cyclotomic squarings plus Frobenius maps.
Projective lines differ from the host's affine ones by a factor in Fq2, which the final exponentiation removes, so
pairing values are equal to verifier.pairing bit for bit while Miller-loop values are not.

`python -m oracle.pairing_model` prints the constants pairing.cuh pins (Montgomery limbs)."""
from __future__ import annotations

from circom_compat_b200 import verifier as V
from circom_compat_b200.verifier import (F2_ONE, F2_ZERO, F6_ZERO, F12_ONE, P, f2_add, f2_conj, f2_mul, f2_mul_xi, f2_neg,
                                         f2_pow, f2_scale, f2_sqr, f2_sub, f6_add, f6_mul, f6_sub, f12_conj, f12_inv, f12_mul)
from circom_compat_b200.zkey import R_MOD

X = 4965661367192848881                                  # BN parameter x (positive for BN254)
ATE = 6 * X + 2


def naf(k: int) -> list:
    """non-adjacent form, most significant digit first"""
    out = []
    while k:
        if k & 1:
            d = 2 - (k & 3)
            k -= d
        else:
            d = 0
        out.append(d)
        k >>= 1
    return out[::-1]


ATE_NAF = naf(ATE)                                       # ATE_NAF[0] == 1; the loop runs over ATE_NAF[1:]

# Frobenius coefficients: (c w^e)^(p^k) = c^(p^k) w^e xi^(e (p^k - 1) / 6), e = position of the coefficient in w
# (c0.c0 -> 0, c1.c0 -> 1, c0.c1 -> 2, c1.c1 -> 3, c0.c2 -> 4, c1.c2 -> 5)
FROB = {k: [f2_pow(V.XI, e * (P ** k - 1) // 6) for e in range(6)] for k in (1, 2, 3)}
TWIST_FROB_X, TWIST_FROB_Y = f2_pow(V.XI, (P - 1) // 3), f2_pow(V.XI, (P - 1) // 2)         # pi(Q) on the twist
TWIST_FROB2_X, TWIST_FROB2_Y = f2_pow(V.XI, (P * P - 1) // 3), f2_pow(V.XI, (P * P - 1) // 2)
TWIST_B = V.TWIST_B


# ---------------------------------------------------------------------------------------------- Fq12 pieces
def f12_sqr(a):
    """complex squaring: (a0 + a1 w)^2 = (a0 + a1)(a0 + v a1) - a0 a1 - v a0 a1 + 2 a0 a1 w"""
    t = f6_mul(a[0], a[1])
    c0 = f6_sub(f6_sub(f6_mul(f6_add(a[0], a[1]), f6_add(a[0], V.f6_mul_v(a[1]))), t), V.f6_mul_v(t))
    return (c0, f6_add(t, t))


def mul_by_034(f, c0, c3, c4):
    """f * (c0 + c3 w + c4 w^3), c0, c3, c4 in Fq2 (the line as ((c0, 0, 0), (c3, c4, 0)))"""
    a = f6_mul_by_0(f[0], c0)
    b = f6_mul_by_01(f[1], c3, c4)
    c1 = f6_sub(f6_sub(f6_mul_by_01(f6_add(f[0], f[1]), f2_add(c0, c3), c4), a), b)
    return (f6_add(a, V.f6_mul_v(b)), c1)


def f6_mul_by_0(a, c0):
    return (f2_mul(a[0], c0), f2_mul(a[1], c0), f2_mul(a[2], c0))


def f6_mul_by_01(a, b0, b1):
    """a * (b0 + b1 v): five Fq2 products (Karatsuba on the two nonzero coefficients)"""
    t0, t1 = f2_mul(a[0], b0), f2_mul(a[1], b1)
    c0 = f2_add(f2_mul_xi(f2_mul(a[2], b1)), t0)
    c1 = f2_sub(f2_sub(f2_mul(f2_add(a[0], a[1]), f2_add(b0, b1)), t0), t1)
    c2 = f2_add(f2_mul(a[2], b0), t1)
    return (c0, c1, c2)


def frobenius(f, k):
    """f^(p^k), k = 1, 2, 3: coefficient at w^e -> (conj if k odd)(c) * FROB[k][e]"""
    g = FROB[k]
    m = (lambda c: f2_conj(c)) if k & 1 else (lambda c: c)
    return ((m(f[0][0]), f2_mul(m(f[0][1]), g[2]), f2_mul(m(f[0][2]), g[4])),
            (f2_mul(m(f[1][0]), g[1]), f2_mul(m(f[1][1]), g[3]), f2_mul(m(f[1][2]), g[5])))


def cyclotomic_sqr(f):
    """Granger-Scott squaring of an element of the cyclotomic subgroup (f^(p^6 + 1) = 1 after the easy part): Fq12 as
    Fq4^3 with Fq4 = Fq2[s] / (s^2 - xi); three Fq4 squarings, six Fq2 products."""
    z0, z4, z3 = f[0]
    z2, z1, z5 = f[1]

    def fq4_sqr(a, b):                                   # (a + b s)^2 = (a^2 + xi b^2) + 2ab s
        t = f2_mul(a, b)
        return (f2_sub(f2_sub(f2_mul(f2_add(a, b), f2_add(a, f2_mul_xi(b))), t), f2_mul_xi(t)), f2_add(t, t))

    t0, t1 = fq4_sqr(z0, z1)
    t2, t3 = fq4_sqr(z2, z3)
    t4, t5 = fq4_sqr(z4, z5)

    def three_minus_two(t, z): return f2_add(f2_scale(f2_sub(t, z), 2), t)            # 3t - 2z
    def three_plus_two(t, z): return f2_add(f2_scale(f2_add(t, z), 2), t)             # 3t + 2z
    z0 = three_minus_two(t0, z0)
    z1 = three_plus_two(t1, z1)
    z2 = three_plus_two(f2_mul_xi(t5), z2)
    z3 = three_minus_two(t4, z3)
    z4 = three_minus_two(t2, z4)
    z5 = three_plus_two(t3, z5)
    return ((z0, z4, z3), (z2, z1, z5))


def exp_by_x(f):
    """f^x for a cyclotomic f: square-and-multiply over the bits of x (63 cyclotomic squarings)"""
    r = f
    for bit in bin(X)[3:]:
        r = cyclotomic_sqr(r)
        if bit == '1':
            r = f12_mul(r, f)
    return r


def final_exponentiation(f):
    g = f12_mul(f12_conj(f), f12_inv(f))                 # f^(p^6 - 1)
    g = f12_mul(frobenius(g, 2), g)                      # ^(p^2 + 1): now in the cyclotomic subgroup
    fx = exp_by_x(g)
    fx2 = exp_by_x(fx)
    fx3 = exp_by_x(fx2)
    y0 = f12_mul(f12_mul(frobenius(g, 1), frobenius(g, 2)), frobenius(g, 3))
    y1 = f12_conj(g)
    y2 = frobenius(fx2, 2)
    y3 = f12_conj(frobenius(fx, 1))
    y4 = f12_conj(f12_mul(fx, frobenius(fx2, 1)))
    y5 = f12_conj(fx2)
    y6 = f12_conj(f12_mul(fx3, frobenius(fx3, 1)))
    t0 = f12_mul(f12_mul(cyclotomic_sqr(y6), y4), y5)
    t1 = f12_mul(f12_mul(y3, y5), t0)
    t0 = f12_mul(t0, y2)
    t1 = f12_mul(cyclotomic_sqr(t1), t0)
    t1 = cyclotomic_sqr(t1)
    t0 = f12_mul(t1, y1)
    t1 = f12_mul(t1, y0)
    return f12_mul(cyclotomic_sqr(t0), t1)


def hard_chain_exponent() -> int:
    """the exponent final_exponentiation's hard part applies, as an integer (same chain on exponents)"""
    p = P
    fx, fx2, fx3 = X, X * X, X ** 3
    y0, y1, y2, y3 = p + p * p + p ** 3, -1, fx2 * p * p, -fx * p
    y4, y5, y6 = -(fx + fx2 * p), -fx2, -(fx3 + fx3 * p)
    t0 = 2 * y6 + y4 + y5
    t1 = y3 + y5 + t0
    t0 = t0 + y2
    t1 = 2 * (2 * t1 + t0)
    t0, t1 = t1 + y1, t1 + y0
    return 2 * t0 + t1


# ---------------------------------------------------------------------------------------------- projective line steps
def dbl_step(t):
    """T = (X, Y, Z) homogeneous on the twist: 2T and the tangent's coefficients (c0, c1, c2) = (-2YZ, 3X^2, 3b'Z^2 - Y^2);
    the line at P is c0 py + c1 px w + c2 w^3 (= -2 y Z^2 times the affine tangent)"""
    x, y, z = t
    a = f2_scale(f2_mul(x, y), pow(2, -1, P))
    b, c = f2_sqr(y), f2_sqr(z)
    e = f2_mul(TWIST_B, f2_scale(c, 3))
    f = f2_scale(e, 3)
    g = f2_scale(f2_add(b, f), pow(2, -1, P))
    h = f2_sub(f2_sqr(f2_add(y, z)), f2_add(b, c))
    i = f2_sub(e, b)
    j = f2_sqr(x)
    e2 = f2_sqr(e)
    t2 = (f2_mul(a, f2_sub(b, f)), f2_sub(f2_sqr(g), f2_scale(e2, 3)), f2_mul(b, h))
    return t2, (f2_neg(h), f2_scale(j, 3), i)


def add_step(t, q):
    """T + Q for affine Q and the chord's coefficients (c0, c1, c2) = (X - qx Z, -(Y - qy Z), theta qx - lambda qy)"""
    x, y, z = t
    qx, qy = q
    theta = f2_sub(y, f2_mul(qy, z))
    lam = f2_sub(x, f2_mul(qx, z))
    c, d = f2_sqr(theta), f2_sqr(lam)
    e = f2_mul(lam, d)
    f = f2_mul(z, c)
    g = f2_mul(x, d)
    h = f2_sub(f2_add(e, f), f2_scale(g, 2))
    t2 = (f2_mul(lam, h), f2_sub(f2_mul(theta, f2_sub(g, h)), f2_mul(e, y)), f2_mul(z, e))
    return t2, (lam, f2_neg(theta), f2_sub(f2_mul(theta, qx), f2_mul(lam, qy)))


def twist_frobenius(q):
    return (f2_mul(f2_conj(q[0]), TWIST_FROB_X), f2_mul(f2_conj(q[1]), TWIST_FROB_Y))


def twist_frobenius2_neg(q):
    return (f2_mul(q[0], TWIST_FROB2_X), f2_neg(f2_mul(q[1], TWIST_FROB2_Y)))


def prepare_g2(q) -> list:
    """coefficient triples of every step of the loop for the fixed G2 point q (affine, not infinity), in the order the
    Miller loop consumes them: per digit one doubling, then one addition of +-q if the digit is nonzero; then pi(q), -pi^2(q)"""
    t = (q[0], q[1], F2_ONE)
    nq = (q[0], f2_neg(q[1]))
    out = []
    for d in ATE_NAF[1:]:
        t, l = dbl_step(t)
        out.append(l)
        if d:
            t, l = add_step(t, q if d == 1 else nq)
            out.append(l)
    t, l = add_step(t, twist_frobenius(q))
    out.append(l)
    _, l = add_step(t, twist_frobenius2_neg(q))
    out.append(l)
    return out


def ell(f, coeffs, p):
    c0, c1, c2 = coeffs
    return mul_by_034(f, f2_scale(c0, p[1]), f2_scale(c1, p[0]), c2)


def miller_loop(pairs) -> tuple:
    """pairs = [(P affine G1 or None, Q affine G2 or None or a prepare_g2 list)]; a pair with infinity contributes 1"""
    live = [(p, q if isinstance(q, list) else prepare_g2(q)) for p, q in pairs if p is not None and q is not None]
    f = F12_ONE
    idx = 0
    for k, d in enumerate(ATE_NAF[1:]):
        if k:
            f = f12_sqr(f)
        for p, c in live:
            f = ell(f, c[idx], p)
        idx += 1
        if d:
            for p, c in live:
                f = ell(f, c[idx], p)
            idx += 1
    for _ in range(2):
        for p, c in live:
            f = ell(f, c[idx], p)
        idx += 1
    return f


def pairing(p, q):
    return final_exponentiation(miller_loop([(p, q)]))


# ---------------------------------------------------------------------------------------------- batched verifier
def verify_batch(pvk, inputs_list, proofs) -> list:
    """verdicts as b2g_verify_many computes them: prepared inputs from IC, one multi-Miller loop over (A, B), (prepared, -gamma)
    and (C, -delta) with the fixed arguments prepared once, the final exponentiation compared with e(alpha, beta).  Proof
    coordinates are canonical integers; one >= p makes the proof invalid (the host verifier reduces it instead)."""
    vk = pvk.vk
    lines_g = prepare_g2(pvk.gamma_g2_neg) if pvk.gamma_g2_neg is not None else None
    lines_d = prepare_g2(pvk.delta_g2_neg) if pvk.delta_g2_neg is not None else None
    out = []
    for xs, proof in zip(inputs_list, proofs):
        a, b, c = V._proof_points(proof)
        coords = [v for pt in (a, c) if pt is not None for v in pt] + ([v for xy in b for v in xy] if b is not None else [])
        if any(v >= P for v in coords) or not (V.g1_on_curve(a) and V.g1_on_curve(c) and V.g2_on_curve(b)):
            out.append(False)
            continue
        prepared = V.prepare_inputs(pvk, xs)
        f = miller_loop([(a, b), (prepared, lines_g), (c, lines_d)])
        out.append(final_exponentiation(f) == pvk.alpha_g1_beta_g2)
    return out


# ---------------------------------------------------------------------------------------------- constants for pairing.cuh
_R = 1 << 256


def mont_limbs(v: int) -> list:
    m = v * _R % P
    return [(m >> (32 * i)) & 0xFFFFFFFF for i in range(8)]


def pinned_constants() -> dict:
    """name -> list of Fq2 values, the constants pairing.cuh pins (the twist Frobenius reuses FROB1 / FROB2)"""
    return {'FROB1': FROB[1][1:], 'FROB2': FROB[2][1:], 'FROB3': FROB[3][1:], 'TWIST_B3': [f2_scale(TWIST_B, 3)],
            'INV2': [((P + 1) // 2, 0)]}


def ate_digits_cuda() -> str:
    return ', '.join(str(d) for d in ATE_NAF[1:])


if __name__ == '__main__':
    for name, vals in pinned_constants().items():
        print(f"// {name}")
        for v in vals:
            print('    {{' + ', '.join(f'0x{w:08x}u' for w in mont_limbs(v[0])) + '}, {' +
                  ', '.join(f'0x{w:08x}u' for w in mont_limbs(v[1])) + '}},')
    print(f"// ATE_NAF ({len(ATE_NAF) - 1} digits after the leading 1)")
    print('    ' + ate_digits_cuda())
