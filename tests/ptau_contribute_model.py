"""Big-int model of b2g_points_scale's scalar decomposition and signed-window recoding, and of a phase-1 contribution.

G1 (GLV): phi(x, y) = (beta x, y), beta a primitive cube root of unity in Fq, acts on G1 as [lambda], lambda a primitive cube
root of unity mod r.  Of the two roots, LAMBDA is the one that matches BETA (checked on the generator).  A short basis
(A1, B1), (A2, B2) of the lattice {(a, b): a + b lambda = 0 mod r} comes from the extended Euclidean algorithm; Babai rounding
    c1 = (k G1R) >> 256,  c2 = (k G2R) >> 256,  G1R = round(2^256 B2 / r),  G2R = round(-2^256 B1 / r)
    k1 = k - c1 A1 - c2 A2,  k2 = -c1 B1 - c2 B2
gives k = k1 + k2 lambda (mod r) with |k1|, |k2| < 2^128.  The device computes k1, k2 in two's complement mod 2^192.
G2 (GLS): psi, the twist Frobenius, acts on G2 as [6x^2] (p = r + 6x^2), so k1 = k mod 6x^2 and k2 = k div 6x^2, both < 2^127.
Recoding: a half h < 2^128 is read as 33 signed digits d_i = nib_i(h) + bit_(4i-1)(h) - 16 bit_(4i+3)(h) in [-8, 8], so that
h = sum d_i 16^i; the device reads them from the top with no stored digits.
"""
from oracle.pairing_model import X as BN_X
from oracle.pyref import Q_MOD, R_MOD

WINDOW, DIGITS = 4, 33
GLS_D = 6 * BN_X * BN_X                       # p mod r: psi acts on G2 as [GLS_D]
GLS_MU = (1 << 256) // GLS_D                  # floor(2^256 / GLS_D): the device's quotient estimate


def _cube_roots(m):
    """the two primitive cube roots of unity mod the prime m"""
    for g in range(2, 100):
        w = pow(g, (m - 1) // 3, m)
        if w != 1:
            return sorted((w, w * w % m))
    raise AssertionError


def _lambda_for(beta):
    """the cube root of unity mod r that phi with this beta multiplies G1 by: phi(G) == lambda G on the generator"""
    from oracle.pyref import G1, G1_GEN
    phi_g = (beta * G1_GEN[0] % Q_MOD, G1_GEN[1])
    for lam in _cube_roots(R_MOD):
        if G1.mul(G1_GEN, lam) == phi_g:
            return lam
    raise AssertionError("no cube root of unity mod r matches beta")


BETA = _cube_roots(Q_MOD)[0]
LAMBDA = _lambda_for(BETA)


def _short_basis(lam):
    """two short vectors (a, b) with a + b lam = 0 (mod r), by the extended Euclidean algorithm on (r, lam) (GLV, section 4)"""
    r0, r1, t0, t1 = R_MOD, lam, 0, 1
    rows = [(r0, t0), (r1, t1)]
    while r1 * r1 >= R_MOD:
        q = r0 // r1
        r0, r1, t0, t1 = r1, r0 - q * r1, t1, t0 - q * t1
        rows.append((r1, t1))
    # rows[-2] is the last remainder >= sqrt(r); rows[-1] the first below.  v1 = (r_(l+1), -t_(l+1))
    (rl, tl), (rl1, tl1) = rows[-2], rows[-1]
    r2, t2 = rl - (rl // rl1) * rl1, tl - (rl // rl1) * tl1
    v1 = (rl1, -tl1)
    v2 = min(((rl, -tl), (r2, -t2)), key=lambda v: v[0] * v[0] + v[1] * v[1])
    for a, b in (v1, v2):
        assert (a + b * lam) % R_MOD == 0
    return v1, v2


(A1, B1), (A2, B2) = _short_basis(LAMBDA)
if B2 < 0:                                    # signs chosen so that both rounding constants are positive
    A2, B2 = -A2, -B2
if B1 > 0:
    A1, B1 = -A1, -B1
G1R = ((B2 << 256) + R_MOD // 2) // R_MOD
G2R = ((-B1 << 256) + R_MOD // 2) // R_MOD
HALF_BOUND = 1 << 128
_M192 = (1 << 192) - 1


def glv_split(k):
    """(k1, k2) signed, as the device computes them: k = k1 + k2 LAMBDA (mod r)"""
    c1, c2 = (k * G1R) >> 256, (k * G2R) >> 256
    k1 = (k - c1 * A1 - c2 * A2) & _M192
    k2 = (-c1 * B1 - c2 * B2) & _M192
    k1 = k1 - (1 << 192) if k1 >> 191 else k1
    k2 = k2 - (1 << 192) if k2 >> 191 else k2
    return k1, k2


def gls_split(k):
    """(k1, k2) = (k mod 6x^2, k div 6x^2) by the device's route: a quotient estimate from GLS_MU, then corrections"""
    q = (k * GLS_MU) >> 256
    rem = k - q * GLS_D
    while rem >= GLS_D:
        rem -= GLS_D
        q += 1
    return rem, q


def digits(h):
    """the 33 signed digits of a half h in [0, 2^128), lowest first"""
    bit = lambda i: (h >> i) & 1 if i >= 0 else 0
    return [((h >> (4 * i)) & 15) + bit(4 * i - 1) - 16 * bit(4 * i + 3) for i in range(DIGITS)]


def edge_scalars():
    """scalars at the decomposition's edges: 0, 1, 2, r - 1, lambda and its neighbours, 6x^2 and its neighbours, 2^127, 2^128
    and their neighbours, and the scalars where the G1 rounding steps (c1 or c2 changes) and their neighbours"""
    out = {0, 1, 2, R_MOD - 1, R_MOD - 2, LAMBDA - 1, LAMBDA, LAMBDA + 1, GLS_D - 1, GLS_D, GLS_D + 1, 2 * GLS_D,
           1 << 127, (1 << 128) - 1, 1 << 128, (1 << 128) + 1, LAMBDA * LAMBDA % R_MOD, R_MOD - GLS_D}
    for g in (G1R, G2R):
        for c in (1, 2, 12345, (1 << 100) + 7):
            k = -((-c << 256) // g)           # the least k with (k g) >> 256 >= c
            out.update(x for x in (k - 1, k, k + 1) if 0 <= x < R_MOD)
    return sorted(out)


def mont_limbs(v):
    """the four little-endian u64 words of v in Montgomery form over Fq"""
    m = (v << 256) % Q_MOD
    return [(m >> (64 * i)) & (2 ** 64 - 1) for i in range(4)]
