"""Raw XYZZ records for the device's group-operation test ops, built and checked in plain big-int arithmetic.
TEST INFRASTRUCTURE ONLY.

A record is X || Y || ZZ || ZZZ, each coordinate a Montgomery residue (G1: 4 words each, G2: c0 || c1, 8 words each), with
x = X / ZZ, y = Y / ZZZ, ZZ^3 = ZZZ^2 and infinity iff ZZ == 0.  Affine points are the oracle's: (x, y) canonical ints (G2:
(c0, c1) pairs) or None, as rows of Montgomery words with all-zero = infinity."""
from __future__ import annotations

import numpy as np

from .pyref import Q_MOD, G1, G2, _Fq, _Fq2, _fq_sqrt, _fq2_sqrt

R = 1 << 256
RINV = pow(R, -1, Q_MOD)


def _ints(words):
    b = np.ascontiguousarray(words, dtype='<u8').tobytes()
    return [int.from_bytes(b[i:i + 32], 'little') for i in range(0, len(b), 32)]


def _words(vals):
    return np.frombuffer(b''.join(int(v).to_bytes(32, 'little') for v in vals), dtype='<u8').copy()


class _G:
    def __init__(self, g2):
        self.g2 = g2
        self.F = _Fq2 if g2 else _Fq
        self.curve = G2 if g2 else G1
        self.k = 2 if g2 else 1                       # Fq limbs-of-32-bytes per element

    def flat(self, e):
        return list(e) if self.g2 else [e]

    def group(self, raw):                             # list of raw residues -> elements (still raw)
        return [tuple(raw[i:i + 2]) for i in range(0, len(raw), 2)] if self.g2 else list(raw)

    def canon(self, e):
        return tuple(v * RINV % Q_MOD for v in e) if self.g2 else e * RINV % Q_MOD

    def mont(self, e):
        return tuple(v * R % Q_MOD for v in e) if self.g2 else e * R % Q_MOD


G1X, G2X = _G(False), _G(True)


def gx(g2):
    return G2X if g2 else G1X


def aff(row, g2):
    """oracle affine row (Montgomery words) -> (x, y) canonical, or None"""
    G = gx(g2)
    raw = _ints(row)
    if not any(raw):
        return None
    x, y = G.group(raw)
    return G.canon(x), G.canon(y)


def aff_row(P, g2):
    """(x, y) canonical or None -> affine row of Montgomery words"""
    G = gx(g2)
    if P is None:
        return np.zeros(8 * G.k, dtype=np.uint64)
    return _words(G.flat(G.mont(P[0])) + G.flat(G.mont(P[1])))


def record(P, z, g2):
    """the XYZZ record of P with X = x z^2, Y = y z^3, ZZ = z^2, ZZZ = z^3 (all-zero for P = None)"""
    G = gx(g2)
    if P is None:
        return np.zeros(16 * G.k, dtype=np.uint64)
    F = G.F
    zz = F.sqr(z)
    zzz = F.mul(zz, z)
    coords = (F.mul(P[0], zz), F.mul(P[1], zzz), zz, zzz)
    return _words([v for e in coords for v in G.flat(G.mont(e))])


def z_for_raw_x(P, target_raw, g2):
    """a z that makes the record's stored X (Montgomery residue) equal target_raw, or None when x-ratio is not a square"""
    G = gx(g2)
    F = G.F
    t = G.canon(target_raw if not g2 else tuple(target_raw))
    zz = F.mul(t, F.inv(P[0]))
    z = _fq2_sqrt(zz) if g2 else _fq_sqrt(zz)
    if z is None or (g2 and None in z) or F.sqr(z) != zz:
        return None
    return z


def z_for_raw_zz(target_raw, g2):
    """a z whose stored ZZ equals target_raw, or None"""
    G = gx(g2)
    F = G.F
    zz = G.canon(target_raw if not g2 else tuple(target_raw))
    z = _fq2_sqrt(zz) if g2 else _fq_sqrt(zz)
    if z is None or (g2 and None in z) or F.sqr(z) != zz:
        return None
    return z


def check_record(words, P, g2, strict_inf=False):
    """None if the raw record `words` holds the point P (None = infinity), else a description of what is wrong.
    Every coordinate must be fully reduced; strict_inf: infinity must be all four coordinates zero."""
    G = gx(g2)
    F = G.F
    raw = _ints(words)
    if any(v >= Q_MOD for v in raw):
        return 'coordinate not reduced below q'
    X, Y, ZZ, ZZZ = (G.canon(e) for e in G.group(raw))
    if P is None:
        if not F.is_zero(ZZ):
            return 'expected infinity, ZZ != 0'
        if strict_inf and any(raw):
            return 'infinity record not all zero'
        return None
    if F.is_zero(ZZ):
        return 'unexpected infinity'
    if F.mul(F.sqr(ZZ), ZZ) != F.sqr(ZZZ):
        return 'ZZ^3 != ZZZ^2'
    if X != F.mul(P[0], ZZ):
        return 'X != x ZZ'
    if Y != F.mul(P[1], ZZZ):
        return 'Y != y ZZZ'
    return None


def addition_cases(rng, g2, pts):
    """(label, acc point, z, q point) for acc += q over the points `pts` (affine tuples, at least three): a generic sum,
    acc == q, acc == -q, q at infinity, acc at infinity and both, each for every z of z_values (z = 1: an affine
    accumulator), plus accumulators whose stored X has extreme limbs"""
    curve = gx(g2).curve
    cases = []
    for j, z in enumerate(z_values(rng, g2)):
        P, Q = pts[j % len(pts)], pts[(j + 1) % len(pts)]
        cases += [('generic', P, z, Q), ('acc == q', P, z, P), ('acc == -q', P, z, curve.neg(P)), ('q inf', P, z, None),
                  ('acc inf', None, z, P), ('both inf', None, z, None)]
    for j, t in enumerate(extreme_raw(rng)):
        P = pts[j % len(pts)]
        z = z_for_raw_x(P, (t, t) if g2 else t, g2)
        if z is not None:
            cases += [('extreme X, generic', P, z, pts[(j + 2) % len(pts)]), ('extreme X, acc == q', P, z, P),
                      ('extreme X, acc == -q', P, z, curve.neg(P))]
    return cases


def z_values(rng, g2):
    """z = 1, -1, random, components zero (G2), and z that put limb-extreme values into the stored ZZ"""
    q = Q_MOD
    if not g2:
        zs = [1, q - 1, rng.randrange(2, q), rng.randrange(2, q)]
        for t in extreme_raw(rng):
            z = z_for_raw_zz(t, False)
            if z is not None:
                zs.append(z)
    else:
        zs = [(1, 0), (q - 1, 0), (rng.randrange(q), rng.randrange(q)), (0, rng.randrange(1, q)), (rng.randrange(2, q), 0),
              (0, 1), (0, q - 1)]
        ext = extreme_raw(rng)
        for t0, t1 in zip(ext, ext[::-1]):
            z = z_for_raw_zz((t0, t1), True)
            if z is not None:
                zs.append(z)
    return zs


def extreme_raw(rng):
    """Montgomery residues with extreme 32-bit limb patterns (all below q)"""
    m = 0xffffffff
    pats = [Q_MOD - 1, Q_MOD - 2, 1, 2, m, (1 << 64) - 1, (1 << 224) - 1, (1 << 253) - 1, 1 << 253, 1 << 31, m << 224,
            sum(m << (32 * i) for i in range(0, 8, 2)) % Q_MOD, sum(0x80000000 << (32 * i) for i in range(8)) % Q_MOD,
            Q_MOD - (1 << 32), Q_MOD >> 1]
    return pats + [sum(rng.choice([0, 1, m, m - 1, 0x80000000, 0x7fffffff]) << (32 * i) for i in range(8)) % Q_MOD for _ in range(4)]
