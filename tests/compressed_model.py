"""Strict big-int model of Proof::<Bn254>::deserialize_compressed (ark-serialize, ark-ec and ark-ff 0.5, Validate::Yes), shared
by tests/test_compressed_model.py (CPU) and tests/test_verify_compressed.py (GPU).  TEST INFRASTRUCTURE ONLY.

oracle.pyref.decompress_proof inverts the encoding of a valid proof and checks nothing.  This decoder restates every rule the
device decoder (csrc/verify.cu) follows and refuses what arkworks refuses:
  - layout: A = bytes 0-31, B = 32-95 (x.c0, then x.c1), C = 96-127, little-endian; a point's flags are the top two bits of
    its last byte (bit 7: y is the larger of {y, -y}; bit 6: infinity); both bits set is invalid
  - every Fq value, flags masked off, is below p, even under the infinity flag; the infinity flag ignores x otherwise
  - y^2 = x^3 + b must have a root; the flag picks the larger or smaller root in canonical order (Fq2: c1, then c0)
  - B lies in G2 (G1 has cofactor 1)"""
from batch_model import g2_in_subgroup
from oracle import pyref as o

P = o.Q_MOD
FLAG_NEG, FLAG_INF = 0x80, 0x40
SENTINEL = b'\xff' * 256                  # the row of an undecodable proof


class Undecodable(ValueError):
    pass


def _fq(b: bytes, flagged: bool):
    """an Fq value (32 B little-endian) and the flags of its last byte (flagged) or none"""
    v, flags = int.from_bytes(b, 'little'), 0
    if flagged:
        flags = b[31] & 0xC0
        v &= (1 << 254) - 1
    if flags == FLAG_NEG | FLAG_INF:
        raise Undecodable("both flag bits set")
    if v >= P:
        raise Undecodable("a coordinate is not below p")
    return v, flags


def _key2(y):
    return (y[1], y[0])


def g1_decompress(b: bytes):
    """a compressed G1 point (32 B) -> (x, y), or None at infinity; raises Undecodable"""
    x, f = _fq(b, True)
    if f & FLAG_INF:
        return None
    y = o._fq_sqrt((x * x * x + o.G1_B) % P)
    if y is None:
        raise Undecodable("x^3 + 3 has no square root")
    small, big = sorted((y, (P - y) % P))
    return (x, big if f & FLAG_NEG else small)


def g2_decompress(b: bytes, subgroup: bool = True):
    """a compressed G2 point (64 B) -> ((x0, x1), (y0, y1)), or None at infinity; raises Undecodable"""
    x0, _ = _fq(b[:32], False)
    x1, f = _fq(b[32:64], True)
    if f & FLAG_INF:
        return None
    x = (x0, x1)
    rhs = o.FQ2.add(o.FQ2.mul(o.FQ2.sqr(x), x), o.G2_B)
    y = o._fq2_sqrt(rhs)
    if y is None or o.FQ2.sqr(y) != rhs:
        raise Undecodable("x^3 + b' has no square root")
    small, big = sorted((y, o.FQ2.neg(y)), key=_key2)
    q = (x, big if f & FLAG_NEG else small)
    if subgroup and not g2_in_subgroup(q):
        raise Undecodable("B is not in G2")
    return q


def decompress_proof_checked(data: bytes):
    """(A, B, C) with None at infinity, or None when arkworks refuses the 128 bytes"""
    if len(data) != 128:
        return None
    try:
        return g1_decompress(data[0:32]), g2_decompress(data[32:96]), g1_decompress(data[96:128])
    except Undecodable:
        return None


def proof_row(a, b, c) -> bytes:
    """the 256-byte canonical row of b2g_prove (zeros at infinity)"""
    vals = ([0, 0] if a is None else list(a)) + ([0] * 4 if b is None else [b[0][0], b[0][1], b[1][0], b[1][1]]) + \
           ([0, 0] if c is None else list(c))
    return b''.join(int(v).to_bytes(32, 'little') for v in vals)


def decoded_row(data: bytes) -> bytes:
    """what b2g_proofs_decompress writes for these 128 bytes"""
    d = decompress_proof_checked(data)
    return SENTINEL if d is None else proof_row(*d)


def g1_no_root_x(start: int = 1) -> int:
    """the least x >= start whose x^3 + 3 is not a square"""
    x = start
    while o._fq_sqrt((x ** 3 + 3) % P) is not None:
        x += 1
    return x


def g2_no_root_x(start: int = 1):
    """the least (x0, 1), x0 >= start, whose x^3 + b' is not a square"""
    x0 = start
    while True:
        x = (x0, 1)
        rhs = o.FQ2.add(o.FQ2.mul(o.FQ2.sqr(x), x), o.G2_B)
        y = o._fq2_sqrt(rhs)
        if y is None or o.FQ2.sqr(y) != rhs:
            return x
        x0 += 1


def twist_point_real_y():
    """a twist point (x, y) with y.c1 = 0, the tie of the sign rule: x = (x0, x1) with x0^2 = (x1^2 - b'_1 / x1) / 3 makes
    x^3 + b' lie in Fq, and y = (y0, 0) when that value is a square"""
    inv3 = pow(3, -1, P)
    x1 = 2
    while True:
        x0 = o._fq_sqrt((x1 * x1 - o.G2_B[1] * pow(x1, -1, P)) * inv3 % P)
        if x0 is not None:
            x = (x0, x1)
            rhs = o.FQ2.add(o.FQ2.mul(o.FQ2.sqr(x), x), o.G2_B)
            assert rhs[1] == 0
            y0 = o._fq_sqrt(rhs[0])
            if y0 is not None and y0 != 0:
                return x, (y0, 0)
        x1 += 1


def g2_bytes(x, flags: int = 0) -> bytes:
    """a compressed G2 point from its x and flags"""
    b = bytearray(int(x[0]).to_bytes(32, 'little') + int(x[1]).to_bytes(32, 'little'))
    b[63] |= flags
    return bytes(b)
