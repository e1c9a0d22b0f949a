"""Strict big-int model of CanonicalSerialize / CanonicalDeserialize (ark-serialize, ark-ec, ark-ff and ark-groth16 0.5,
Validate::Yes) of ProvingKey<Bn254> and VerifyingKey<Bn254>, shared by tests/test_ark_key_model.py (CPU) and
tests/test_ark_serialize.py (GPU).  TEST INFRASTRUCTURE ONLY.  The compressed point rules are compressed_model's; this adds:
  - uncompressed points: x then y (G2: x.c0, x.c1, y.c0, y.c1), the flags on the last byte of y (of y.c1); bit 7 is written
    for the larger y and ignored on read; bit 6 = infinity (zero coordinates on write; on read every coordinate must still be
    below p, and the point is infinity whatever its coordinates); both set is invalid; otherwise the point must be on its
    curve, and a G2 point must lie in G2
  - keys: fields in declaration order, a Vec = u64 little-endian length then its elements.
Keys are dicts {field: point or [points]} of canonical affine points, None = infinity."""
import struct

from batch_model import g2_in_subgroup
from compressed_model import FLAG_INF, FLAG_NEG, P, Undecodable, _fq, _key2, g1_decompress, g2_decompress
from oracle import pyref as o

VK_FIELDS = (('alpha_g1', False, False), ('beta_g2', False, True), ('gamma_g2', False, True), ('delta_g2', False, True),
             ('gamma_abc_g1', True, False))
PK_FIELDS = VK_FIELDS + (('beta_g1', False, False), ('delta_g1', False, False), ('a_query', True, False),
                         ('b_g1_query', True, False), ('b_g2_query', True, True), ('h_query', True, False), ('l_query', True, False))


class Refused(ValueError):
    """a refusal: .where names the field and index, as the library's SerializationError does"""

    def __init__(self, where, why):
        super().__init__(f"{where}: {why}")
        self.where = where


def point_size(g2: bool, compress: bool) -> int:
    return (64 if g2 else 32) * (1 if compress else 2)


def _larger(y, g2: bool) -> bool:
    if g2:
        return _key2(y) > _key2(o.FQ2.neg(y))
    return y > (P - y) % P


def _le(vals) -> bytearray:
    return bytearray(b''.join(int(v).to_bytes(32, 'little') for v in vals))


def point_bytes(pt, g2: bool, compress: bool) -> bytes:
    """CanonicalSerialize of one affine point (None = infinity)"""
    k = 2 if g2 else 1
    if pt is None:
        b = _le([0] * (k if compress else 2 * k))
        flags = FLAG_INF
    else:
        x, y = (list(pt[0]), list(pt[1])) if g2 else ([pt[0]], [pt[1]])
        b = _le(x if compress else x + y)
        flags = FLAG_NEG if _larger(pt[1], g2) else 0
    b[-1] |= flags
    return bytes(b)


def on_curve(pt, g2: bool) -> bool:
    if g2:
        x, y = pt
        return o.FQ2.sqr(y) == o.FQ2.add(o.FQ2.mul(o.FQ2.sqr(x), x), o.G2_B)
    x, y = pt
    return (y * y - x * x * x - o.G1_B) % P == 0


def decode_point(b: bytes, g2: bool, compress: bool):
    """CanonicalDeserialize (Validate::Yes) of one point -> affine point or None; raises Undecodable"""
    if compress:
        return g2_decompress(b) if g2 else g1_decompress(b)
    k = 2 if g2 else 1
    vals = [_fq(b[32 * i:32 * i + 32], False)[0] for i in range(2 * k - 1)]
    last, flags = _fq(b[32 * (2 * k - 1):32 * 2 * k], True)
    vals.append(last)
    if flags & FLAG_INF:
        return None
    pt = ((vals[0], vals[1]), (vals[2], vals[3])) if g2 else (vals[0], vals[1])
    if not on_curve(pt, g2):
        raise Undecodable("the point is not on its curve")
    if g2 and not g2_in_subgroup(pt):
        raise Undecodable("the point is not in G2")
    return pt


def serialize(key: dict, fields, compress: bool) -> bytes:
    out = []
    for name, vec, g2 in fields:
        if vec:
            out.append(struct.pack('<Q', len(key[name])))
            out += [point_bytes(p, g2, compress) for p in key[name]]
        else:
            out.append(point_bytes(key[name], g2, compress))
    return b''.join(out)


def deserialize(data: bytes, fields, compress: bool):
    """(key, bytes read); raises Refused at the first refusal in the serialized order"""
    pos, key = 0, {}

    def take(n, where):
        nonlocal pos
        if n > len(data) - pos:
            raise Refused(where, "the input ends early")
        pos += n
        return data[pos - n:pos]

    for name, vec, g2 in fields:
        size = point_size(g2, compress)
        if vec:
            count = struct.unpack('<Q', take(8, name))[0]
            raw = take(count * size, name)
            pts = []
            for i in range(count):
                try:
                    pts.append(decode_point(raw[i * size:(i + 1) * size], g2, compress))
                except Undecodable as e:
                    raise Refused(f"{name}[{i}]", str(e))
            key[name] = pts
        else:
            try:
                key[name] = decode_point(take(size, name), g2, compress)
            except Undecodable as e:
                raise Refused(name, str(e))
    return key, pos


def key_from_pk(pk, fields=PK_FIELDS) -> dict:
    """the canonical points of a ProvingKey's arrays (Montgomery words, all zero = infinity)"""
    from circom_compat_b200.verifier import _g1_from_words, _g2_from_words
    key = {}
    for name, vec, g2 in fields:
        rows = [_g2_from_words(r) if g2 else _g1_from_words(r) for r in getattr(pk, name).reshape(-1, 16 if g2 else 8)]
        key[name] = rows if vec else rows[0]
    return key
