"""Groth16 keys in the form arkworks stores them: CanonicalSerialize / CanonicalDeserialize (ark-serialize 0.5, Validate::Yes)
of ProvingKey<Bn254> and VerifyingKey<Bn254> (ark-groth16 0.5), compressed or not.

    serialize_proving_key(pk)        <- pk.serialize_compressed(&mut w) / serialize_uncompressed
    deserialize_proving_key(src)     <- ProvingKey::<Bn254>::deserialize_compressed(&mut r) / deserialize_uncompressed
    serialize_verifying_key(vk)      <- vk.serialize_compressed(&mut w) / serialize_uncompressed
    deserialize_verifying_key(src)   <- VerifyingKey::<Bn254>::deserialize_compressed(&mut r) / deserialize_uncompressed
    deserialize_verifying_keys(srcs) <- the same for many keys, decoded in one device pass

The layout (the arkworks sources are not vendored here; DESIGN.md section 7 restates it):
  - fields in declaration order.  VerifyingKey: alpha_g1, beta_g2, gamma_g2, delta_g2, gamma_abc_g1 (Vec).  ProvingKey: vk,
    beta_g1, delta_g1, a_query, b_g1_query, b_g2_query (Vec<G2>), h_query, l_query - h_query BEFORE l_query.
  - a Vec is a u64 little-endian length, then its elements.
  - points as b2g_points_serialize / b2g_points_deserialize write and read them (include/b2groth.h): every point is encoded
    and decoded on the device, all G1 points of a call in one device call and all G2 points in one more; this module parses
    lengths and offsets only.
Every refusal raises r1cs.SerializationError naming the field and the index, e.g. "b_g2_query[17]"."""
from __future__ import annotations

import ctypes as C
import re
import struct

import numpy as np

from . import _native as N
from .r1cs import SerializationError
from .zkey import ProvingKey

# (field, is a Vec, is a G2 point) in serialization order
_VK_FIELDS = (('alpha_g1', False, False), ('beta_g2', False, True), ('gamma_g2', False, True), ('delta_g2', False, True),
              ('gamma_abc_g1', True, False))
_PK_FIELDS = _VK_FIELDS + (('beta_g1', False, False), ('delta_g1', False, False), ('a_query', True, False),
                           ('b_g1_query', True, False), ('b_g2_query', True, True), ('h_query', True, False),
                           ('l_query', True, False))
_READ_CHUNK = 1 << 26


def _point_bytes(g2: bool, compress: bool) -> int:
    return (64 if g2 else 32) * (1 if compress else 2)


def _ctx(ctx):
    from .groth16 import default_context
    return ctx or default_context()


def _ptr(a):
    return C.c_void_p(a.ctypes.data)


class _Source:
    """bytes (read in place; bytes after the key are ignored) or a binary reader (read exactly as far as the key goes)"""

    def __init__(self, src):
        if isinstance(src, (bytes, bytearray, memoryview)):
            self.buf, self.pos, self.reader = memoryview(src).cast('B'), 0, None
        elif hasattr(src, 'read'):
            self.reader = src
        else:
            raise TypeError("expected bytes or a binary reader")

    def take(self, n: int, what: str) -> bytes:
        if self.reader is None:
            left = len(self.buf) - self.pos
            if n > left:
                raise SerializationError(f"{what}: needs {n} bytes, {left} remain")
            out = self.buf[self.pos:self.pos + n]
            self.pos += n
            return out
        chunks, got = [], 0
        while got < n:                                     # in chunks: a huge length prefix never allocates its size
            c = self.reader.read(min(n - got, _READ_CHUNK))
            if not c:
                raise SerializationError(f"{what}: needs {n} bytes, {got} remain")
            chunks.append(c)
            got += len(c)
        return b''.join(chunks)


def _parse(src: _Source, fields, compress: bool, at: str) -> dict:
    """{field: (its point bytes, its point count)}; the lengths and truncation are checked here"""
    out = {}
    for name, vec, g2 in fields:
        size = _point_bytes(g2, compress)
        count = struct.unpack('<Q', src.take(8, f"{at}{name}: length"))[0] if vec else 1
        out[name] = (src.take(count * size, f"{at}{name}: {count} points" if vec else f"{at}{name}"), count)
    return out


def _decode(ctx, parsed: list, fields, compress: bool, ats: list) -> list:
    """one b2g_points_deserialize call for every G1 point of every key in `parsed`, one for every G2 point: per key {field:
    (count, 8 | 16) Montgomery words}.  The refused point that comes first in the serialized order raises."""
    lib, ctx = N.lib(), _ctx(ctx)
    out = [{} for _ in parsed]
    bad = []                                               # (key, field position, index, message) of each call's lowest bad point
    for g2 in (False, True):
        segs = [(k, pos, name, vec) for k, keyp in enumerate(parsed) for pos, (name, vec, g) in enumerate(fields) if g == g2]
        counts = [parsed[k][name][1] for k, _, name, _ in segs]
        n = sum(counts)
        words = 16 if g2 else 8
        pts = np.zeros((n, words), dtype='<u8')
        if n:
            raw = np.frombuffer(b''.join(parsed[k][name][0] for k, _, name, _ in segs), dtype=np.uint8)
            first = C.c_uint64()
            N.check(lib.b2g_points_deserialize(ctx._h, int(g2), int(compress), n, _ptr(raw), _ptr(pts), C.byref(first)))
            if first.value < n:
                j = first.value
                for (k, pos, name, vec), c in zip(segs, counts):
                    if j < c:
                        kind = ('compressed ' if compress else 'uncompressed ') + ('G2' if g2 else 'G1')
                        bad.append((k, pos, j, f"{ats[k]}{name}[{j}]" if vec else f"{ats[k]}{name}",
                                    f"not a valid {kind} point (Validate::Yes)"))
                        break
                    j -= c
        o = 0
        for (k, _, name, _), c in zip(segs, counts):
            out[k][name] = pts[o:o + c]
            o += c
    if bad:
        _, _, _, where, why = min(bad)
        raise SerializationError(f"{where}: {why}")
    return out


_POINT_AT = re.compile(r'.*: point (\d+) has a coordinate >= p')


def _encode(ctx, arrays: list, compress: bool) -> bytes:
    """arrays = [(field, is a Vec, is G2, Montgomery words)] in serialization order -> the serialized fields, every G1 point
    encoded in one b2g_points_serialize call and every G2 point in one more"""
    lib, ctx = N.lib(), _ctx(ctx)
    enc = {}
    for g2 in (False, True):
        words = 16 if g2 else 8
        segs = [(name, vec, np.ascontiguousarray(a, dtype='<u8').reshape(-1, words)) for name, vec, g, a in arrays if g == g2]
        n = sum(len(a) for _, _, a in segs)
        if not n:
            continue
        pts = np.ascontiguousarray(np.concatenate([a for _, _, a in segs]))
        size = _point_bytes(g2, compress)
        out = np.zeros(n * size, dtype=np.uint8)
        try:
            N.check(lib.b2g_points_serialize(ctx._h, int(g2), int(compress), n, _ptr(pts), _ptr(out)))
        except N.B2gError as e:
            m = _POINT_AT.fullmatch(e.msg)
            if e.code != N.B2G_E_INPUT or not m:
                raise
            j = int(m.group(1))
            for name, vec, a in segs:
                if j < len(a):
                    raise SerializationError(f"{name}[{j}]: a coordinate is >= p" if vec else f"{name}: a coordinate is >= p") from e
                j -= len(a)
            raise
        raw, o = out.tobytes(), 0
        for name, vec, a in segs:
            enc[name] = raw[o:o + len(a) * size]
            o += len(a) * size
    parts = []
    for name, vec, g2, a in arrays:
        if vec:
            parts.append(struct.pack('<Q', len(enc.get(name, b'')) // _point_bytes(g2, compress)))
        parts.append(enc.get(name, b''))
    return b''.join(parts)


# ---------------------------------------------------------------------------------------------- verifying keys
def _vk_arrays(vk) -> list:
    from .groth16 import _vk_desc
    _, keep = _vk_desc(vk)
    return [(name, vec, g2, keep[name]) for name, vec, g2 in _VK_FIELDS]


def _check_vk_lengths(parsed: dict, at: str) -> None:
    if parsed['gamma_abc_g1'][1] == 0:
        raise SerializationError(f"{at}gamma_abc_g1: empty (a key has at least the constant term's point)")


def _verifying_key(pts: dict):
    from .verifier import VerifyingKey, _g1_from_words, _g2_from_words
    return VerifyingKey(_g1_from_words(pts['alpha_g1'][0]), _g2_from_words(pts['beta_g2'][0]), _g2_from_words(pts['gamma_g2'][0]),
                        _g2_from_words(pts['delta_g2'][0]), [_g1_from_words(p) for p in pts['gamma_abc_g1']])


def serialize_verifying_key(vk, compress: bool = True, ctx=None) -> bytes:
    """VerifyingKey::<Bn254>::serialize_compressed (compress) or serialize_uncompressed.  `vk` is a verifier.VerifyingKey, a
    PreparedVerifyingKey or a ProvingKey (its vk part)."""
    return _encode(ctx, _vk_arrays(vk), compress)


def deserialize_verifying_keys(blobs, compress: bool = True, ctx=None) -> list:
    """VerifyingKey::<Bn254>::deserialize_compressed (compress) or deserialize_uncompressed, Validate::Yes, for many keys:
    every G1 point of every key is decoded in one device call and every G2 point in one more, whatever the number of keys.
    Each blob is bytes or a binary reader, as for deserialize_verifying_key.  A refusal names the key: "key 3: beta_g2: ..."."""
    srcs = [_Source(b) for b in blobs]
    ats = [f"key {k}: " for k in range(len(srcs))]
    parsed = []
    for src, at in zip(srcs, ats):
        parsed.append(_parse(src, _VK_FIELDS, compress, at))
        _check_vk_lengths(parsed[-1], at)
    if not parsed:
        return []
    return [_verifying_key(p) for p in _decode(ctx, parsed, _VK_FIELDS, compress, ats)]


def deserialize_verifying_key(src, compress: bool = True, ctx=None):
    """VerifyingKey::<Bn254>::deserialize_compressed (compress) or deserialize_uncompressed, Validate::Yes -> a
    verifier.VerifyingKey.  src = bytes (bytes after the key are ignored) or a binary reader (left just past the key).
    gamma_abc_g1 must hold at least one point."""
    parsed = _parse(_Source(src), _VK_FIELDS, compress, '')
    _check_vk_lengths(parsed, '')
    return _verifying_key(_decode(ctx, [parsed], _VK_FIELDS, compress, [''])[0])


# ---------------------------------------------------------------------------------------------- proving keys
def serialize_proving_key(pk: ProvingKey, compress: bool = True, ctx=None) -> bytes:
    """ProvingKey::<Bn254>::serialize_compressed (compress) or serialize_uncompressed of a ProvingKey (read_zkey, the GPU
    setup or deserialize_proving_key): vk, beta_g1, delta_g1, a_query, b_g1_query, b_g2_query, h_query, l_query."""
    arrays = [(name, vec, g2, getattr(pk, name)) for name, vec, g2 in _PK_FIELDS]
    return _encode(ctx, arrays, compress)


def deserialize_proving_key(src, compress: bool = True, ctx=None) -> ProvingKey:
    """ProvingKey::<Bn254>::deserialize_compressed (compress) or deserialize_uncompressed, Validate::Yes -> a ProvingKey with
    n_vars = len(a_query), n_public = len(gamma_abc_g1) - 1 and domain_size = len(h_query).  src = bytes (bytes after the key
    are ignored) or a binary reader (left just past the key).

    A key carries no reduction: it proves under the reduction the caller passes, which checks the H query's length.  Keys
    whose vector lengths disagree (b_g1_query or b_g2_query not of n_vars points, l_query not of n_vars - n_public - 1
    points, an empty gamma_abc_g1) are refused although arkworks reads them: no proof can be made with such a key, and
    b2g_pk_desc cannot describe it."""
    parsed = _parse(_Source(src), _PK_FIELDS, compress, '')
    _check_vk_lengths(parsed, '')
    n_vars, n_public = parsed['a_query'][1], parsed['gamma_abc_g1'][1] - 1
    if n_public + 1 > n_vars:
        raise SerializationError(f"gamma_abc_g1: {n_public + 1} points, more than a_query's {n_vars}")
    for name, want in (('b_g1_query', n_vars), ('b_g2_query', n_vars), ('l_query', n_vars - n_public - 1)):
        if parsed[name][1] != want:
            raise SerializationError(f"{name}: {parsed[name][1]} points, the key's a_query and gamma_abc_g1 need {want}")
    p = _decode(ctx, [parsed], _PK_FIELDS, compress, [''])[0]
    return ProvingKey(n_vars, n_public, parsed['h_query'][1], p['alpha_g1'], p['beta_g1'], p['beta_g2'], p['gamma_g2'], p['delta_g1'],
                      p['delta_g2'], p['gamma_abc_g1'], p['a_query'], p['b_g1_query'], p['b_g2_query'], p['l_query'], p['h_query'])
