"""The big-int model of arkworks-serialized Groth16 keys (tests/ark_key_model.py): it round-trips test.zkey's keys in both
forms, its point bytes equal the proof encoder's (ethereum._g1_bytes / _g2_bytes), and it refuses one constructed instance of
every rule of the format.  CPU only."""
import struct

import pytest

import ark_key_model as M
from compressed_model import FLAG_INF, FLAG_NEG, P, g1_no_root_x, g2_bytes, g2_no_root_x, twist_point_real_y
from circom_compat_b200 import ethereum as E
from circom_compat_b200 import read_zkey
from oracle import pyref as o


@pytest.fixture(scope='module')
def zkey_key(test_zkey_bytes):
    pk, _ = read_zkey(test_zkey_bytes)
    return M.key_from_pk(pk)


def _vk(key):
    return {name: key[name] for name, _, _ in M.VK_FIELDS}


@pytest.mark.parametrize('compress', [True, False])
def test_model_round_trips_test_zkey(zkey_key, compress):
    """deserialize(serialize(key)) is the key for the proving key and its verifying key; bytes after a key are not read"""
    for key, fields in ((zkey_key, M.PK_FIELDS), (_vk(zkey_key), M.VK_FIELDS)):
        data = M.serialize(key, fields, compress)
        back, used = M.deserialize(data + b'\x07' * 5, fields, compress)
        assert back == key and used == len(data)
    assert any(p is None for p in zkey_key['b_g2_query']) and any(p is None for p in zkey_key['b_g1_query'])


def test_model_layout_of_test_zkey(zkey_key):
    """field order, length prefixes and sizes: h_query is written before l_query (the zkey order is the other way round)"""
    data = M.serialize(zkey_key, M.PK_FIELDS, True)
    pos = 32 + 3 * 64
    assert struct.unpack_from('<Q', data, pos)[0] == len(zkey_key['gamma_abc_g1'])
    pos += 8 + 32 * len(zkey_key['gamma_abc_g1']) + 2 * 32
    for name, size in (('a_query', 32), ('b_g1_query', 32), ('b_g2_query', 64), ('h_query', 32), ('l_query', 32)):
        assert struct.unpack_from('<Q', data, pos)[0] == len(zkey_key[name]), name
        pos += 8 + size * len(zkey_key[name])
    assert pos == len(data)
    assert len(zkey_key['h_query']) != len(zkey_key['l_query'])


@pytest.mark.parametrize('compress', [True, False])
def test_point_bytes_equal_the_proof_encoder(zkey_key, compress):
    """every point of test.zkey, infinity, both signs of y and the y.c1 = 0 tie: the model's bytes are ethereum's"""
    g1s = [zkey_key['alpha_g1'], zkey_key['beta_g1'], zkey_key['delta_g1'], None] + zkey_key['gamma_abc_g1'] + \
        zkey_key['a_query'] + zkey_key['b_g1_query'] + zkey_key['h_query'] + zkey_key['l_query']
    g1s += [(p[0], (P - p[1]) % P) for p in g1s if p is not None][:8]
    g2s = [zkey_key['beta_g2'], zkey_key['gamma_g2'], zkey_key['delta_g2'], None, twist_point_real_y()] + zkey_key['b_g2_query']
    g2s += [(q[0], o.FQ2.neg(q[1])) for q in g2s if q is not None][:8]
    signs = set()
    for p in g1s:
        b = M.point_bytes(p, False, compress)
        assert b == E._g1_bytes(E.G1.from_affine(p), compress)
        signs.add(b[-1] & 0xC0)
    for q in g2s:
        assert M.point_bytes(q, True, compress) == E._g2_bytes(E.G2.from_affine(q), compress)
    assert signs == {0, FLAG_NEG, FLAG_INF}


def _refuses(data, fields, compress, where):
    with pytest.raises(M.Refused) as e:
        M.deserialize(data, fields, compress)
    assert e.value.where == where, str(e.value)


def _vk_with(vk, compress, name, raw):
    """the serialized vk with field `name` (a single point) replaced by raw bytes"""
    out = b''
    for f, vec, g2 in M.VK_FIELDS:
        out += raw if f == name else M.serialize({f: vk[f]}, ((f, vec, g2),), compress)
    return out


@pytest.mark.parametrize('compress', [True, False])
def test_model_refuses_every_rule(zkey_key, compress):
    vk = _vk(zkey_key)
    data = M.serialize(vk, M.VK_FIELDS, compress)
    g1 = M.point_bytes(vk['alpha_g1'], False, compress)
    # both flag bits set
    bad = bytearray(g1); bad[-1] |= 0xC0
    _refuses(_vk_with(vk, compress, 'alpha_g1', bytes(bad)), M.VK_FIELDS, compress, 'alpha_g1')
    # a coordinate >= p under the infinity flag (p itself, flags masked off)
    inf = bytearray(P.to_bytes(32, 'little') * (1 if compress else 2)); inf[-1] |= FLAG_INF
    _refuses(_vk_with(vk, compress, 'alpha_g1', bytes(inf)), M.VK_FIELDS, compress, 'alpha_g1')
    # ... while the infinity flag over zero coordinates, or over any coordinates below p, decodes as infinity
    zero_inf = bytearray(32 * (1 if compress else 2)); zero_inf[0] = 5; zero_inf[-1] |= FLAG_INF
    assert M.deserialize(_vk_with(vk, compress, 'alpha_g1', bytes(zero_inf)), M.VK_FIELDS, compress)[0]['alpha_g1'] is None
    # truncated input and an oversized length prefix
    _refuses(data[:-1], M.VK_FIELDS, compress, 'gamma_abc_g1')
    _refuses(data[:10], M.VK_FIELDS, compress, 'alpha_g1')
    n = len(vk['gamma_abc_g1'])
    pos = len(data) - 8 - n * M.point_size(False, compress)
    assert struct.unpack_from('<Q', data, pos)[0] == n
    _refuses(data[:pos] + struct.pack('<Q', n + 1) + data[pos + 8:], M.VK_FIELDS, compress, 'gamma_abc_g1')
    _refuses(data[:pos] + struct.pack('<Q', 1 << 62) + data[pos + 8:], M.VK_FIELDS, compress, 'gamma_abc_g1')
    # a G2 point on the twist but outside G2, as gamma_abc_g1's neighbour beta_g2
    x, y = twist_point_real_y()
    assert M.on_curve((x, y), True)
    _refuses(_vk_with(vk, compress, 'beta_g2', M.point_bytes((x, y), True, compress)), M.VK_FIELDS, compress, 'beta_g2')
    # a bad point inside a Vec is named by its index
    ic = list(vk['gamma_abc_g1'])
    raw = bytearray(M.serialize({'gamma_abc_g1': ic}, (M.VK_FIELDS[4],), compress))
    raw[8 + M.point_size(False, compress) * 2 - 1] |= 0xC0
    _refuses(data[:pos] + bytes(raw), M.VK_FIELDS, compress, 'gamma_abc_g1[1]')


def test_model_refuses_compressed_x_without_root(zkey_key):
    vk = _vk(zkey_key)
    _refuses(_vk_with(vk, True, 'alpha_g1', g1_no_root_x().to_bytes(32, 'little')), M.VK_FIELDS, True, 'alpha_g1')
    _refuses(_vk_with(vk, True, 'delta_g2', g2_bytes(g2_no_root_x())), M.VK_FIELDS, True, 'delta_g2')


def test_model_uncompressed_rules(zkey_key):
    """off-curve points are refused (G1 and G2, and (0, 0) without the infinity flag); bit 7 is ignored on read"""
    vk = _vk(zkey_key)
    x, y = vk['alpha_g1']
    _refuses(_vk_with(vk, False, 'alpha_g1', M._le([x, (y + 1) % P])), M.VK_FIELDS, False, 'alpha_g1')
    _refuses(_vk_with(vk, False, 'alpha_g1', bytes(64)), M.VK_FIELDS, False, 'alpha_g1')
    q = vk['gamma_g2']
    _refuses(_vk_with(vk, False, 'gamma_g2', M._le([q[0][0], q[0][1], q[1][0], (q[1][1] + 1) % P])), M.VK_FIELDS, False, 'gamma_g2')
    flipped = bytearray(M.point_bytes(vk['alpha_g1'], False, False)); flipped[-1] ^= FLAG_NEG
    assert M.deserialize(_vk_with(vk, False, 'alpha_g1', bytes(flipped)), M.VK_FIELDS, False)[0] == vk
