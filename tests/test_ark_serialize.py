"""Arkworks-serialized Groth16 keys on the device (b2g_points_serialize / b2g_points_deserialize, ark_serialize.py): the
point bytes equal the big-int model's (tests/ark_key_model.py), keys round-trip bit for bit, proofs under a deserialized key
equal proofs under the original, every refusal names its field and index, and many verifying keys decode in two calls."""
import io
import os
import random
import struct

import numpy as np
import pytest

import ark_key_model as M
from compressed_model import FLAG_INF, P, g1_no_root_x, g2_bytes, g2_no_root_x, twist_point_real_y
from circom_compat_b200 import (Groth16, LibsnarkReduction, Proof, R1CS, R1CSFile, deserialize_proving_key,
                                deserialize_verifying_key, deserialize_verifying_keys, fr_to_mont, read_wtns, read_zkey,
                                release, serialize_proving_key, serialize_verifying_key, synth)
from circom_compat_b200 import _native as N
from circom_compat_b200 import verifier as V
from circom_compat_b200.groth16 import _mont_points
from circom_compat_b200.r1cs import SerializationError
from oracle import pyref as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
R = o.R_MOD
ARRAYS = ('alpha_g1', 'beta_g1', 'beta_g2', 'gamma_g2', 'delta_g1', 'delta_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query',
          'b_g2_query', 'l_query', 'h_query')
pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def synth_pk(ctx):
    """a 2^16 synthetic key (setup on the GPU), about 2^18 G1 and 2^16 G2 points"""
    pk, _ = synth.setup(ctx, synth.chain_circuit(1 << 16))
    return pk


def _serialize_raw(ctx, pts, g2, compress):
    pts = np.ascontiguousarray(pts, dtype='<u8')
    n = pts.size // (16 if g2 else 8)
    out = np.zeros(n * M.point_size(g2, compress), dtype=np.uint8)
    N.check(N.lib().b2g_points_serialize(ctx._h, int(g2), int(compress), n, pts.ctypes.data, out.ctypes.data))
    return out.tobytes()


def _canon(rows, g2):
    return [V._g2_from_words(r) if g2 else V._g1_from_words(r) for r in rows]


@pytest.mark.parametrize('compress', [True, False])
def test_point_bytes_equal_the_model(ctx, test_zkey_bytes, compress):
    """every point of test.zkey and of a 2^11 synthetic key, plus infinity, negated points (y both smaller and larger than
    -y) and the y.c1 = 0 tie, serialized on the device, byte for byte the model's"""
    pk, _ = read_zkey(test_zkey_bytes)
    spk, _ = synth.setup(ctx, synth.chain_circuit(1 << 11))
    g1 = np.concatenate([k.reshape(-1, 8) for key in (pk, spk) for k in
                         (key.alpha_g1, key.beta_g1, key.delta_g1, key.gamma_abc_g1, key.a_query, key.b_g1_query, key.h_query, key.l_query)])
    g2 = np.concatenate([k.reshape(-1, 16) for key in (pk, spk) for k in (key.beta_g2, key.gamma_g2, key.delta_g2, key.b_g2_query)])
    p1, p2 = _canon(g1, False), _canon(g2, True)
    p1 += [None] + [(p[0], (P - p[1]) % P) for p in p1[:64] if p is not None]
    p2 += [None, twist_point_real_y()] + [(q[0], o.FQ2.neg(q[1])) for q in p2[:64] if q is not None]
    assert len(p1) + len(p2) >= 1 << 12 and None in _canon(pk.b_g2_query.reshape(-1, 16), True)
    for pts, g2 in ((p1, False), (p2, True)):
        raw = _serialize_raw(ctx, _mont_points(pts, g2), g2, compress)
        size = M.point_size(g2, compress)
        flags = set()
        for i, p in enumerate(pts):
            assert raw[i * size:(i + 1) * size] == M.point_bytes(p, g2, compress), (g2, i)
            flags.add(raw[(i + 1) * size - 1] & 0xC0)
        assert flags == {0x00, 0x40, 0x80}


def test_serialize_refuses_a_coordinate_not_below_p(ctx):
    pts = _mont_points([(1, 2)] * 5, False).reshape(5, 8)
    pts[3, 4:8] = np.frombuffer(P.to_bytes(32, 'little'), dtype='<u8')
    with pytest.raises(N.B2gError, match='point 3 has a coordinate >= p') as e:
        _serialize_raw(ctx, pts, False, True)
    assert e.value.code == N.B2G_E_INPUT


def _same_key(a, b):
    assert (a.n_vars, a.n_public, a.domain_size) == (b.n_vars, b.n_public, b.domain_size)
    for name in ARRAYS:
        x, y = np.ascontiguousarray(getattr(a, name), dtype='<u8'), getattr(b, name)
        assert x.shape == y.shape and x.tobytes() == y.tobytes(), name


@pytest.mark.parametrize('compress', [True, False])
@pytest.mark.parametrize('which', ['test_zkey', 'bench_zkey', 'synth_2_16'])
def test_proving_key_round_trips_bit_for_bit(ctx, request, test_zkey_bytes, complex_zkey_bytes, which, compress):
    """deserialize(serialize(pk)) reproduces every array; from bytes with a tail and from a reader left just past the key"""
    pk = {'test_zkey': lambda: read_zkey(test_zkey_bytes)[0], 'bench_zkey': lambda: read_zkey(complex_zkey_bytes)[0],
          'synth_2_16': lambda: request.getfixturevalue('synth_pk')}[which]()
    data = serialize_proving_key(pk, compress, ctx)
    if which == 'test_zkey':
        assert data == M.serialize(M.key_from_pk(pk), M.PK_FIELDS, compress)
    _same_key(deserialize_proving_key(data + b'tail', compress, ctx), pk)
    f = io.BytesIO(data + b'tail')
    _same_key(deserialize_proving_key(f, compress, ctx), pk)
    assert f.tell() == len(data)
    vk_data = serialize_verifying_key(pk, compress, ctx)
    assert data.startswith(vk_data)
    assert deserialize_verifying_key(vk_data, compress, ctx) == V.VerifyingKey.from_proving_key(pk)


@pytest.mark.parametrize('compress', [True, False])
def test_proof_under_deserialized_zkey_is_identical(ctx, golden, test_zkey_bytes, compress):
    """CircomReduction: test.zkey's key through both forms proves the golden proof bytes"""
    pk, cm = read_zkey(test_zkey_bytes)
    pk2 = deserialize_proving_key(serialize_proving_key(pk, compress, ctx), compress, ctx)
    g = golden['test_zkey']
    wm = fr_to_mont([int(x) for x in g['witness']])
    case = g['proofs'][0]
    for key in (pk, pk2):
        p = Groth16.create_proof_with_reduction_and_matrices(key, int(case['r']), int(case['s']), cm, cm.num_instance_variables,
                                                             cm.num_constraints, wm, ctx)
        assert p.data.hex() == case['proof_hex']
    release(pk2)


@pytest.mark.parametrize('compress', [True, False])
def test_libsnark_setup_serialize_deserialize_prove(ctx, compress):
    """the tests/groth16.rs flow on circuit2: GPU setup, serialize, deserialize, prove; same proof as under the original key"""
    r1cs = R1CS.from_file(R1CSFile.new(open(os.path.join(GOLDEN, 'circuit2.r1cs'), 'rb').read()))
    w = read_wtns(open(os.path.join(GOLDEN, 'circuit2_witness.wtns'), 'rb').read())
    circ = r1cs.to_circuit()
    cm = circ.matrices(with_c=True)
    pk = Groth16.generate_random_parameters_with_reduction(circ, random.Random(7), ctx, LibsnarkReduction)
    pk2 = deserialize_proving_key(serialize_proving_key(pk, compress, ctx), compress, ctx)
    _same_key(pk2, pk)
    wm = fr_to_mont(w)
    r, s = 0x1234567, 0x7654321
    proofs = [Groth16.create_proof_with_reduction_and_matrices(key, r, s, cm, circ.num_inputs, circ.num_constraints, wm, ctx,
                                                               LibsnarkReduction) for key in (pk, pk2)]
    assert proofs[0].data == proofs[1].data
    assert Groth16.verify_many(pk2, [w[1:r1cs.num_inputs]], [proofs[1]], ctx) == [True]
    release(pk); release(pk2); release(cm)


# ---------------------------------------------------------------------------------------------- refusals
def _offset(pk, name, i, compress):
    """byte offset of point i of field `name` in serialize_proving_key(pk)"""
    pos = 0
    for f, vec, g2 in M.PK_FIELDS:
        size = M.point_size(g2, compress)
        if vec:
            pos += 8
        if f == name:
            return pos + i * size
        pos += size * (len(getattr(pk, f).reshape(-1, 16 if g2 else 8)) if vec else 1)
    raise KeyError(name)


def _put(data, pos, raw):
    return data[:pos] + raw + data[pos + len(raw):]


def _refused(ctx, data, compress, where):
    with pytest.raises(SerializationError) as e:
        deserialize_proving_key(data, compress, ctx)
    assert str(e.value).startswith(where + ':'), str(e.value)


@pytest.fixture(scope='module')
def zkey_pk(complex_zkey_bytes):
    """the bench key (10 000 wires): room for a bad point at any index the tests name"""
    return read_zkey(complex_zkey_bytes)[0]


def test_refusals_compressed(ctx, zkey_pk):
    pk, z = zkey_pk, True
    data = serialize_proving_key(pk, z, ctx)
    x, y = twist_point_real_y()
    outside = M.point_bytes((x, y), True, z)
    _refused(ctx, _put(data, _offset(pk, 'b_g2_query', 17, z), outside), z, 'b_g2_query[17]')
    inf_p = bytearray(P.to_bytes(32, 'little')); inf_p[-1] |= FLAG_INF
    _refused(ctx, _put(data, _offset(pk, 'h_query', 2, z), bytes(inf_p)), z, 'h_query[2]')
    both = bytearray(data[_offset(pk, 'l_query', 1, z):_offset(pk, 'l_query', 1, z) + 32]); both[-1] |= 0xC0
    _refused(ctx, _put(data, _offset(pk, 'l_query', 1, z), bytes(both)), z, 'l_query[1]')
    _refused(ctx, _put(data, _offset(pk, 'b_g1_query', 4, z), g1_no_root_x().to_bytes(32, 'little')), z, 'b_g1_query[4]')
    _refused(ctx, _put(data, _offset(pk, 'delta_g2', 0, z), g2_bytes(g2_no_root_x())), z, 'delta_g2')
    _refused(ctx, data[:-1], z, 'l_query')
    n_h = len(pk.h_query)
    at = _offset(pk, 'h_query', 0, z) - 8
    assert struct.unpack_from('<Q', data, at)[0] == n_h
    _refused(ctx, _put(data, at, struct.pack('<Q', 1 << 40)), z, 'h_query')
    _refused(ctx, io.BytesIO(_put(data, at, struct.pack('<Q', n_h + 10 ** 6))), z, 'h_query')
    # the lowest bad point wins: two in a_query; a G1 point before a G2 point; a vk G2 point before a G1 Vec
    bad = bytes(32 * [0xFF])
    two = _put(_put(data, _offset(pk, 'a_query', 5, z), bad), _offset(pk, 'a_query', 2, z), bad)
    _refused(ctx, two, z, 'a_query[2]')
    _refused(ctx, _put(_put(data, _offset(pk, 'b_g2_query', 0, z), outside), _offset(pk, 'a_query', 1, z), bad), z, 'a_query[1]')
    _refused(ctx, _put(_put(data, _offset(pk, 'beta_g2', 0, z), outside), _offset(pk, 'a_query', 1, z), bad), z, 'beta_g2')
    # the context stays usable
    _same_key(deserialize_proving_key(data, z, ctx), pk)


def test_refusals_uncompressed(ctx, zkey_pk):
    pk, z = zkey_pk, False
    data = serialize_proving_key(pk, z, ctx)
    i = next(i for i in range(3, len(pk.a_query)) if pk.a_query[i].any())
    at = _offset(pk, 'a_query', i, z)
    x, y = (int.from_bytes(data[at + 32 * k:at + 32 * k + 32], 'little') & ((1 << 254) - 1) for k in (0, 1))
    _refused(ctx, _put(data, at, M._le([x, (y + 1) % P])), z, f'a_query[{i}]')
    q = twist_point_real_y()
    _refused(ctx, _put(data, _offset(pk, 'b_g2_query', 6, z), M.point_bytes(q, True, z)), z, 'b_g2_query[6]')
    inf_p = bytearray(P.to_bytes(32, 'little') + bytes(32)); inf_p[-1] |= FLAG_INF
    _refused(ctx, _put(data, _offset(pk, 'gamma_abc_g1', 1, z), bytes(inf_p)), z, 'gamma_abc_g1[1]')
    _refused(ctx, _put(data, _offset(pk, 'alpha_g1', 0, z), bytes(64)), z, 'alpha_g1')
    _refused(ctx, data[:100], z, 'beta_g2')
    # bit 7 is ignored on read; the infinity flag over coordinates below p decodes as infinity
    flipped = bytearray(data); flipped[at + 63] ^= 0x80
    inf_any = bytearray(M._le([1, 2])); inf_any[-1] |= FLAG_INF
    pk2 = deserialize_proving_key(_put(bytes(flipped), _offset(pk, 'h_query', 0, z), bytes(inf_any)), z, ctx)
    assert pk2.a_query.tobytes() == np.ascontiguousarray(pk.a_query).tobytes() and not pk2.h_query[0].any()


@pytest.mark.parametrize('compress', [True, False])
def test_inconsistent_lengths_are_refused(ctx, test_zkey_bytes, compress):
    key = M.key_from_pk(read_zkey(test_zkey_bytes)[0])
    for name in ('b_g1_query', 'b_g2_query', 'l_query'):
        bad = dict(key, **{name: key[name][:-1]})
        _refused(ctx, M.serialize(bad, M.PK_FIELDS, compress), compress, name)


# ---------------------------------------------------------------------------------------------- many verifying keys
def _synthetic_keys(ctx, n):
    """n keys with 0, 1 or 2 public inputs and one valid proof each, every point from the device's fixed-base products"""
    rng = random.Random(0xA4C)
    specs, s1, s2 = [], [], []
    for k in range(n):
        al, be, ga, de = (rng.randrange(1, R) for _ in range(4))
        ic = [rng.randrange(1, R) for _ in range(k % 3 + 1)]
        xs = [rng.randrange(R) for _ in range(k % 3)]
        prep = (ic[0] + sum(x * c for x, c in zip(xs, ic[1:]))) % R
        a, b = rng.randrange(1, R), rng.randrange(1, R)
        c = (a * b - al * be - prep * ga) * pow(de, -1, R) % R
        specs.append((len(s1), len(ic), len(s2), xs))
        s1 += [al] + ic + [a, c]
        s2 += [be, ga, de, b]
    g1 = _canon(ctx.fixed_base_g1(synth._ints_to_limbs(s1)), False)
    g2 = _canon(ctx.fixed_base_g2(synth._ints_to_limbs(s2)), True)
    out = []
    for o1, n_ic, o2, xs in specs:
        vk = V.VerifyingKey(g1[o1], g2[o2], g2[o2 + 1], g2[o2 + 2], g1[o1 + 1:o1 + 1 + n_ic])
        a, c = g1[o1 + 1 + n_ic], g1[o1 + 2 + n_ic]
        vals = list(a) + [g2[o2 + 3][0][0], g2[o2 + 3][0][1], g2[o2 + 3][1][0], g2[o2 + 3][1][1]] + list(c)
        out.append((vk, xs, Proof(b''.join(int(v).to_bytes(32, 'little') for v in vals))))
    return out


@pytest.mark.parametrize('compress', [True, False])
def test_many_verifying_keys_in_two_device_calls(ctx, monkeypatch, compress):
    keys = _synthetic_keys(ctx, 256)
    blobs = [M.serialize({'alpha_g1': vk.alpha_g1, 'beta_g2': vk.beta_g2, 'gamma_g2': vk.gamma_g2, 'delta_g2': vk.delta_g2,
                          'gamma_abc_g1': vk.gamma_abc_g1}, M.VK_FIELDS, compress) for vk, _, _ in keys]
    assert blobs[5] == serialize_verifying_key(keys[5][0], compress, ctx)
    lib, calls = N.lib(), []
    real = lib.b2g_points_deserialize

    def counted(*args):
        calls.append(args[1])
        return real(*args)
    monkeypatch.setattr(lib, 'b2g_points_deserialize', counted)
    many = deserialize_verifying_keys([b if k % 2 else io.BytesIO(b) for k, b in enumerate(blobs)], compress, ctx)
    assert sorted(calls) == [0, 1]
    monkeypatch.undo()
    assert many == [vk for vk, _, _ in keys]
    assert many == [deserialize_verifying_key(b, compress, ctx) for b in blobs]
    assert Groth16.verify_batch_keys([(vk, [xs], [p]) for vk, (_, xs, p) in zip(many, keys)], ctx) == [True] * 256
    bad = bytearray(blobs[200]); bad[-1] |= 0xC0
    with pytest.raises(SerializationError, match=r'^key 200: gamma_abc_g1\[\d+\]:'):
        deserialize_verifying_keys(blobs[:200] + [bytes(bad)] + blobs[201:], compress, ctx)


# ---------------------------------------------------------------------------------------------- the C++ mirror
def _fnv(data: bytes) -> int:
    h = 1469598103934665603
    for b in data:
        h = ((h ^ b) * 1099511628211) & ((1 << 64) - 1)
    return h


def test_cpp_mirror_writes_the_same_bytes(ctx, golden, complex_zkey_bytes, tmp_path):
    """groth16_bench's B2G_ARK_KEYS mode on the bench key: both forms read back identical, and their bytes are the Python
    side's, byte for byte (size and FNV-1a digest, and the written files themselves)"""
    import subprocess
    exe = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench')
    base = str(tmp_path / 'bench_key')
    out = subprocess.check_output([exe, os.path.join(GOLDEN, 'complex-circuit-10000-10000.zkey'),
                                   'chain:%d' % int(golden['complex_zkey']['a']), '0'], text=True, env=dict(os.environ, B2G_ARK_KEYS=base))
    pk, _ = read_zkey(complex_zkey_bytes)
    for compress, name in ((True, 'compressed'), (False, 'uncompressed')):
        data = serialize_proving_key(pk, compress, ctx)
        line = [l for l in out.splitlines() if l.startswith(f'ark_keys {name} ')][0]
        assert f'bytes={len(data)} fnv={_fnv(data):016x} identical=1' in line, line
        assert open(f'{base}.{name}', 'rb').read() == data
