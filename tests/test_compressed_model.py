"""The strict decoder of arkworks' compressed proofs (tests/compressed_model.py) against the encoder the product ships
(ethereum.serialize_compressed) and against the unchecked oracle decoder: round trips on golden proofs, points at infinity and
both signs, and a refusal for every malformed kind.  Also the C++ encoder (ark_circom::serialize_compressed) against the
Python one.  CPU only."""
import json
import os
import random
import subprocess

import pytest

from batch_model import twist_point_outside_g2
from compressed_model import (P, decompress_proof_checked, g1_decompress, g1_no_root_x, g2_bytes, g2_decompress, g2_no_root_x,
                              proof_row, twist_point_real_y, Undecodable)
from circom_compat_b200 import Proof
from circom_compat_b200 import ethereum as eth
from oracle import pyref as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = o.R_MOD


def _golden():
    return json.load(open(os.path.join(ROOT, 'tests', 'golden', 'golden_vectors.json')))


def _compress(a, b, c) -> bytes:
    return eth.serialize_compressed(eth.Proof.from_proof(Proof(proof_row(a, b, c))))


def _points(seed):
    rng = random.Random(seed)
    return o.G1.mul(o.G1_GEN, rng.randrange(1, R)), o.G2.mul(o.G2_GEN, rng.randrange(1, R)), o.G1.mul(o.G1_GEN, rng.randrange(1, R))


def test_golden_proofs_round_trip():
    for case in _golden()['test_zkey']['proofs']:
        p = Proof(bytes.fromhex(case['proof_hex']))
        blob = eth.serialize_compressed(eth.Proof.from_proof(p))
        assert len(blob) == 128
        got = decompress_proof_checked(blob)
        assert got == (p.a, p.b, p.c)
        assert got == o.decompress_proof(blob)
        assert proof_row(*got) == p.data


def test_infinity_points_round_trip():
    a, b, c = _points(1)
    for pts in ((None, b, c), (a, None, c), (a, b, None), (None, None, None)):
        blob = _compress(*pts)
        assert decompress_proof_checked(blob) == pts
    assert _compress(None, None, None) == bytes(31) + b'\x40' + bytes(63) + b'\x40' + bytes(31) + b'\x40'


def test_both_signs_round_trip():
    for seed in range(4):
        a, b, c = _points(10 + seed)
        for pts in ((a, b, c), (o.G1.neg(a), o.G2.neg(b), o.G1.neg(c))):
            assert decompress_proof_checked(_compress(*pts)) == pts
        flags = [_compress(a, b, c)[k] & 0x80 for k in (31, 95, 127)]
        neg = [_compress(o.G1.neg(a), o.G2.neg(b), o.G1.neg(c))[k] & 0x80 for k in (31, 95, 127)]
        assert [f ^ g for f, g in zip(flags, neg)] == [0x80] * 3


def test_twist_point_with_real_y():
    x, y = twist_point_real_y()
    small, big = sorted((y[0], P - y[0]))
    assert g2_decompress(g2_bytes(x), subgroup=False) == (x, (small, 0))
    assert g2_decompress(g2_bytes(x, 0x80), subgroup=False) == (x, (big, 0))


def _refused(blob):
    return decompress_proof_checked(blob) is None


def test_malformed_proofs_are_refused():
    a, b, c = _points(2)
    good = bytearray(_compress(a, b, c))
    assert not _refused(bytes(good))
    for k in (31, 95, 127):                                         # both flag bits on A, B, C
        bad = bytearray(good)
        bad[k] |= 0xC0
        assert _refused(bytes(bad)), k
    for off in (0, 96):                                             # x = p and x = 2^254 - 1 on A and C
        for v in (P, (1 << 254) - 1):
            bad = bytearray(good)
            bad[off:off + 32] = v.to_bytes(32, 'little')
            assert _refused(bytes(bad)), (off, v)
            bad[off + 31] |= 0x40                                   # out of range even under the infinity flag
            assert _refused(bytes(bad)), (off, v)
    for off in (32, 64):                                            # x.c0 >= p, x.c1 >= p on B
        bad = bytearray(good)
        bad[off:off + 32] = P.to_bytes(32, 'little')
        assert _refused(bytes(bad)), off
    x = g1_no_root_x()
    with pytest.raises(Undecodable):
        g1_decompress(x.to_bytes(32, 'little'))
    for off in (0, 96):
        bad = bytearray(good)
        bad[off:off + 32] = x.to_bytes(32, 'little')
        assert _refused(bytes(bad)), off
    bad = bytearray(good)
    bad[32:96] = g2_bytes(g2_no_root_x())
    assert _refused(bytes(bad))
    q = twist_point_outside_g2(random.Random(3))
    bad = bytearray(good)
    bad[32:96] = _compress(None, q, None)[32:96]
    assert g2_decompress(bytes(bad[32:96]), subgroup=False) == q
    assert _refused(bytes(bad))
    assert _refused(bytes(good[:127])) and _refused(bytes(good) + b'\x00')


def test_infinity_flag_ignores_x_below_p():
    a, b, c = _points(4)
    blob = bytearray(_compress(a, b, c))
    blob[31] = (blob[31] & 0x3F) | 0x40
    blob[95] = (blob[95] & 0x3F) | 0x40
    assert decompress_proof_checked(bytes(blob)) == (None, None, c)


def test_cpp_and_python_compressed_bytes_agree():
    """ark_circom::serialize_compressed (host/ark_circom_ethereum.hpp, printed by groth16_bench --ethereum) against
    ethereum.serialize_compressed on the golden test.zkey proofs"""
    exe = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench')
    zk = os.path.join(ROOT, 'tests', 'golden', 'test.zkey')
    for case in _golden()['test_zkey']['proofs']:
        out = subprocess.check_output([exe, '--ethereum', zk, case['proof_hex'], '33'], text=True)
        kv = dict(line.split('=', 1) for line in out.split())
        want = eth.serialize_compressed(eth.Proof.from_proof(Proof(bytes.fromhex(case['proof_hex']))))
        assert kv['compressed'] == want.hex()
