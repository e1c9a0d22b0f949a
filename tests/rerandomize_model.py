"""Big-int model of Groth16::rerandomize_proof (ark-groth16 0.5.0, src/prover.rs), on oracle.pyref's Curve arithmetic, shared
by the CPU and GPU tests of tests/test_rerandomize.py.  TEST INFRASTRUCTURE ONLY: product code never imports it.

For a proof (A, B, C) and nonzero factors r1, r2 of Fr:
    A' = r1^-1 A,   B' = r1 B + (r1 r2) delta_2,   C' = C + r2 A
with r1^-1 and r1 r2 taken mod r.  Points are affine canonical ints, None at infinity; B is not checked for membership in G2."""
from oracle import pyref as o

R = o.R_MOD


def rerandomize_proof(delta_g2, proof, r1: int, r2: int):
    """(A', B', C') of proof = (A, B, C) under the key's delta_g2 and the factors r1, r2 in [1, r)"""
    assert 0 < r1 < R and 0 < r2 < R
    a, b, c = proof
    a2 = o.G1.mul(a, pow(r1, -1, R))
    b2 = o.G2.add(o.G2.mul(b, r1), o.G2.mul(delta_g2, r1 * r2 % R))
    c2 = o.G1.add(c, o.G1.mul(a, r2))
    return a2, b2, c2


def proof_bytes(proof) -> bytes:
    """the 256-byte canonical row of b2g_prove (zeros at infinity)"""
    return o.proof_to_bytes(*proof)


def proof_points(data: bytes):
    """a 256-byte row -> (A, B, C), None for an all-zero point"""
    v = [int.from_bytes(data[32 * i:32 * i + 32], 'little') for i in range(8)]
    a = None if v[0] == v[1] == 0 else (v[0], v[1])
    b = None if not any(v[2:6]) else ((v[2], v[3]), (v[4], v[5]))
    c = None if v[6] == v[7] == 0 else (v[6], v[7])
    return a, b, c
